/* ratelimit_oracle.c — TEST-ONLY: the CPU oracle (oracle/ork_core.c, compiled in here unchanged) with a report mode for
 * arks_set_ratelimit_report. With the mode on, ork_request_batch reads every row's figures from the oracle's SERIAL state
 * right after that row was decided: the request-type counters with this row's own increment applied, the token-type
 * counters as the checks read them (N4 pre-charges land when the batch commits). This is a second statement of the numbers
 * the device derives in closed form (arrival rank, admitted count, duplicate entries), and the tests hold one to the other.
 * Built as its own library (tests/_build/libarks_oracle_rl.so) next to ork_json.c; every other ork_* entry point is the
 * oracle's. */
#define ork_request_batch ork_request_batch_plain
#include "../oracle/ork_core.c"
#undef ork_request_batch

int ork_request_batch(ork* o, const arks_request_batch* b, arks_request_result* r);
void ork_set_ratelimit_report(ork* o, int on);

/* oracles with the mode on (a test process holds a handful) */
static const ork* g_on[64];
static pthread_mutex_t g_on_mu = PTHREAD_MUTEX_INITIALIZER;

static int report_on(const ork* o) {
  int on = 0;
  pthread_mutex_lock(&g_on_mu);
  for (int k = 0; k < 64; k++) on |= g_on[k] == o;
  pthread_mutex_unlock(&g_on_mu);
  return on;
}
void ork_set_ratelimit_report(ork* o, int on) {
  pthread_mutex_lock(&g_on_mu);
  for (int k = 0; k < 64; k++)
    if (g_on[k] == o) g_on[k] = NULL;
  for (int k = 0; on && k < 64; k++)
    if (!g_on[k]) { g_on[k] = o; break; }
  pthread_mutex_unlock(&g_on_mu);
}

/* the figures of row i: per kind the entry with the least remaining, the first one in qos.RateLimits order on a tie */
static void report_request(const ork* o, const arks_request_batch* b, arks_request_result* r, uint32_t i) {
  uint8_t e[2] = {ARKS_RL_NONE, ARKS_RL_NONE};
  int64_t lim[2] = {0, 0}, rem[2] = {0, 0};
  const uint8_t reason = r->reason[i];
  if (reason == ARKS_R_OK || reason == ARKS_R_RATE_LIMIT || reason == ARKS_R_QUOTA) {
    const uint32_t q = (uint32_t)r->qos[i], j0 = o->qos_rl_off[q];
    for (uint32_t j = j0; j < o->qos_rl_off[q + 1]; j++) {
      const int rule = o->rl_rule[j], t = RULE_IS_REQUEST[rule] ? 0 : 1;
      const int64_t c = rate_get(o, q, rule, ork_window_start(b->now_unix, rule)), l = o->rl_value[j];
      const int64_t left = c >= l ? 0 : l - c;
      if (e[t] == ARKS_RL_NONE || left < rem[t]) {
        e[t] = (uint8_t)(j - j0);
        lim[t] = l;
        rem[t] = left;
      }
    }
  }
  for (int t = 0; t < 2; t++) {
    if (r->rl_entry) r->rl_entry[2 * (size_t)i + t] = e[t];
    if (r->rl_limit) r->rl_limit[2 * (size_t)i + t] = lim[t];
    if (r->rl_remaining) r->rl_remaining[2 * (size_t)i + t] = rem[t];
  }
}

/* ork_request_batch_plain with the report after every row */
int ork_request_batch(ork* o, const arks_request_batch* b, arks_request_result* r) {
  if (!report_on(o)) return ork_request_batch_plain(o, b, r);
  int rc = check_time(o, b->now_unix);
  if (rc) return rc;
  for (uint32_t i = 0; i < b->n; i++) {
    handle_request(o, b, r, i, i);
    report_request(o, b, r, i);
  }
  for (uint32_t k = 0; k < o->pc_n; k++) rate_incr(o, o->pc[k].q, o->pc[k].rule, ork_window_start(b->now_unix, o->pc[k].rule), o->pc[k].amount);
  o->pc_n = 0;
  o->est = NULL;
  o->est_n = 0;
  return 0;
}
