/* sliding_oracle.c — TEST-ONLY: the CPU oracle (oracle/ork_core.c, compiled in here unchanged) with the sliding-window mode of
 * arks_set_sliding_window and the rate-limit report (arks_set_ratelimit_report) under it, reset / retry included.
 *
 * The statement is Redis's: every counter keeps a second (window start, value) slot, the key its current slot held before a
 * newer window replaced it, and prev = GET(window start - W) over both slots. A request batch decides serially, row by row:
 * the limiter's GET of the current key returns cur + floor(prev * (W - e) / W), because the oracle adds that share to the
 * current key for the length of the batch (one timestamp per batch: the share is constant) and takes it back when the batch
 * commits. Every INCRBY in between lands on the same key, so the counters come out exact. reset / retry are found by
 * bisection with 128-bit products (the device splits the product instead; tests/test_sliding_window.py holds this bisection
 * to a linear scan). Built as its own library (tests/_build/libarks_oracle_sw.so) next to ork_json.c. */
#define ork_request_batch ork_request_batch_plain
#define ork_response_batch ork_response_batch_plain
#define ork_reload ork_reload_plain
#define ork_destroy ork_destroy_plain
#include "../oracle/ork_core.c"
#undef ork_request_batch
#undef ork_response_batch
#undef ork_reload
#undef ork_destroy

int ork_request_batch(ork* o, const arks_request_batch* b, arks_request_result* r);
int ork_response_batch(ork* o, const arks_response_batch* b, arks_response_result* r);
int ork_reload(ork* o, const arks_tables* t);
void ork_destroy(ork* o);
void ork_set_sliding_window(ork* o, int on);
void ork_set_ratelimit_report(ork* o, int on);
int ork_snapshot_rate_prev(ork* o, int64_t now, int64_t* c);
void ork_sliding_times(int64_t c, int64_t p, int64_t left, int64_t w, int64_t limit, int req, uint32_t* reset, uint32_t* retry);

/* per oracle: the switches and the second slot of each of its n_qos * 4 counters */
typedef struct {
  const ork* o;
  int sliding, report;
  uint32_t n;
  int64_t *win, *val;
} side;
static side g_side[64];
static pthread_mutex_t g_side_mu = PTHREAD_MUTEX_INITIALIZER;

static side* side_of(ork* o) {
  side* s = NULL;
  pthread_mutex_lock(&g_side_mu);
  for (int k = 0; k < 64 && !s; k++)
    if (g_side[k].o == o) s = &g_side[k];
  for (int k = 0; k < 64 && !s; k++)
    if (!g_side[k].o) {
      s = &g_side[k];
      memset(s, 0, sizeof *s);
      s->o = o;
    }
  pthread_mutex_unlock(&g_side_mu);
  if (s && s->n != o->n_qos * 4) { /* first use: no older key anywhere */
    s->n = o->n_qos * 4;
    s->win = (int64_t*)realloc(s->win, 8 * (size_t)s->n + 8);
    s->val = (int64_t*)calloc((size_t)s->n + 1, 8);
    for (uint32_t k = 0; k < s->n; k++) s->win[k] = INT64_MIN;
  }
  return s;
}

void ork_set_sliding_window(ork* o, int on) { side_of(o)->sliding = on != 0; }
void ork_set_ratelimit_report(ork* o, int on) { side_of(o)->report = on != 0; }

void ork_destroy(ork* o) {
  pthread_mutex_lock(&g_side_mu);
  for (int k = 0; k < 64; k++)
    if (g_side[k].o == o) {
      free(g_side[k].win);
      free(g_side[k].val);
      memset(&g_side[k], 0, sizeof g_side[k]);
    }
  pthread_mutex_unlock(&g_side_mu);
  ork_destroy_plain(o);
}

/* GET over both slots */
static int64_t get2(const ork* o, const side* s, size_t k, int64_t ws) {
  if (o->rate_win[k] == ws) return o->rate_val[k];
  return s->win[k] == ws ? s->val[k] : 0;
}
/* a key the next INCRBY would replace (its window is not now's) moves to the second slot first */
static void keep_older_keys(ork* o, side* s, int64_t now) {
  for (uint32_t q = 0; q < o->n_qos; q++)
    for (int rule = 0; rule < 4; rule++) {
      const size_t k = (size_t)q * 4 + (size_t)rule;
      if (o->rate_win[k] != ork_window_start(now, rule) && o->rate_win[k] != s->win[k]) {
        s->win[k] = o->rate_win[k];
        s->val[k] = o->rate_val[k];
      }
    }
}
static int64_t prev_of(const ork* o, const side* s, uint32_t q, int rule, int64_t now) {
  return get2(o, s, (size_t)q * 4 + (size_t)rule, ork_window_start(now, rule) - RULE_WINDOW[rule]);
}
static int64_t floordiv(__int128 a, int64_t w) {
  __int128 q = a / w;
  if (a % w != 0 && a < 0) q -= 1;
  return (int64_t)q;
}
static int64_t share_of(int64_t prev, int rule, int64_t now) {
  const int64_t w = RULE_WINDOW[rule], left = ork_window_start(now, rule) + w - now;
  return floordiv((__int128)prev * left, w);
}

/* E(d): the estimate d seconds ahead with no further traffic (c, p >= 0) */
static __int128 projected(int64_t c, int64_t p, int64_t d, int64_t left, int64_t w) {
  if (d < left) return (__int128)c + floordiv((__int128)p * (left - d), w);
  if (d < left + w) return floordiv((__int128)c * (left + w - d), w);
  return 0;
}
static uint32_t first_at_most(int64_t c, int64_t p, int64_t left, int64_t w, __int128 bound) {
  int64_t lo = 0, hi = left + w;
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo) / 2;
    if (projected(c, p, mid, left, w) <= bound) hi = mid;
    else lo = mid + 1;
  }
  return (uint32_t)lo;
}
void ork_sliding_times(int64_t c, int64_t p, int64_t left, int64_t w, int64_t limit, int req, uint32_t* reset, uint32_t* retry) {
  c = c < 0 ? 0 : c;
  p = p < 0 ? 0 : p;
  *reset = first_at_most(c, p, left, w, 0);
  *retry = limit >= req ? first_at_most(c, p, left, w, (__int128)limit - req) : *reset;
}

/* the figures of row i (tests/ratelimit_oracle.c's rule: per kind the entry with the least remaining, the first on a tie),
 * read from the serial state right after the row; with the sliding window also reset / retry */
static void report_row(const ork* o, const side* s, const int64_t* shares, const arks_request_batch* b, arks_request_result* r,
                       uint32_t i) {
  uint8_t e[2] = {ARKS_RL_NONE, ARKS_RL_NONE};
  int64_t lim[2] = {0, 0}, rem[2] = {0, 0};
  uint32_t reset[2] = {0, 0}, retry = 0;
  const int64_t now = b->now_unix;
  const uint8_t reason = r->reason[i];
  if (reason == ARKS_R_OK || reason == ARKS_R_RATE_LIMIT || reason == ARKS_R_QUOTA) {
    const uint32_t q = (uint32_t)r->qos[i], j0 = o->qos_rl_off[q];
    for (uint32_t j = j0; j < o->qos_rl_off[q + 1]; j++) {
      const int rule = o->rl_rule[j], t = RULE_IS_REQUEST[rule] ? 0 : 1;
      const int64_t c = rate_get(o, q, rule, ork_window_start(now, rule)), l = o->rl_value[j];
      const int64_t left = c >= l ? 0 : l - c;
      if (e[t] == ARKS_RL_NONE || left < rem[t]) {
        e[t] = (uint8_t)(j - j0);
        lim[t] = l;
        rem[t] = left;
        if (s->sliding) {
          const int64_t cc = (int64_t)((uint64_t)c - (uint64_t)shares[(size_t)q * 4 + rule]);
          uint32_t unused;
          ork_sliding_times(cc, prev_of(o, s, q, rule, now), ork_window_start(now, rule) + RULE_WINDOW[rule] - now,
                            RULE_WINDOW[rule], 0, 0, &reset[t], &unused);
        }
      }
    }
    if (reason == ARKS_R_RATE_LIMIT && s->sliding) {
      const int rule = o->rl_rule[j0 + r->detail[i]];
      const int64_t cc = (int64_t)((uint64_t)r->cur_usage[i] - (uint64_t)shares[(size_t)q * 4 + rule]);
      uint32_t unused;
      ork_sliding_times(cc, prev_of(o, s, q, rule, now), ork_window_start(now, rule) + RULE_WINDOW[rule] - now, RULE_WINDOW[rule],
                        r->limit_max[i], RULE_IS_REQUEST[rule], &unused, &retry);
    }
  }
  for (int t = 0; t < 2; t++) {
    if (r->rl_entry) r->rl_entry[2 * (size_t)i + t] = e[t];
    if (r->rl_limit) r->rl_limit[2 * (size_t)i + t] = lim[t];
    if (r->rl_remaining) r->rl_remaining[2 * (size_t)i + t] = rem[t];
    if (s->sliding && r->rl_reset) r->rl_reset[2 * (size_t)i + t] = reset[t];
  }
  if (s->sliding && r->rl_retry) r->rl_retry[i] = retry;
}

int ork_request_batch(ork* o, const arks_request_batch* b, arks_request_result* r) {
  int rc = check_time(o, b->now_unix);
  if (rc) return rc;
  side* s = side_of(o);
  const int64_t now = b->now_unix;
  keep_older_keys(o, s, now);
  int64_t* shares = (int64_t*)calloc((size_t)o->n_qos * 4 + 1, 8);
  if (s->sliding)
    for (uint32_t q = 0; q < o->n_qos; q++)
      for (int rule = 0; rule < 4; rule++) {
        const size_t k = (size_t)q * 4 + (size_t)rule;
        shares[k] = share_of(prev_of(o, s, q, rule, now), rule, now);
        if (shares[k]) rate_incr(o, q, rule, ork_window_start(now, rule), shares[k]); /* the older key is in the second slot */
      }
  for (uint32_t i = 0; i < b->n; i++) {
    handle_request(o, b, r, i, i);
    if (s->report) report_row(o, s, shares, b, r, i);
  }
  for (uint32_t k = 0; k < o->pc_n; k++) rate_incr(o, o->pc[k].q, o->pc[k].rule, ork_window_start(now, o->pc[k].rule), o->pc[k].amount);
  o->pc_n = 0;
  o->est = NULL;
  o->est_n = 0;
  for (uint32_t q = 0; q < o->n_qos; q++)
    for (int rule = 0; rule < 4; rule++)
      if (shares[(size_t)q * 4 + rule]) rate_incr(o, q, rule, ork_window_start(now, rule), (int64_t)(0 - (uint64_t)shares[(size_t)q * 4 + rule]));
  free(shares);
  return 0;
}

int ork_response_batch(ork* o, const arks_response_batch* b, arks_response_result* r) {
  int rc = check_time(o, b->now_unix);
  if (rc) return rc;
  keep_older_keys(o, side_of(o), b->now_unix);
  return ork_response_batch_plain(o, b, r);
}

int ork_snapshot_rate_prev(ork* o, int64_t now, int64_t* c) {
  const side* s = side_of(o);
  for (uint32_t q = 0; q < o->n_qos; q++)
    for (int rule = 0; rule < 4; rule++) c[(size_t)q * 4 + rule] = prev_of(o, s, q, rule, now);
  return 0;
}

/* both slots follow their key (namespace, user, model) into the new tables, as Redis keys outlive a CRD edit */
static void key_of(const ork* o, uint32_t q, char* out, size_t cap) {
  size_t a, b, c;
  const uint32_t tk = o->qos_token[q];
  const uint8_t* ns = S(o, o->tok_ns_str[tk], &a);
  const uint8_t* us = S(o, o->tok_name_str[tk], &b);
  const uint8_t* md = S(o, o->qos_model_str[q], &c);
  memset(out, 0, cap);
  snprintf(out, cap, "%.*s%c%.*s%c%.*s", (int)a, (const char*)ns, 0, (int)b, (const char*)us, 0, (int)c, (const char*)md);
}
int ork_reload(ork* o, const arks_tables* t) {
  side* s = side_of(o);
  const uint32_t n_old = o->n_qos;
  char(*old_keys)[800] = malloc(((size_t)n_old + 1) * 800);
  for (uint32_t q = 0; q < n_old; q++) key_of(o, q, old_keys[q], 800);
  int64_t *ow = s->win, *ov = s->val;
  const int rc = ork_reload_plain(o, t);
  if (rc) {
    free(old_keys);
    return rc;
  }
  s->n = o->n_qos * 4;
  s->win = (int64_t*)malloc(8 * (size_t)s->n + 8);
  s->val = (int64_t*)calloc((size_t)s->n + 1, 8);
  for (uint32_t k = 0; k < s->n; k++) s->win[k] = INT64_MIN;
  char key[800];
  for (uint32_t q = 0; q < o->n_qos; q++) {
    key_of(o, q, key, sizeof key);
    for (uint32_t p = 0; p < n_old; p++)
      if (!memcmp(key, old_keys[p], 800)) {
        memcpy(s->win + 4 * (size_t)q, ow + 4 * (size_t)p, 32);
        memcpy(s->val + 4 * (size_t)q, ov + 4 * (size_t)p, 32);
        break;
      }
  }
  free(ow);
  free(ov);
  free(old_keys);
  return 0;
}
