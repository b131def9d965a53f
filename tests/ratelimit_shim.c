/* ratelimit_shim.c — TEST-ONLY: tests/abi_shim.c (the CPU oracle behind the entry points the C++ host calls) with the
 * rate-limit report (arks_set_ratelimit_report) added around it, so that tests/test_ratelimit_headers.py can hold the C++
 * host's x-ratelimit-* / retry-after headers to the Python server's on the CPU. The figures come from the oracle's own report
 * mode (ork_set_ratelimit_report), parked per slot like the rest of a request batch's answer. */
#define arks_submit_request_async abi_shim_submit_request_async
#define arks_wait_request abi_shim_wait_request
#include "abi_shim.c"
#undef arks_submit_request_async
#undef arks_wait_request

static int g_report;
static struct {
  uint32_t cap;
  int on;
  uint8_t* entry;
  int64_t *limit, *remaining;
} g_rl[SHIM_SLOTS];

int arks_set_ratelimit_report(arks_ctx* c, int on) {
  g_report = on != 0;
  ork_set_ratelimit_report(c->o, on);
  return 0;
}

int arks_submit_request_async(arks_ctx* c, const arks_request_batch* b) {
  struct slot_res* s = &c->rq[c->cur];
  const uint32_t n = b->n ? b->n : 1;
  grow(s, n);
  s->n = b->n;
  if (g_rl[c->cur].cap < n) {
    g_rl[c->cur].cap = n;
    g_rl[c->cur].entry = realloc(g_rl[c->cur].entry, 2 * (size_t)n);
    g_rl[c->cur].limit = realloc(g_rl[c->cur].limit, 16 * (size_t)n);
    g_rl[c->cur].remaining = realloc(g_rl[c->cur].remaining, 16 * (size_t)n);
  }
  g_rl[c->cur].on = g_report;
  arks_request_result r = {s->reason, s->detail, s->flags, s->qos, s->token, s->pick, s->cur, s->lim, s->moff, s->mlen, s->bpe,
                           g_rl[c->cur].entry, g_rl[c->cur].limit, g_rl[c->cur].remaining};
  s->rc = shim_request(c, b, &r);
  return s->rc;
}

int arks_wait_request(arks_ctx* c, int slot, arks_request_result* out) {
  const int rc = abi_shim_wait_request(c, slot, out);
  const size_t n = c->rq[slot].n;
  if (g_rl[slot].on) {  /* like the library: a batch run without the report leaves the caller's arrays untouched */
    if (out->rl_entry) memcpy(out->rl_entry, g_rl[slot].entry, 2 * n);
    if (out->rl_limit) memcpy(out->rl_limit, g_rl[slot].limit, 16 * n);
    if (out->rl_remaining) memcpy(out->rl_remaining, g_rl[slot].remaining, 16 * n);
  }
  return rc;
}
