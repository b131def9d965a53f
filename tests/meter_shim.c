/* meter_shim.c — TEST-ONLY: tests/abi_shim.c (the CPU oracle behind the entry points the C++ host calls) with stream metering
 * (N5, arks_set_stream_metering) added around it, so that tests/test_stream_metering.py can check on the CPU that the host's
 * StreamProcessor carries ARKS_FLAG_METERED from a request decision to every response chunk of that stream.
 *   requests: with metering on, a stream:true body without "include_usage":true is decided as the same body with
 *             ,"stream_options":{"include_usage":true} appended as its last member, and marked ARKS_FLAG_METERED if admitted;
 *   responses: the flags of every row are logged (meter_shim_log) before the oracle answers the batch.
 * The billing itself is not modelled here (tests/meter_model.py does that). */
#define arks_submit_request_async abi_shim_submit_request_async
#define arks_submit_response_async abi_shim_submit_response_async
#include "abi_shim.c"
#undef arks_submit_request_async
#undef arks_submit_response_async

static int g_meter;
static uint8_t g_log_flags[1 << 16];
static int32_t g_log_qos[1 << 16];
static uint32_t g_log_n;

int arks_set_stream_metering(arks_ctx* c, int on) { (void)c; g_meter = on != 0; return 0; }

static int metered_body(const uint8_t* p, uint32_t n) {
  const char* s = "\"stream\":true";
  const char* u = "\"include_usage\":true";
  int stream = 0, usage = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (i + 13 <= n && !memcmp(p + i, s, 13)) stream = 1;
    if (i + 20 <= n && !memcmp(p + i, u, 20)) usage = 1;
  }
  return stream && !usage;
}

int arks_submit_request_async(arks_ctx* c, const arks_request_batch* b) {
  if (!g_meter || !b->n) return abi_shim_submit_request_async(c, b);
  static const char add[] = ",\"stream_options\":{\"include_usage\":true}";
  const uint32_t extra = sizeof add - 1;
  uint8_t* mark = (uint8_t*)calloc(b->n, 1);
  uint32_t* off = (uint32_t*)malloc(4 * (size_t)b->n);
  uint32_t* len = (uint32_t*)malloc(4 * (size_t)b->n);
  uint8_t* bodies = (uint8_t*)malloc(b->bodies_bytes + (size_t)b->n * (extra + 16) + 16);
  uint64_t w = 0;
  for (uint32_t i = 0; i < b->n; i++) {
    const uint8_t* p = b->bodies + b->body_off[i];
    uint32_t n = b->body_len[i], k = n;
    mark[i] = (uint8_t)metered_body(p, n);
    while (mark[i] && k > 0 && p[k - 1] != '}') k--;
    if (!k) mark[i] = 0;
    off[i] = (uint32_t)w;
    if (mark[i]) {
      memcpy(bodies + w, p, k - 1);
      memcpy(bodies + w + k - 1, add, extra);
      memcpy(bodies + w + k - 1 + extra, p + k - 1, n - k + 1);
      n += extra;
    } else {
      memcpy(bodies + w, p, n);
    }
    len[i] = n;
    w = (w + n + 15) & ~(uint64_t)15;
  }
  arks_request_batch b2 = *b;
  b2.bodies = bodies; b2.body_off = off; b2.body_len = len; b2.bodies_bytes = w;
  const int rc = abi_shim_submit_request_async(c, &b2);
  struct slot_res* s = &c->rq[c->cur];
  for (uint32_t i = 0; i < b->n; i++)
    if (mark[i] && s->reason[i] == ARKS_R_OK) s->flags[i] |= ARKS_FLAG_METERED;
  free(mark); free(off); free(len); free(bodies);
  return rc;
}

int arks_submit_response_async(arks_ctx* c, const arks_response_batch* b) {
  for (uint32_t i = 0; i < b->n && g_log_n < sizeof g_log_flags; i++, g_log_n++) {
    g_log_flags[g_log_n] = b->flags[i];
    g_log_qos[g_log_n] = b->qos[i];
  }
  return abi_shim_submit_response_async(c, b);
}

/* response rows seen since the last call: their flags and qos, in submission order */
uint32_t meter_shim_log(uint8_t* flags, int32_t* qos, uint32_t cap) {
  const uint32_t n = g_log_n < cap ? g_log_n : cap;
  memcpy(flags, g_log_flags, n);
  memcpy(qos, g_log_qos, 4 * (size_t)n);
  g_log_n = 0;
  return n;
}
