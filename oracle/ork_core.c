/*
 * ork_core.c — oracle: config lookup, fixed-window limiter, quota, the four phase handlers.
 * TEST INFRASTRUCTURE ONLY (see arks_oracle.h). Redis is replaced by in-memory int64 counters with the
 * Redis semantics the decisions depend on: GET of a missing key = 0, INCRBY creates at 0, the
 * rate-limit key embeds the window start so TTLs never influence a decision (SURVEY.md §8c).
 *
 * Restated reference functions (paths relative to the reference tree):
 *   HandleRequestHeaders   pkg/gateway/handle_request.go:33-81
 *   HandleRequestBody      pkg/gateway/handle_request.go:83-249
 *   HandleResponseBody     pkg/gateway/handle_response.go:80-268
 *   checkRateLimit / checkTokenQuotaLimit / do*Limit   pkg/gateway/check.go:31-156
 *   RedisRateLimter.CheckLimit / DoLimit               pkg/gateway/ratelimiter/redis_impl.go:47-168
 *   CacheKeyGenerator.Generate / getWindowStart        pkg/gateway/ratelimiter/cache_key.go:42-80
 *   RedisQuotaService.IncrUsage/SetUsage/GetUsage      pkg/gateway/quota/redis_impl.go:38-107
 *   QosToQuotaRequests                                 pkg/gateway/qosconfig/types.go:45-72
 *   GetQosByToken / GetQuotaConfig / GetModelList      pkg/gateway/qosconfig/arks_impl.go:303-376
 */
#define _POSIX_C_SOURCE 200809L
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "ork_internal.h"

typedef struct {
  uint32_t* slot; /* value + 1, 0 = empty */
  uint32_t mask;
} strmap;

struct ork {
  /* deep copy of the tables */
  uint8_t* str_bytes;
  uint32_t* str_off;
  uint32_t n_str;
  uint32_t n_tokens, *tok_token_str, *tok_ns_str, *tok_name_str, *tok_qos_off;
  uint32_t n_qos, *qos_model_str, *qos_rl_off;
  int32_t* qos_quota;
  uint32_t n_rl;
  uint8_t* rl_rule;
  int64_t* rl_value;
  uint32_t n_quotas, *quota_ns_str, *quota_name_str, *quota_item_off;
  uint32_t n_qitems;
  uint8_t* qitem_type;
  int64_t* qitem_value;
  uint32_t n_endpoints, *ep_ns_str, *ep_name_str, *ep_backend_off;
  uint32_t n_backends;
  int32_t* backend_weight;
  /* derived */
  uint32_t* qos_token; /* qos entry -> owning token */
  strmap tok_map;      /* spec.token bytes -> token index (first wins) */
  strmap ep_map;       /* namespace \0 name -> endpoint index */
  /* mutable state: what Redis holds in the reference */
  int64_t* rate_win; /* n_qos * 4: window start the value belongs to (the key suffix) */
  int64_t* rate_val; /* n_qos * 4 */
  int64_t* quota_use; /* n_quotas * 3 */
  int64_t* metrics;   /* n_qos * ARKS_METRIC_COLS: the Prometheus series that are functions of the request stream */
  int64_t last_win[4];
  /* N4 (opt-in precharge, include/arks_gateway.h arks_set_precharge): the estimates of the NEXT request batch (the oracle has
   * no tokenizer: the test hands it the counts) and what that batch charges when it commits */
  int precharge;
  const uint32_t* est;
  uint32_t est_n;
  struct { uint32_t q; int rule; int64_t amount; }* pc;
  uint32_t pc_n, pc_cap;
};

/* ---------- small helpers ---------- */
static const int64_t RULE_WINDOW[4] = {60, 86400, 60, 86400}; /* rate_limiter.go:35-65, types.go:35-47 */
static const int RULE_IS_REQUEST[4] = {1, 1, 0, 0};
static const char* RULE_NAME[4] = {"rpm", "rpd", "tpm", "tpd"};
static const char* QT_NAME[3] = {"prompt", "response", "total"};

static const uint8_t* S(const ork* o, uint32_t id, size_t* len) {
  *len = o->str_off[id + 1] - o->str_off[id];
  return o->str_bytes + o->str_off[id];
}
static int str_eq(const ork* o, uint32_t id, const uint8_t* p, size_t n) {
  size_t l;
  const uint8_t* s = S(o, id, &l);
  return l == n && memcmp(s, p, n) == 0;
}
static uint64_t fnv64(const uint8_t* p, size_t n, uint64_t h) {
  for (size_t i = 0; i < n; i++) {
    h ^= p[i];
    h *= 0x100000001b3ull;
  }
  return h;
}
static void* dup_arr(const void* p, size_t n, size_t sz) {
  void* q = malloc(n * sz + 1);
  if (n && p) memcpy(q, p, n * sz);
  return q;
}
static void map_init(strmap* m, uint32_t n) {
  uint32_t cap = 16;
  while (cap < 2 * n + 2) cap <<= 1;
  m->slot = (uint32_t*)calloc(cap, sizeof(uint32_t));
  m->mask = cap - 1;
}

/* getWindowStart: time.Unix(now,0).Truncate(W).Unix(). Go truncates relative to year 1; the offset
 * 62135596800 s is a multiple of 1, 60, 3600 and 86400, so this is floor(now / W) * W. */
int64_t ork_window_start(int64_t now, int rule) {
  int64_t w = RULE_WINDOW[rule & 3];
  int64_t abs = now + 62135596800LL; /* seconds since year 1, as time.Time stores it */
  int64_t r = abs % w;
  if (r < 0) r += w;
  return now - r;
}

size_t ork_rate_key(const char* prefix, const char* ns, const char* user, const char* model, int rule,
                    int64_t now, char* out, size_t cap) {
  return (size_t)snprintf(out, cap, "%s:namespace=%s.user=%s.model=%s.%s:%lld", prefix, ns, user, model,
                          RULE_NAME[rule & 3], (long long)ork_window_start(now, rule));
}
size_t ork_quota_key(const char* prefix, const char* ns, const char* quota, int type, char* out, size_t cap) {
  return (size_t)snprintf(out, cap, "%s:namespace=%s.quotaname=%s.type=%s.", prefix, ns, quota, QT_NAME[type % 3]);
}

int32_t ork_weighted_pick(const int32_t* w, uint32_t n, uint64_t r) {
  uint64_t sum = 0;
  for (uint32_t i = 0; i < n; i++) sum += (uint64_t)(w[i] > 0 ? w[i] : 0);
  if (sum == 0) return -1;
  uint64_t x = r % sum, acc = 0;
  for (uint32_t i = 0; i < n; i++) {
    acc += (uint64_t)(w[i] > 0 ? w[i] : 0);
    if (x < acc) return (int32_t)i;
  }
  return -1;
}

/* HandleRequestHeaders, handle_request.go:38-46: strings.ToLower(key) == "authorization",
 * value has prefix "Bearer " -> rest of the value; stop at the first such header even if the rest is
 * empty?  No: `break` is inside the HasPrefix branch, so a header with prefix "Bearer " ends the scan
 * (token may be ""), one without the prefix does not. */
size_t ork_extract_bearer(const uint8_t* const* keys, const size_t* key_lens, const uint8_t* const* values,
                          const size_t* value_lens, size_t n_headers, const uint8_t** token) {
  static const char A[] = "authorization";
  *token = NULL;
  for (size_t i = 0; i < n_headers; i++) {
    if (key_lens[i] != 13) continue;
    int ok = 1;
    for (int k = 0; k < 13; k++) {
      uint8_t c = keys[i][k];
      if (c >= 'A' && c <= 'Z') c += 32; /* strings.ToLower on an ASCII key; non-ASCII keys cannot match */
      if (c != (uint8_t)A[k]) ok = 0;
    }
    if (!ok) continue;
    if (value_lens[i] >= 7 && memcmp(values[i], "Bearer ", 7) == 0) {
      *token = values[i] + 7;
      return value_lens[i] - 7;
    }
  }
  return 0;
}

/* ---------- table load ---------- */
static void ork_free_tables(ork* o) {
  free(o->str_bytes); free(o->str_off);
  free(o->tok_token_str); free(o->tok_ns_str); free(o->tok_name_str); free(o->tok_qos_off);
  free(o->qos_model_str); free(o->qos_rl_off); free(o->qos_quota);
  free(o->rl_rule); free(o->rl_value);
  free(o->quota_ns_str); free(o->quota_name_str); free(o->quota_item_off);
  free(o->qitem_type); free(o->qitem_value);
  free(o->ep_ns_str); free(o->ep_name_str); free(o->ep_backend_off); free(o->backend_weight);
  free(o->qos_token); free(o->tok_map.slot); free(o->ep_map.slot);
}

static uint64_t ep_hash(const uint8_t* ns, size_t nl, const uint8_t* nm, size_t ml) {
  uint64_t h = fnv64(ns, nl, 0xcbf29ce484222325ull);
  h = fnv64((const uint8_t*)"\0", 1, h);
  return fnv64(nm, ml, h);
}

static int ork_load(ork* o, const arks_tables* t) {
  o->n_str = t->n_str;
  o->str_off = (uint32_t*)dup_arr(t->str_off, t->n_str + 1, 4);
  o->str_bytes = (uint8_t*)dup_arr(t->str_bytes, t->n_str ? t->str_off[t->n_str] : 0, 1);
  o->n_tokens = t->n_tokens;
  o->tok_token_str = (uint32_t*)dup_arr(t->tok_token_str, t->n_tokens, 4);
  o->tok_ns_str = (uint32_t*)dup_arr(t->tok_ns_str, t->n_tokens, 4);
  o->tok_name_str = (uint32_t*)dup_arr(t->tok_name_str, t->n_tokens, 4);
  o->tok_qos_off = (uint32_t*)dup_arr(t->tok_qos_off, t->n_tokens + 1, 4);
  o->n_qos = t->n_qos;
  o->qos_model_str = (uint32_t*)dup_arr(t->qos_model_str, t->n_qos, 4);
  o->qos_quota = (int32_t*)dup_arr(t->qos_quota, t->n_qos, 4);
  o->qos_rl_off = (uint32_t*)dup_arr(t->qos_rl_off, t->n_qos + 1, 4);
  o->n_rl = t->n_rl;
  o->rl_rule = (uint8_t*)dup_arr(t->rl_rule, t->n_rl, 1);
  o->rl_value = (int64_t*)dup_arr(t->rl_value, t->n_rl, 8);
  o->n_quotas = t->n_quotas;
  o->quota_ns_str = (uint32_t*)dup_arr(t->quota_ns_str, t->n_quotas, 4);
  o->quota_name_str = (uint32_t*)dup_arr(t->quota_name_str, t->n_quotas, 4);
  o->quota_item_off = (uint32_t*)dup_arr(t->quota_item_off, t->n_quotas + 1, 4);
  o->n_qitems = t->n_qitems;
  o->qitem_type = (uint8_t*)dup_arr(t->qitem_type, t->n_qitems, 1);
  o->qitem_value = (int64_t*)dup_arr(t->qitem_value, t->n_qitems, 8);
  o->n_endpoints = t->n_endpoints;
  o->ep_ns_str = (uint32_t*)dup_arr(t->ep_ns_str, t->n_endpoints, 4);
  o->ep_name_str = (uint32_t*)dup_arr(t->ep_name_str, t->n_endpoints, 4);
  o->ep_backend_off = (uint32_t*)dup_arr(t->ep_backend_off, t->n_endpoints + 1, 4);
  o->n_backends = t->n_backends;
  o->backend_weight = (int32_t*)dup_arr(t->backend_weight, t->n_backends, 4);

  for (uint32_t i = 0; i < o->n_rl; i++)
    if (o->rl_rule[i] >= ARKS_N_RULES) return ARKS_E_BAD_TABLE;
  for (uint32_t i = 0; i < o->n_qitems; i++)
    if (o->qitem_type[i] >= ARKS_N_QT) return ARKS_E_BAD_TABLE;
  for (uint32_t q = 0; q < o->n_qos; q++) {
    if (o->qos_rl_off[q + 1] - o->qos_rl_off[q] > 255) return ARKS_E_BAD_TABLE;
    if (o->qos_quota[q] >= (int32_t)o->n_quotas || o->qos_quota[q] < ARKS_QUOTA_MISSING) return ARKS_E_BAD_TABLE;
  }
  for (uint32_t q = 0; q < o->n_quotas; q++)
    if (o->quota_item_off[q + 1] - o->quota_item_off[q] > 255) return ARKS_E_BAD_TABLE;

  o->qos_token = (uint32_t*)malloc((o->n_qos + 1) * 4);
  for (uint32_t k = 0; k < o->n_tokens; k++)
    for (uint32_t q = o->tok_qos_off[k]; q < o->tok_qos_off[k + 1]; q++) o->qos_token[q] = k;

  map_init(&o->tok_map, o->n_tokens);
  for (uint32_t k = 0; k < o->n_tokens; k++) {
    size_t l;
    const uint8_t* s = S(o, o->tok_token_str[k], &l);
    uint32_t h = (uint32_t)fnv64(s, l, 0xcbf29ce484222325ull) & o->tok_map.mask;
    for (;;) {
      uint32_t v = o->tok_map.slot[h];
      if (!v) {
        o->tok_map.slot[h] = k + 1;
        break;
      }
      if (str_eq(o, o->tok_token_str[v - 1], s, l)) break; /* first object with this spec.token wins */
      h = (h + 1) & o->tok_map.mask;
    }
  }
  map_init(&o->ep_map, o->n_endpoints);
  for (uint32_t e = 0; e < o->n_endpoints; e++) {
    size_t nl, ml;
    const uint8_t* ns = S(o, o->ep_ns_str[e], &nl);
    const uint8_t* nm = S(o, o->ep_name_str[e], &ml);
    uint32_t h = (uint32_t)ep_hash(ns, nl, nm, ml) & o->ep_map.mask;
    for (;;) {
      uint32_t v = o->ep_map.slot[h];
      if (!v) {
        o->ep_map.slot[h] = e + 1;
        break;
      }
      if (str_eq(o, o->ep_ns_str[v - 1], ns, nl) && str_eq(o, o->ep_name_str[v - 1], nm, ml)) break;
      h = (h + 1) & o->ep_map.mask;
    }
  }
  return 0;
}

ork* ork_create(const arks_tables* t) {
  ork* o = (ork*)calloc(1, sizeof(ork));
  if (ork_load(o, t) != 0) {
    ork_free_tables(o);
    free(o);
    return NULL;
  }
  o->rate_win = (int64_t*)calloc((size_t)o->n_qos * 4 + 1, 8);
  o->rate_val = (int64_t*)calloc((size_t)o->n_qos * 4 + 1, 8);
  o->quota_use = (int64_t*)calloc((size_t)o->n_quotas * 3 + 1, 8);
  o->metrics = (int64_t*)calloc((size_t)o->n_qos * ARKS_METRIC_COLS + 1, 8);
  for (int r = 0; r < 4; r++) o->last_win[r] = INT64_MIN;
  return o;
}
void ork_destroy(ork* o) {
  if (!o) return;
  ork_free_tables(o);
  free(o->rate_win);
  free(o->rate_val);
  free(o->quota_use);
  free(o->metrics);
  free(o->pc);
  free(o);
}

/* reload: counters are carried over by key — (namespace,user,model) and (namespace,quotaName) —
 * exactly as Redis keys outlive a CRD edit. */
int ork_reload(ork* o, const arks_tables* t) {
  ork* n = ork_create(t);
  if (!n) return ARKS_E_BAD_TABLE;
  for (uint32_t q = 0; q < n->n_qos; q++) {
    uint32_t tk = n->qos_token[q];
    size_t a, b, c;
    const uint8_t* ns = S(n, n->tok_ns_str[tk], &a);
    const uint8_t* us = S(n, n->tok_name_str[tk], &b);
    const uint8_t* md = S(n, n->qos_model_str[q], &c);
    for (uint32_t p = 0; p < o->n_qos; p++) {
      uint32_t tp = o->qos_token[p];
      if (str_eq(o, o->tok_ns_str[tp], ns, a) && str_eq(o, o->tok_name_str[tp], us, b) &&
          str_eq(o, o->qos_model_str[p], md, c)) {
        memcpy(n->rate_win + 4 * (size_t)q, o->rate_win + 4 * (size_t)p, 32);
        memcpy(n->rate_val + 4 * (size_t)q, o->rate_val + 4 * (size_t)p, 32);
        memcpy(n->metrics + ARKS_METRIC_COLS * (size_t)q, o->metrics + ARKS_METRIC_COLS * (size_t)p, 8 * ARKS_METRIC_COLS);
        break;
      }
    }
  }
  for (uint32_t q = 0; q < n->n_quotas; q++) {
    size_t a, b;
    const uint8_t* ns = S(n, n->quota_ns_str[q], &a);
    const uint8_t* nm = S(n, n->quota_name_str[q], &b);
    for (uint32_t p = 0; p < o->n_quotas; p++)
      if (str_eq(o, o->quota_ns_str[p], ns, a) && str_eq(o, o->quota_name_str[p], nm, b)) {
        memcpy(n->quota_use + 3 * (size_t)q, o->quota_use + 3 * (size_t)p, 24);
        break;
      }
  }
  memcpy(n->last_win, o->last_win, sizeof o->last_win);
  ork tmp = *o;
  *o = *n;
  *n = tmp;
  ork_destroy(n);
  return 0;
}

int ork_update_endpoint_weights(ork* o, uint32_t ep, uint32_t n, const int32_t* w) {
  if (ep >= o->n_endpoints) return ARKS_E_INVALID_ARG;
  if (o->ep_backend_off[ep + 1] - o->ep_backend_off[ep] != n) return ARKS_E_INVALID_ARG;
  memcpy(o->backend_weight + o->ep_backend_off[ep], w, n * 4);
  return 0;
}

/* ---------- lookups (qosconfig/arks_impl.go:303-376) ---------- */
static int32_t find_token(const ork* o, const uint8_t* tk, size_t n) {
  uint32_t h = (uint32_t)fnv64(tk, n, 0xcbf29ce484222325ull) & o->tok_map.mask;
  for (;;) {
    uint32_t v = o->tok_map.slot[h];
    if (!v) return -1;
    if (str_eq(o, o->tok_token_str[v - 1], tk, n)) return (int32_t)(v - 1);
    h = (h + 1) & o->tok_map.mask;
  }
}
static int32_t find_endpoint(const ork* o, uint32_t ns_str, const uint8_t* model, size_t ml) {
  size_t nl;
  const uint8_t* ns = S(o, ns_str, &nl);
  uint32_t h = (uint32_t)ep_hash(ns, nl, model, ml) & o->ep_map.mask;
  for (;;) {
    uint32_t v = o->ep_map.slot[h];
    if (!v) return -1;
    if (str_eq(o, o->ep_ns_str[v - 1], ns, nl) && str_eq(o, o->ep_name_str[v - 1], model, ml))
      return (int32_t)(v - 1);
    h = (h + 1) & o->ep_map.mask;
  }
}

/* Redis GET of "<prefix>:<identifier>.<rule>:<windowStart>" */
static int64_t rate_get(const ork* o, uint32_t q, int rule, int64_t ws) {
  size_t k = (size_t)q * 4 + (size_t)rule;
  return o->rate_win[k] == ws ? o->rate_val[k] : 0;
}
/* Redis INCRBY on the same key */
static void rate_incr(ork* o, uint32_t q, int rule, int64_t ws, int64_t n) {
  size_t k = (size_t)q * 4 + (size_t)rule;
  if (o->rate_win[k] != ws) {
    o->rate_win[k] = ws;
    o->rate_val[k] = 0;
  }
  o->rate_val[k] = (int64_t)((uint64_t)o->rate_val[k] + (uint64_t)n);
}

static int check_time(ork* o, int64_t now) {
  for (int r = 0; r < 4; r++) {
    int64_t ws = ork_window_start(now, r);
    if (ws < o->last_win[r]) return ARKS_E_TIME_WENT_BACK;
  }
  for (int r = 0; r < 4; r++) o->last_win[r] = ork_window_start(now, r);
  return 0;
}

/* ---------- HandleRequestBody ---------- */
/* row i of the batch; results go to row `out` of r (out == i except for the threaded baseline's private buffers) */
static void handle_request(ork* o, const arks_request_batch* b, arks_request_result* r, uint32_t i, uint32_t out) {
  const uint8_t* body = b->bodies + b->body_off[i];
  size_t len = b->body_len[i];
  const uint8_t* tk = b->tokens + b->token_off[i];
  size_t tkl = b->token_off[i + 1] - b->token_off[i];
  r->reason[out] = ARKS_R_OK;
  r->detail[out] = 0;
  r->flags[out] = 0;
  r->qos[out] = -1;
  r->token[out] = -1;
  r->pick[out] = -1;
  r->cur_usage[out] = 0;
  r->limit_max[out] = 0;

  /* 1. jsonUnmarshal(body, &reqBody)                                   handle_request.go:97-104 */
  uint8_t mbuf[1024];
  ork_sink model = {mbuf, 0, sizeof mbuf, 0, 0};
  int stream3, so_present, iu3;
  uint32_t span[2];
  int bad = ork_json_request(body, len, &model, &stream3, &so_present, &iu3, span);
  if (r->model_off) r->model_off[out] = span[0];
  if (r->model_len) r->model_len[out] = span[1];
  if (r->bpe_count) r->bpe_count[out] = 0; /* the BPE counter has no reference implementation: its oracle is HF tokenizers */
  if (bad) {
    r->reason[out] = ARKS_R_REQUEST_BODY;
    return;
  }
  /* 2. model == ""                                                     :106-115 */
  if (model.len == 0) {
    r->reason[out] = ARKS_R_NO_MODEL;
    return;
  }
  /* 3. GetQosByToken(token, model)                                     :118-134, arks_impl.go:303-338 */
  int32_t t = find_token(o, tk, tkl);
  if (t < 0) {
    r->reason[out] = ARKS_R_TOKEN_NOT_FOUND;
    return;
  }
  r->token[out] = t;
  int32_t q = -1;
  if (model.len <= model.cap) /* names longer than the sink cannot equal a (<= 253 byte) object name */
    for (uint32_t k = o->tok_qos_off[t]; k < o->tok_qos_off[t + 1]; k++)
      if (str_eq(o, o->qos_model_str[k], mbuf, model.len)) {
        q = (int32_t)k;
        break;
      }
  if (q < 0) {
    r->reason[out] = ARKS_R_MODEL_NOT_IN_TOKEN;
    return;
  }
  r->qos[out] = q;
  /* 4. GetModelList(qos.Namespace) contains model                      :137-154, arks_impl.go:364-376 */
  int32_t ep = find_endpoint(o, o->tok_ns_str[t], mbuf, model.len);
  if (ep < 0) {
    r->reason[out] = ARKS_R_NO_MODEL_BACKENDS;
    return;
  }
  /* 5. stream requires stream_options.include_usage == true            :156-171 */
  int stream = stream3 == 2;
  if (stream && !(so_present && iu3 == 2)) {
    r->reason[out] = ARKS_R_STREAM_OPTIONS;
    return;
  }
  /* 6. checkRateLimit -> CheckLimit                                    check.go:108-156, redis_impl.go:47-114 */
  uint32_t rl0 = o->qos_rl_off[q], rl1 = o->qos_rl_off[q + 1];
  for (uint32_t j = rl0; j < rl1; j++) {
    int rule = o->rl_rule[j];
    int64_t ws = ork_window_start(b->now_unix, rule);
    int64_t cur = rate_get(o, (uint32_t)q, rule, ws);
    int64_t req = RULE_IS_REQUEST[rule] ? 1 : 0; /* "token is not caculated in request" check.go:124-126 */
    if ((int64_t)((uint64_t)cur + (uint64_t)req) > o->rl_value[j]) {
      r->reason[out] = ARKS_R_RATE_LIMIT;
      o->metrics[(size_t)q * ARKS_METRIC_COLS + ARKS_METRIC_HITS + rule]++; /* RecordRateLimitHit, check.go:145 */
      r->detail[out] = (uint8_t)(j - rl0);
      r->cur_usage[out] = cur;
      r->limit_max[out] = o->rl_value[j];
      return;
    }
  }
  /* 7. checkTokenQuotaLimit -> GetUsage: cur > limit (strict)          check.go:75-106, quota/redis_impl.go:63-107 */
  int32_t qt = o->qos_quota[q];
  if (qt == ARKS_QUOTA_MISSING) {
    r->reason[out] = ARKS_R_QUOTA_CONFIG;
    return;
  }
  if (qt >= 0) {
    uint32_t i0 = o->quota_item_off[qt], i1 = o->quota_item_off[qt + 1];
    for (uint32_t j = i0; j < i1; j++) {
      int64_t cur = o->quota_use[(size_t)qt * 3 + o->qitem_type[j]];
      if (cur > o->qitem_value[j]) {
        r->reason[out] = ARKS_R_QUOTA;
        r->detail[out] = (uint8_t)(j - i0);
        r->cur_usage[out] = cur;
        r->limit_max[out] = o->qitem_value[j];
        return;
      }
    }
  }
  /* 8. doRequestRateLimit -> DoLimit: INCRBY 1 per request-type entry  check.go:31-44, redis_impl.go:116-168 */
  for (uint32_t j = rl0; j < rl1; j++) {
    int rule = o->rl_rule[j];
    if (RULE_IS_REQUEST[rule]) rate_incr(o, (uint32_t)q, rule, ork_window_start(b->now_unix, rule), 1);
    else if (o->precharge && o->est && i < o->est_n && o->est[i] && o->est[i] != 0xFFFFFFFFu) {
      /* N4: the estimate is charged when the batch commits (ork_request_batch): checks inside the batch see the batch's start */
      if (o->pc_n == o->pc_cap) {
        o->pc_cap = o->pc_cap ? 2 * o->pc_cap : 1024;
        o->pc = realloc(o->pc, o->pc_cap * sizeof *o->pc);
      }
      o->pc[o->pc_n].q = (uint32_t)q; o->pc[o->pc_n].rule = rule; o->pc[o->pc_n].amount = o->est[i];
      o->pc_n++;
    }
  }
  /* 9. BodyResponse{model, namespace, username}; weighted pick is Envoy's (A12) */
  r->flags[out] = stream ? 1 : 0;
  if (b->pick_rand) {
    uint32_t b0 = o->ep_backend_off[ep], b1 = o->ep_backend_off[ep + 1];
    r->pick[out] = ork_weighted_pick(o->backend_weight + b0, b1 - b0, b->pick_rand[i]);
  }
}

/* bucket of gateway_token_distribution: ExponentialBuckets(1, 2, 17) + Inf, metrics.go:62-69 */
static int token_bucket(int64_t v) {
  int64_t le = 1;
  for (int k = 0; k < ARKS_METRIC_HIST_BUCKETS - 1; k++, le *= 2)
    if (v <= le) return k;
  return ARKS_METRIC_HIST_BUCKETS - 1;
}
static void handle_response_inner(ork* o, const arks_response_batch* b, arks_response_result* r, uint32_t i, uint32_t out);
/* Server.Process + the deferred block of HandleResponseBody: gateway.go:122-129, handle_response.go:99-109 */
static void handle_response(ork* o, const arks_response_batch* b, arks_response_result* r, uint32_t i, uint32_t out) {
  if (b->qos[i] < 0 || (uint32_t)b->qos[i] >= o->n_qos) { /* the stream's qos entry is not in these tables: nothing to bill */
    r->reason[out] = ARKS_R_QOS_GONE;
    r->counted[out] = 0;
    r->usage[3 * (size_t)out] = r->usage[3 * (size_t)out + 1] = r->usage[3 * (size_t)out + 2] = 0;
    return;
  }
  handle_response_inner(o, b, r, i, out);
  int64_t* row = o->metrics + (size_t)b->qos[i] * ARKS_METRIC_COLS;
  row[ARKS_METRIC_MESSAGES]++; /* RecordRequest(ns, user, model, dur, "200") for every response-body message */
  /* `!hasCompleted && complete && EndOfStream`: complete was set by THIS message (usage.total_tokens != 0) */
  if (r->counted[out] && (b->flags[i] & ARKS_RESP_END_OF_STREAM) && !(b->flags[i] & ARKS_RESP_COMPLETED)) {
    row[ARKS_METRIC_USAGE + 0] = (int64_t)((uint64_t)row[ARKS_METRIC_USAGE + 0] + (uint64_t)r->usage[3 * (size_t)out + 0]);
    row[ARKS_METRIC_USAGE + 1] = (int64_t)((uint64_t)row[ARKS_METRIC_USAGE + 1] + (uint64_t)r->usage[3 * (size_t)out + 1]);
    row[ARKS_METRIC_HIST_IN + token_bucket(r->usage[3 * (size_t)out + 0])]++;
    row[ARKS_METRIC_HIST_OUT + token_bucket(r->usage[3 * (size_t)out + 1])]++;
  }
}
static void handle_response_inner(ork* o, const arks_response_batch* b, arks_response_result* r, uint32_t i, uint32_t out) {
  const uint8_t* body = b->bodies + b->body_off[i];
  size_t len = b->body_len[i];
  int32_t q = b->qos[i];
  int64_t usage[3] = {0, 0, 0};
  r->reason[out] = ARKS_R_OK;
  r->counted[out] = 0;
  r->usage[3 * (size_t)out] = r->usage[3 * (size_t)out + 1] = r->usage[3 * (size_t)out + 2] = 0;
  if (b->flags[i] & ARKS_RESP_STREAM) {
    /* handle_response.go:113-133 — every chunk decoded in isolation */
    if (ork_sse_chunk(body, len, usage)) {
      r->reason[out] = ARKS_R_STREAMING;
      return;
    }
  } else {
    if (!(b->flags[i] & ARKS_RESP_END_OF_STREAM)) { /* :141-149 */
      r->reason[out] = ARKS_R_PENDING;
      return;
    }
    ork_sink model = {NULL, 0, 0, 0, 0};
    if (ork_json_response(body, len, &model, usage)) { /* :157-166 */
      r->reason[out] = ARKS_R_RESPONSE_UNMARSHAL;
      return;
    }
    if (model.len == 0) { /* :167-181 */
      r->reason[out] = ARKS_R_RESPONSE_UNKNOWN;
      return;
    }
  }
  r->usage[3 * (size_t)out] = usage[0];
  r->usage[3 * (size_t)out + 1] = usage[1];
  r->usage[3 * (size_t)out + 2] = usage[2];
  if (usage[2] != 0) { /* :186 */
    r->counted[out] = 1;
    /* doTokenRateLimit: INCRBY total per token-type entry              check.go:47-59 */
    for (uint32_t j = o->qos_rl_off[q]; j < o->qos_rl_off[q + 1]; j++) {
      int rule = o->rl_rule[j];
      if (!RULE_IS_REQUEST[rule]) /* N4: minus what the request phase charged for this stream, if the host says so */
        rate_incr(o, (uint32_t)q, rule, ork_window_start(b->now_unix, rule), (int64_t)((uint64_t)usage[2] - (b->precharged ? (uint64_t)b->precharged[i] : 0)));
    }
    /* doTokenQuotaLimit: QosToQuotaRequests(conf, countMap) -> IncrUsage   check.go:62-72 */
    int32_t qt = o->qos_quota[q];
    if (qt == ARKS_QUOTA_MISSING) {
      r->reason[out] = ARKS_R_QUOTA_CONFIG_RESP;
      return;
    }
    if (qt >= 0)
      for (uint32_t j = o->quota_item_off[qt]; j < o->quota_item_off[qt + 1]; j++) {
        int ty = o->qitem_type[j];
        size_t k = (size_t)qt * 3 + (size_t)ty;
        o->quota_use[k] = (int64_t)((uint64_t)o->quota_use[k] + (uint64_t)usage[ty]);
      }
  }
}

int ork_request_batch(ork* o, const arks_request_batch* b, arks_request_result* r) {
  int rc = check_time(o, b->now_unix);
  if (rc) return rc;
  for (uint32_t i = 0; i < b->n; i++) handle_request(o, b, r, i, i);
  for (uint32_t k = 0; k < o->pc_n; k++) rate_incr(o, o->pc[k].q, o->pc[k].rule, ork_window_start(b->now_unix, o->pc[k].rule), o->pc[k].amount);
  o->pc_n = 0;
  o->est = NULL; /* estimates belong to one batch */
  o->est_n = 0;
  return 0;
}
void ork_set_precharge(ork* o, int on) { o->precharge = on != 0; }
void ork_set_estimates(ork* o, const uint32_t* est, uint32_t n) { o->est = est; o->est_n = n; }
int ork_response_batch(ork* o, const arks_response_batch* b, arks_response_result* r) {
  int rc = check_time(o, b->now_unix);
  if (rc) return rc;
  for (uint32_t i = 0; i < b->n; i++) handle_response(o, b, r, i, i);
  return 0;
}

/* ---------- tenant-sharded threads (cpu baseline; SURVEY.md §8d) ----------
 * All state of a request lives inside its namespace, so worker t owns the namespaces that hash to t and handles their
 * rows in arrival order: the decisions equal the serial ones. Three passes per batch, a barrier between them:
 *   1. (rows split evenly) owner of every row;   2. every worker handles ITS rows, writing results to a private, densely
 *   packed buffer (neighbouring rows belong to different workers: writing the shared result arrays directly makes every
 *   cache line bounce between all of them);   3. (rows split evenly) results copied to their rows. */
typedef struct {
  uint8_t *reason, *detail, *flags, *counted;
  int32_t *qos, *token, *pick;
  int64_t *cur, *lim, *usage;
  uint32_t *moff, *mlen;
  uint32_t n;
} mt_priv;
typedef struct {
  ork* o;
  const arks_request_batch* rb;
  arks_request_result* rr;
  const arks_response_batch* pb;
  arks_response_result* pr;
  int tid, nt;
  uint16_t* shard;   /* per row: owning worker */
  uint32_t* slot;    /* per row: position inside its owner's private buffer */
  mt_priv* priv;     /* nt private buffers */
  pthread_barrier_t* bar;
} mt_arg;
static uint32_t ns_shard(const ork* o, uint32_t tok, int nt) {
  size_t l;
  const uint8_t* s = S(o, o->tok_ns_str[tok], &l);
  return (uint32_t)(fnv64(s, l, 0x9e3779b97f4a7c15ull) % (uint64_t)nt);
}
static void priv_alloc(mt_priv* p, uint32_t n, int req) {
  memset(p, 0, sizeof *p);
  p->n = n;
  size_t m = n ? n : 1;
  p->reason = (uint8_t*)malloc(m);
  if (req) {
    p->detail = (uint8_t*)malloc(m); p->flags = (uint8_t*)malloc(m);
    p->qos = (int32_t*)malloc(4 * m); p->token = (int32_t*)malloc(4 * m); p->pick = (int32_t*)malloc(4 * m);
    p->cur = (int64_t*)malloc(8 * m); p->lim = (int64_t*)malloc(8 * m);
    p->moff = (uint32_t*)malloc(4 * m); p->mlen = (uint32_t*)malloc(4 * m);
  } else {
    p->counted = (uint8_t*)malloc(m);
    p->usage = (int64_t*)malloc(24 * m);
  }
}
static void priv_free(mt_priv* p) {
  free(p->reason); free(p->detail); free(p->flags); free(p->counted);
  free(p->qos); free(p->token); free(p->pick); free(p->cur); free(p->lim); free(p->usage); free(p->moff); free(p->mlen);
}
static void* mt_req(void* p) {
  mt_arg* a = (mt_arg*)p;
  const uint32_t n = a->rb->n;
  const uint32_t lo = (uint32_t)((uint64_t)n * a->tid / a->nt), hi = (uint32_t)((uint64_t)n * (a->tid + 1) / a->nt);
  for (uint32_t i = lo; i < hi; i++) {
    int32_t t = find_token(a->o, a->rb->tokens + a->rb->token_off[i], a->rb->token_off[i + 1] - a->rb->token_off[i]);
    a->shard[i] = (uint16_t)(t >= 0 ? ns_shard(a->o, (uint32_t)t, a->nt) : i % (uint32_t)a->nt);
  }
  pthread_barrier_wait(a->bar);
  uint32_t mine = 0;
  for (uint32_t i = 0; i < n; i++) mine += a->shard[i] == a->tid;
  mt_priv* me = &a->priv[a->tid];
  priv_alloc(me, mine, 1);
  arks_request_result pr = {me->reason, me->detail, me->flags, me->qos, me->token, me->pick, me->cur, me->lim, me->moff, me->mlen, NULL};
  uint32_t k = 0;
  for (uint32_t i = 0; i < n; i++)
    if (a->shard[i] == a->tid) {
      a->slot[i] = k;
      handle_request(a->o, a->rb, &pr, i, k++);
    }
  pthread_barrier_wait(a->bar);
  arks_request_result* r = a->rr;
  for (uint32_t i = lo; i < hi; i++) {
    const mt_priv* w = &a->priv[a->shard[i]];
    const uint32_t j = a->slot[i];
    r->reason[i] = w->reason[j]; r->detail[i] = w->detail[j]; r->flags[i] = w->flags[j];
    r->qos[i] = w->qos[j]; r->token[i] = w->token[j]; r->pick[i] = w->pick[j];
    r->cur_usage[i] = w->cur[j]; r->limit_max[i] = w->lim[j];
    if (r->model_off) r->model_off[i] = w->moff[j];
    if (r->model_len) r->model_len[i] = w->mlen[j];
    if (r->bpe_count) r->bpe_count[i] = 0;
  }
  return NULL;
}
static void* mt_resp(void* p) {
  mt_arg* a = (mt_arg*)p;
  const uint32_t n = a->pb->n;
  const uint32_t lo = (uint32_t)((uint64_t)n * a->tid / a->nt), hi = (uint32_t)((uint64_t)n * (a->tid + 1) / a->nt);
  for (uint32_t i = lo; i < hi; i++) a->shard[i] = (uint16_t)ns_shard(a->o, a->o->qos_token[a->pb->qos[i]], a->nt);
  pthread_barrier_wait(a->bar);
  uint32_t mine = 0;
  for (uint32_t i = 0; i < n; i++) mine += a->shard[i] == a->tid;
  mt_priv* me = &a->priv[a->tid];
  priv_alloc(me, mine, 0);
  arks_response_result pr = {me->reason, me->counted, me->usage, NULL};
  uint32_t k = 0;
  for (uint32_t i = 0; i < n; i++)
    if (a->shard[i] == a->tid) {
      a->slot[i] = k;
      handle_response(a->o, a->pb, &pr, i, k++);
    }
  pthread_barrier_wait(a->bar);
  arks_response_result* r = a->pr;
  for (uint32_t i = lo; i < hi; i++) {
    const mt_priv* w = &a->priv[a->shard[i]];
    const size_t j = a->slot[i];
    r->reason[i] = w->reason[j]; r->counted[i] = w->counted[j];
    r->usage[3 * (size_t)i] = w->usage[3 * j]; r->usage[3 * (size_t)i + 1] = w->usage[3 * j + 1]; r->usage[3 * (size_t)i + 2] = w->usage[3 * j + 2];
  }
  return NULL;
}
/* Workers are created once (first threaded call, or when the thread count changes) and parked on a barrier between
 * batches: creating and joining 128 threads per batch costs more than the batch itself. */
typedef struct {
  pthread_t th[256];
  mt_arg args[256];
  mt_priv priv[256];
  pthread_barrier_t start, done, mid; /* start / done: nt workers + the caller; mid: the workers' own barrier */
  void* (*fn)(void*);
  int nt, quit;
} mt_pool;
static mt_pool* g_pool; /* one pool per process: the baseline runs one oracle at a time */
static void* pool_worker(void* p) {
  mt_arg* a = (mt_arg*)p;
  for (;;) {
    pthread_barrier_wait(&g_pool->start);
    if (g_pool->quit) return NULL;
    g_pool->fn(a);
    pthread_barrier_wait(&g_pool->done);
  }
}
static void pool_stop(void) {
  if (!g_pool) return;
  g_pool->quit = 1;
  pthread_barrier_wait(&g_pool->start);
  for (int t = 0; t < g_pool->nt; t++) pthread_join(g_pool->th[t], NULL);
  pthread_barrier_destroy(&g_pool->start);
  pthread_barrier_destroy(&g_pool->done);
  pthread_barrier_destroy(&g_pool->mid);
  free(g_pool);
  g_pool = NULL;
}
static int run_mt(void* (*fn)(void*), mt_arg* base, int nt, uint32_t n) {
  if (nt < 1) nt = 1;
  if (nt > 256) nt = 256;
  if (g_pool && g_pool->nt != nt) pool_stop();
  if (!g_pool) {
    g_pool = (mt_pool*)calloc(1, sizeof *g_pool);
    g_pool->nt = nt;
    pthread_barrier_init(&g_pool->start, NULL, (unsigned)nt + 1);
    pthread_barrier_init(&g_pool->done, NULL, (unsigned)nt + 1);
    pthread_barrier_init(&g_pool->mid, NULL, (unsigned)nt);
    for (int t = 0; t < nt; t++) pthread_create(&g_pool->th[t], NULL, pool_worker, &g_pool->args[t]);
  }
  uint16_t* shard = (uint16_t*)malloc((size_t)n * 2 + 2);
  uint32_t* slot = (uint32_t*)malloc((size_t)n * 4 + 4);
  memset(g_pool->priv, 0, sizeof g_pool->priv);
  for (int t = 0; t < nt; t++) {
    g_pool->args[t] = *base;
    g_pool->args[t].tid = t;
    g_pool->args[t].nt = nt;
    g_pool->args[t].shard = shard;
    g_pool->args[t].slot = slot;
    g_pool->args[t].priv = g_pool->priv;
    g_pool->args[t].bar = &g_pool->mid;
  }
  g_pool->fn = fn;
  pthread_barrier_wait(&g_pool->start);
  pthread_barrier_wait(&g_pool->done);
  for (int t = 0; t < nt; t++) priv_free(&g_pool->priv[t]);
  free(shard);
  free(slot);
  return 0;
}
int ork_request_batch_mt(ork* o, const arks_request_batch* b, arks_request_result* r, int nt) {
  int rc = check_time(o, b->now_unix);
  if (rc) return rc;
  mt_arg a = {o, b, r, NULL, NULL, 0, nt, NULL, NULL, NULL, NULL};
  return run_mt(mt_req, &a, nt, b->n);
}
int ork_response_batch_mt(ork* o, const arks_response_batch* b, arks_response_result* r, int nt) {
  int rc = check_time(o, b->now_unix);
  if (rc) return rc;
  for (uint32_t i = 0; i < b->n; i++)
    if (b->qos[i] < 0 || (uint32_t)b->qos[i] >= o->n_qos) return ARKS_E_INVALID_ARG;
  mt_arg a = {o, NULL, NULL, b, r, 0, nt, NULL, NULL, NULL, NULL};
  return run_mt(mt_resp, &a, nt, b->n);
}

/* ---------- quota.QuotaService surface + snapshots ---------- */
int ork_snapshot_quota(ork* o, int64_t* usage) {
  memcpy(usage, o->quota_use, (size_t)o->n_quotas * 24);
  return 0;
}
int ork_set_quota_usage(ork* o, uint32_t quota, const int64_t usage[3]) {
  if (quota >= o->n_quotas) return ARKS_E_INVALID_ARG;
  memcpy(o->quota_use + 3 * (size_t)quota, usage, 24);
  return 0;
}
int ork_incr_quota_usage(ork* o, uint32_t quota, const int64_t delta[3]) {
  if (quota >= o->n_quotas) return ARKS_E_INVALID_ARG;
  for (int k = 0; k < 3; k++)
    o->quota_use[3 * (size_t)quota + k] = (int64_t)((uint64_t)o->quota_use[3 * (size_t)quota + k] + (uint64_t)delta[k]);
  return 0;
}
/* syncQuotaUsage for one ArksQuota (qosconfig/arks_impl.go:226-296). status_present: bit t set when
 * quota.Status.QuotaStatus has an entry of type t; status_used[t] its Used. Returns bit0 = shouldUpdateCR, bit1 =
 * shouldUpdateQuota. The CR side is updated in place; on shouldUpdateQuota the reference calls SetUsage with requests
 * built by QosToQuotaRequests(conf, nil), i.e. Request == 0 for every item: the usage of every spec'd type is ZEROED
 * (restore == 0). restore == 1 is the repaired behaviour: the store is raised to the CR's value instead. */
int ork_sync_quota_usage(ork* o, uint32_t q, uint32_t* status_present, int64_t status_used[3], int restore) {
  if (q >= o->n_quotas) return ARKS_E_INVALID_ARG;
  int update_cr = 0, update_quota = 0;
  for (uint32_t j = o->quota_item_off[q]; j < o->quota_item_off[q + 1]; j++) {
    int ty = o->qitem_type[j];
    int64_t cur = o->quota_use[(size_t)q * 3 + (size_t)ty];
    if (*status_present & (1u << ty)) {
      if (status_used[ty] < cur) { update_cr = 1; status_used[ty] = cur; }
      else if (status_used[ty] > cur) update_quota = 1;
    } else { /* add new status */
      update_cr = 1;
      *status_present |= 1u << ty;
      status_used[ty] = cur;
    }
  }
  if (update_quota)
    for (uint32_t j = o->quota_item_off[q]; j < o->quota_item_off[q + 1]; j++) {
      int ty = o->qitem_type[j];
      int64_t* u = &o->quota_use[(size_t)q * 3 + (size_t)ty];
      if (!restore) *u = 0;
      else if (status_used[ty] > *u) *u = status_used[ty];
    }
  return update_cr | update_quota << 1;
}
int ork_snapshot_metrics(ork* o, int64_t* rows) {
  memcpy(rows, o->metrics, (size_t)o->n_qos * ARKS_METRIC_COLS * 8);
  return 0;
}
int ork_snapshot_rate(ork* o, int64_t now, int64_t* c) {
  for (uint32_t q = 0; q < o->n_qos; q++)
    for (int r = 0; r < 4; r++) c[(size_t)q * 4 + r] = rate_get(o, q, r, ork_window_start(now, r));
  return 0;
}

/* ---------- unit-level wrappers ---------- */
int ork_parse_request_body(const uint8_t* body, size_t len, uint8_t* model_out, size_t model_cap, size_t* model_len,
                           int* stream, int* so_present, int* include_usage) {
  ork_sink m = {model_out, 0, model_cap, 0, 0};
  int rc = ork_json_request(body, len, &m, stream, so_present, include_usage, NULL);
  *model_len = m.len;
  return rc;
}
int ork_parse_response_body(const uint8_t* body, size_t len, size_t* model_len, int64_t usage[3]) {
  ork_sink m = {NULL, 0, 0, 0, 0};
  int rc = ork_json_response(body, len, &m, usage);
  *model_len = m.len;
  return rc;
}
int ork_parse_sse_chunk(const uint8_t* body, size_t len, int64_t usage[3]) { return ork_sse_chunk(body, len, usage); }
