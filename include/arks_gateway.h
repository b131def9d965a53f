/*
 * arks_gateway.h — C ABI of the H100-native arks-gateway-plugins hot path.
 *
 * One object (`arks_ctx`, one per GPU) replaces, together, the three plugin seams the reference
 * ext_proc server calls per request (all paths relative to the reference tree):
 *
 *   ratelimiter.RateLimterInterface   pkg/gateway/ratelimiter/rate_limiter.go:21-28
 *   quota.QuotaService                pkg/gateway/quota/types.go:24-28
 *   qosconfig.ConfigProvider          pkg/gateway/qosconfig/provider.go:29-37
 *
 * plus the per-byte work of the four phase handlers
 *
 *   HandleRequestBody                 pkg/gateway/handle_request.go:83-249
 *   HandleResponseBody                pkg/gateway/handle_response.go:80-268
 *
 * The Go host keeps the ext_proc gRPC server (pkg/gateway/gateway.go:77-138) and calls these entry
 * points through cgo from one OS-thread-locked batcher goroutine per GPU (see INTEGRATION.md).
 *
 * Conventions
 *   - plain pointers and sizes only; every buffer is caller-owned HOST memory unless the name ends
 *     in `_dev`; the library owns all device memory.
 *   - the clock is never read inside: every batch carries `now_unix` (seconds). Batches are applied
 *     in call order; within a batch, requests are applied in index order (the linearisation the
 *     oracle shares, DESIGN.md §3). `now_unix` must not move to an earlier rate-limit window.
 *   - return value: 0 ok, negative `arks_status`. Per-request outcomes only via the result arrays.
 *   - there is no CPU fallback: without a CUDA device `arks_create` fails with ARKS_E_NO_DEVICE.
 *   - threads: a context has ONE batch thread (submit / stage / run / select, arks_commit_tables, arks_update_endpoint_weights)
 *     and may have one config thread (arks_upsert_*, arks_delete_*, arks_config_prepare, arks_prepare_tables: they never
 *     touch the generation the batch thread reads; arks_find_*: they read the current generation's keys under the lock a
 *     commit holds while it swaps them). The snapshot / sync calls (arks_snapshot_*,
 *     arks_sync_quota_usage, arks_set / incr_quota_usage) are ordered on the compute stream and may come from a third thread,
 *     but not while arks_commit_tables runs (host/cpp's Batcher and arks_b200/provider.py arrange exactly that).
 */
#ifndef ARKS_GATEWAY_H
#define ARKS_GATEWAY_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ARKS_ABI_VERSION 2

/* ---- status codes (library-level errors; Go `error` in the reference) ---- */
enum arks_status {
  ARKS_S_OK = 0,
  ARKS_E_INVALID_ARG = -1,
  ARKS_E_NO_DEVICE = -2,
  ARKS_E_CUDA = -3,
  ARKS_E_TIME_WENT_BACK = -4, /* now_unix fell into an earlier window than a previous batch */
  ARKS_E_BAD_TABLE = -5,      /* unknown rate-limit rule / quota type (reference: 500 / panic,
                                 pkg/gateway/check.go:112-121, ratelimiter/types.go:46); or a snapshot whose
                                 offsets / string ids / weights are out of range (checked before anything follows them) */
  ARKS_E_CAPACITY = -6,
  ARKS_E_NOT_LOADED = -7,
};

/* ---- rate-limit rules: compiled in, pkg/gateway/ratelimiter/rate_limiter.go:31-68 ---- */
enum arks_rule {
  ARKS_RULE_RPM = 0, /* request, 1 minute */
  ARKS_RULE_RPD = 1, /* request, 1 day    */
  ARKS_RULE_TPM = 2, /* token,   1 minute */
  ARKS_RULE_TPD = 3, /* token,   1 day    */
  ARKS_N_RULES = 4,
};
/* quota item types: api/v1/arksquota_types.go:28-33 */
enum arks_quota_type {
  ARKS_QT_PROMPT = 0,
  ARKS_QT_RESPONSE = 1,
  ARKS_QT_TOTAL = 2,
  ARKS_N_QT = 3,
};
#define ARKS_QUOTA_NONE (-1)    /* qos.quota.name == ""           handle_request.go:185 */
#define ARKS_QUOTA_MISSING (-2) /* named ArksQuota does not exist check.go:76-84 -> 500 */

/* ---- per-request outcome: (http status, x-error-* header) of SURVEY §8a / pkg/gateway/types.go:24-56 ---- */
enum arks_reason {
  ARKS_R_OK = 0,
  ARKS_R_NO_TOKEN = 1,             /* 401 x-error-token                         handle_request.go:48-56   */
  ARKS_R_REQUEST_BODY = 2,         /* 400 x-error-request-body-processing       handle_request.go:97-104  */
  ARKS_R_NO_MODEL = 3,             /* 400 x-error-no-model-in-request           handle_request.go:108-115 */
  ARKS_R_TOKEN_NOT_FOUND = 4,      /* 500 x-error-token "token not found"       arks_impl.go:313-315      */
  ARKS_R_MODEL_NOT_IN_TOKEN = 5,   /* 500 x-error-token "model not found"       arks_impl.go:337          */
  ARKS_R_NO_MODEL_BACKENDS = 6,    /* 400 x-error-no-model-backends             handle_request.go:147-154 */
  ARKS_R_STREAM_OPTIONS = 7,       /* 400 x-error-no-stream-options-include-usage  :160-171               */
  ARKS_R_RATE_LIMIT = 8,           /* 429 x-error-rate-limit  (detail = index in qos.RateLimits) check.go:140-152 */
  ARKS_R_QUOTA = 9,                /* 429 x-error-quota       (detail = index in quota items)   check.go:95-104  */
  ARKS_R_QUOTA_CONFIG = 10,        /* 500 x-error-quota       (ArksQuota missing)               check.go:76-84   */
  ARKS_R_STREAMING = 11,           /* 500 x-error-streaming                     handle_response.go:125-133 */
  ARKS_R_RESPONSE_UNMARSHAL = 12,  /* 500 x-error-response-unmarshal            handle_response.go:157-166 */
  ARKS_R_RESPONSE_UNKNOWN = 13,    /* 500 x-error-response-unknown              handle_response.go:167-181 */
  ARKS_R_QUOTA_CONFIG_RESP = 14,   /* 500 x-error-quota at response time        handle_response.go:215-223 */
  ARKS_R_PENDING = 15,             /* non-stream chunk without end_of_stream: empty CommonResponse :141-149 */
  ARKS_R_QOS_GONE = 16,            /* response row whose qos entry is unknown to the current tables (never resolved, or
                                      its (namespace,user,model) key was removed by a config reload since the request):
                                      nothing is billed, the row is answered like ARKS_R_OK. The reference keeps the
                                      UserQos by value (gateway.go:78) and would still INCRBY the orphaned Redis keys. */
};

/* ---- config tables: a flat snapshot of the ArksToken / ArksQuota / ArksEndpoint informer cache ----
 * (qosconfig/arks_impl.go:303-397). Strings live in one pool; string i = str_bytes[str_off[i]..str_off[i+1]).
 * Equal strings need not share an id; the library resolves names by content. */
typedef struct arks_tables {
  const uint8_t* str_bytes;
  const uint32_t* str_off; /* n_str + 1 */
  uint32_t n_str;

  /* ArksToken objects, api/v1/arkstoken_types.go:55-61. If two objects carry the same spec.token the
   * first one in this array wins (reference: Items[0] of an unordered index, arks_impl.go:317). */
  uint32_t n_tokens;
  const uint32_t* tok_token_str; /* spec.token                         */
  const uint32_t* tok_ns_str;    /* metadata.namespace                 */
  const uint32_t* tok_name_str;  /* metadata.name == UserQos.User      */
  const uint32_t* tok_qos_off;   /* n_tokens + 1, CSR into qos entries */

  /* spec.qos[] entries, api/v1/arkstoken_types.go:46-52 */
  uint32_t n_qos;
  const uint32_t* qos_model_str; /* arksEndpoint.name                                  */
  const int32_t* qos_quota;      /* index into quotas, ARKS_QUOTA_NONE, ARKS_QUOTA_MISSING */
  const uint32_t* qos_rl_off;    /* n_qos + 1, CSR into rate limits                    */
  uint32_t n_rl;
  const uint8_t* rl_rule;   /* enum arks_rule, in spec order */
  const int64_t* rl_value;  /* limit                          */

  /* ArksQuota objects, api/v1/arksquota_types.go:36-53 */
  uint32_t n_quotas;
  const uint32_t* quota_ns_str;
  const uint32_t* quota_name_str;
  const uint32_t* quota_item_off; /* n_quotas + 1 */
  uint32_t n_qitems;
  const uint8_t* qitem_type;   /* enum arks_quota_type, in spec order */
  const int64_t* qitem_value;  /* limit                                */

  /* ArksEndpoint objects, api/v1/arksendpoint_types.go:28-48; backends in the order the controller
   * emits HTTPRoute backendRefs (internal/controller/arksendpoint_controller.go:283-347): static
   * routeConfigs first, then ready application Services at defaultWeight. */
  uint32_t n_endpoints;
  const uint32_t* ep_ns_str;
  const uint32_t* ep_name_str;    /* == model name */
  const uint32_t* ep_backend_off; /* n_endpoints + 1 */
  uint32_t n_backends;
  const int32_t* backend_weight;  /* >= 0 */
} arks_tables;

/* ---- request phase (ProcessingRequest_RequestBody, handle_request.go:83-249) ---- */
typedef struct arks_request_batch {
  uint32_t n;
  const uint8_t* bodies;      /* concatenated request bodies; each body starts 16-byte aligned  *
                               * (32-byte aligned bodies are read a whole sector at a time)      */
  const uint32_t* body_off;   /* n: byte offset of body i (multiple of 16)                      */
  const uint32_t* body_len;   /* n: exact length                                                */
  uint64_t bodies_bytes;      /* bytes of `bodies` uploaded: must cover body_off[i] + body_len[i] *
                               * of every body (or the batch is refused), at most max_batch_bytes *
                               * of arks_create (the library takes up to that + 16, rounded up   *
                               * to 256). The padding between bodies and whatever follows        *
                               * bodies_bytes may hold anything: the kernels read past a body's  *
                               * end and never let those bytes change a result. Same for         *
                               * arks_response_batch.                                            */
  const uint8_t* tokens;      /* concatenated bearer tokens (output of arks_extract_bearer)     */
  const uint32_t* token_off;  /* n + 1, non-decreasing (a batch that breaks this or the body     *
                               * bounds is refused as a whole: ARKS_E_INVALID_ARG, nothing staged) */
  const uint64_t* pick_rand;  /* n or NULL: per-request random for the weighted pick (A12)      */
  int64_t now_unix;
} arks_request_batch;

typedef struct arks_request_result {
  uint8_t* reason;      /* n: enum arks_reason; ARKS_R_OK == continue (BodyResponse + 3 headers)            */
  uint8_t* detail;      /* n: rule / quota-item index for 429s, else 0                                       */
  uint8_t* flags;       /* n: bit0 = stream, bit1 = ARKS_FLAG_METERED                                        */
  int32_t* qos;         /* n: qos-entry index carried into the response phase, -1 if not resolved            */
  int32_t* token;       /* n: ArksToken index (namespace / username headers), -1 if not found                */
  int32_t* pick;        /* n: backend index within the endpoint, -1 none / not admitted                      */
  int64_t* cur_usage;   /* n: RateLimitResponse.currentUsage / QuotaResult.currentUsage for 429s, else 0     */
  int64_t* limit_max;   /* n: limitMax for 429s, else 0                                                      */
  /* optional outputs (each may be NULL) */
  uint32_t* model_off;  /* n: byte offset, inside body i, of the raw `model` string (first byte after the opening quote) */
  uint32_t* model_len;  /* n: its raw length (escapes not decoded); bit 31 set iff the span contains a backslash. Both 0
                         *    when the body did not parse or its last `model` member is not a string. The host needs the
                         *    name for the x-error-* header values of handle_request.go:112,123,151 and slices its own copy
                         *    of the body                                                                               */
  uint32_t* bpe_count;  /* n: BPE tokens of the prompt text (see arks_load_bpe); 0 when no vocabulary is loaded. A side
                         *    output: the reference counts no tokens at request time (check.go:124-126), so this never
                         *    feeds admit/deny unless arks_set_precharge is switched on                              */
} arks_request_result;
#define ARKS_FLAG_METERED 2u /* admitted under arks_set_stream_metering: the host sets ARKS_RESP_METERED on every chunk */

/* ---- response phase (ProcessingRequest_ResponseBody with :status 200, handle_response.go:80-268) ---- */
#define ARKS_RESP_STREAM 1u        /* the request had stream:true  -> body is one SSE chunk, decoded in isolation */
#define ARKS_RESP_END_OF_STREAM 2u /* non-stream: `body` is the complete concatenated response body; stream: the last
                                    * chunk (only the metrics read it there)                                      */
#define ARKS_RESP_COMPLETED 4u     /* this stream already had a usage-bearing message (`completed`, gateway.go:127):
                                    * read by the metrics only                                                     */
#define ARKS_RESP_METERED 8u       /* with ARKS_RESP_STREAM: a chunk of a stream whose request result had ARKS_FLAG_METERED.
                                    * Billed by its BPE count (arks_set_stream_metering); ignored on non-stream rows */
typedef struct arks_response_batch {
  uint32_t n;
  const uint8_t* bodies;
  const uint32_t* body_off; /* n, multiples of 16 */
  const uint32_t* body_len; /* n */
  uint64_t bodies_bytes;
  const int32_t* qos;    /* n: from arks_request_result.qos */
  const uint8_t* flags;  /* n: ARKS_RESP_* */
  int64_t now_unix;
  const uint32_t* gen;   /* n or NULL: arks_table_generation() at the time each row's request was decided. A qos index is
                          * positional in the tables of ITS generation; rows of an older generation are re-mapped by their
                          * (namespace,user,model) key (the last ARKS_GEN_HISTORY generations are kept) or answered
                          * ARKS_R_QOS_GONE. NULL: every row belongs to the current generation. */
  const uint32_t* precharged; /* n or NULL: what arks_set_precharge charged the token-type rules for this stream at request time
                               * (arks_request_result.bpe_count of its request): the token-type rules are then charged
                               * total_tokens - precharged, the difference between the upstream's count and the estimate */
} arks_response_batch;
#define ARKS_GEN_HISTORY 16

typedef struct arks_response_result {
  uint8_t* reason;   /* n: ARKS_R_OK / STREAMING / RESPONSE_UNMARSHAL / RESPONSE_UNKNOWN / QUOTA_CONFIG_RESP / PENDING */
  uint8_t* counted;  /* n: 1 iff usage.total_tokens != 0 (counters were incremented, `complete = true`)               */
  int64_t* usage;    /* 3n: prompt_tokens, completion_tokens, total_tokens                                           */
  uint32_t* bpe_count; /* n or NULL: BPE tokens of the completion text in this body / SSE chunk (see arks_load_bpe)      */
} arks_response_result;

typedef struct arks_ctx arks_ctx;

/* lifecycle */
int arks_abi_version(void);
int arks_create(int device, uint32_t max_batch, uint64_t max_batch_bytes, arks_ctx** out);
void arks_destroy(arks_ctx* ctx);
const char* arks_last_error(const arks_ctx* ctx);

/* config plane: replaces the informer cache behind qosconfig.ConfigProvider (arks_impl.go:104-189).
 * A load between batches swaps the whole snapshot; counters are carried over by key
 * ((namespace,user,model) and (namespace,quotaName)), like Redis keys survive a CRD edit. */
int arks_load_tables(arks_ctx* ctx, const arks_tables* t);
/* bumped by every table swap that succeeds: the generation the qos / token indices of request results refer to */
uint32_t arks_table_generation(const arks_ctx* ctx);

/* ---- the same swap without stalling the data path ---------------------------------------------------------------------
 * arks_load_tables = prepare + commit + a wait, for cold start. A running gateway splits it:
 *   arks_prepare_tables  (CONFIG thread, any time)  validates, builds the device image of the next generation in fresh
 *                        allocations and uploads it on the library's config stream. Batches keep running; nothing they use
 *                        is touched. Errors leave the context exactly as it was.
 *   arks_commit_tables   (the thread that submits batches, between two submissions)  queues, on the compute stream, the
 *                        kernels that carry every counter into the new arrays BY KEY on the device, swaps the pointers and
 *                        retires the old image stream-ordered. No host wait, no copy through the host: the batch queued
 *                        before runs on the old generation, the one queued after on the new. Fails (ARKS_E_INVALID_ARG) if
 *                        another generation was committed since the prepare; discard and prepare again.
 * This is the informer's OnAdd/OnUpdate/OnDelete (arks_impl.go:104-189) arriving while requests are in flight. */
typedef struct arks_prepared arks_prepared;
int arks_prepare_tables(arks_ctx* ctx, const arks_tables* t, arks_prepared** out);
int arks_commit_tables(arks_ctx* ctx, arks_prepared* p);   /* consumes p on success */
void arks_discard_prepared(arks_ctx* ctx, arks_prepared* p);

/* ---- object-level config plane: one call per informer event ------------------------------------------------------------
 * The library keeps the objects (keyed by namespace/name, like the informer cache); each call is O(that object).
 * arks_config_prepare flattens the store into the next generation (arks_prepare_tables underneath; same commit).
 * Where several ArksToken objects carry the same spec.token the first in (namespace, name) order wins (the reference
 * takes Items[0] of an unordered index, arks_impl.go:317). Strings are (pointer, length), not NUL-terminated. */
typedef struct arks_qos_spec {            /* one spec.qos[] entry, api/v1/arkstoken_types.go:46-52 */
  const char* model;     uint32_t model_len;  /* arksEndpoint.name                                */
  const char* quota;     uint32_t quota_len;  /* quota.name; length 0 = no quota                  */
  uint32_t n_rl;                              /* rateLimits, in spec order                        */
  const uint8_t* rl_rule;                     /* enum arks_rule                                   */
  const int64_t* rl_value;
} arks_qos_spec;
int arks_upsert_token(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const char* token,
                      uint32_t token_len, const arks_qos_spec* qos, uint32_t n_qos);
int arks_delete_token(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len);
int arks_upsert_quota(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const uint8_t* item_type,
                      const int64_t* item_value, uint32_t n_items);
int arks_delete_quota(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len);
int arks_upsert_endpoint(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len,
                         const int32_t* backend_weight, uint32_t n_backends);
int arks_delete_endpoint(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len);
/* delete of an object that is not there: ARKS_E_INVALID_ARG. Nothing reaches the device before: */
int arks_config_prepare(arks_ctx* ctx, arks_prepared** out);
/* index lookups in the CURRENT generation (results carry indices): -1 when absent */
int32_t arks_find_quota(const arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len);
int32_t arks_find_qos(const arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* user, uint32_t user_len, const char* model,
                      uint32_t model_len);
/* ---- BPE token counting (north star). The reference has NO tokenizer: it reads `usage` from the upstream's response
 * (pkg/gateway/handle_response.go:90-93,117-123) and counts 0 tokens at request time (check.go:124-126). The count is
 * therefore a side output with its own oracle (HF `tokenizers`); decisions never depend on it.
 * What is counted: every JSON string that is the value of a key named "content" in the body (escapes decoded), cut by the
 * Qwen2 pre-tokenizer pattern and byte-level BPE-merged with the merge list below.  ARKS_BPE_UNCOUNTED is reported instead
 * of a wrong number when a body is outside what the device handles (invalid UTF-8 / escapes, a lone surrogate, a
 * pre-token longer than 128 bytes, NFC-unsafe text under ARKS_BPE_NFC, work-list overflow). */
#define ARKS_BPE_UNCOUNTED 0xFFFFFFFFu
#define ARKS_BPE_NFC 1u  /* flags: the tokenizer normalises to NFC (Qwen2 does): text NFC could change is not counted */
#define ARKS_BPE_DIGITS3 2u        /* flags: the pre-tokenizer splits numbers as \p{N}{1,3} (Llama 3) instead of \p{N} (Qwen2)  */
#define ARKS_BPE_IGNORE_MERGES 4u  /* flags: a pre-token that is itself a vocabulary entry is one token, whatever the merges say
                                    * (the BPE model's "ignore_merges": true, Llama 3); needs the token strings of
                                    * arks_load_bpe_vocab                                                                  */
#define ARKS_BPE_MAX_VOCABS 8      /* vocabulary slots per context                                                          */
typedef struct arks_bpe_tables {
  const uint32_t* byte_id;  /* 256: token id of every single byte (byte-level alphabet)                           */
  uint32_t n_merges;
  const uint32_t* left;     /* n_merges: merge i joins token left[i] and right[i] into merged[i]; rank = i        */
  const uint32_t* right;
  const uint32_t* merged;
  const uint8_t* cp_class;  /* 0x110000 / 2 bytes, a nibble per Unicode code point (low nibble = even code point):
                             * bits 0-1 class (0 other, 1 \p{L}, 2 \p{N}, 3 \s), bit 2 NFC-unsafe; tools/gen_bpe_unicode.py */
  uint32_t flags;
} arks_bpe_tables;
/* copies the tables to the device and switches the bpe_count columns on (NULL: off). This is vocabulary slot 0, the default
 * every model is counted with unless it is bound to another slot. Refuses ARKS_BPE_IGNORE_MERGES (no token strings here) and
 * NULL while another slot is loaded or stream metering is on. */
int arks_load_bpe(arks_ctx* ctx, const arks_bpe_tables* t);
/* Per-model vocabularies. A gateway fronts many models, and each should be counted with its own tokenizer (the count feeds
 * the pre-charge and stream metering). A context holds up to ARKS_BPE_MAX_VOCABS vocabularies; slot 0 is arks_load_bpe's.
 * arks_load_bpe_vocab loads `t` into `slot` (slot 0: as arks_load_bpe, but ARKS_BPE_IGNORE_MERGES is allowed). With
 * ARKS_BPE_IGNORE_MERGES, tok_bytes / tok_off are the vocabulary's token strings as bytes (token k is
 * tok_bytes[tok_off[k], tok_off[k + 1]), n_tok + 1 offsets; only strings of 2..128 bytes matter); otherwise they may be NULL.
 * All slots share slot 0's Unicode class table: t->cp_class may be NULL for a slot other than 0. A slot other than 0 needs
 * slot 0 loaded (ARKS_E_NOT_LOADED). t == NULL empties the slot; refused while a model is bound to it, in the bindings or in
 * the current generation. A load that is refused or fails leaves the slot as it was. Same thread as arks_load_bpe (it waits
 * for the compute stream). */
int arks_load_bpe_vocab(arks_ctx* ctx, uint32_t slot, const arks_bpe_tables* t, const uint8_t* tok_bytes, const uint32_t* tok_off,
                        uint32_t n_tok);
/* Config thread: count requests and responses of qos entries whose model (the ArksEndpoint name) is `model` with the
 * vocabulary in `slot`; slot 0 removes the binding. ARKS_E_NOT_LOADED when the slot holds no vocabulary. Bindings are read by
 * arks_prepare_tables / arks_load_tables / arks_config_prepare and take effect with the NEXT generation; rows without a qos
 * entry are counted with slot 0. A response row is counted with the binding of the CURRENT generation, the one its qos index
 * is carried into at staging: a stream whose request was decided under an older generation is counted with today's
 * vocabulary of its model, and a row whose entry is gone (ARKS_R_QOS_GONE) with slot 0. */
int arks_bind_model_vocab(arks_ctx* ctx, const char* model, uint32_t model_len, uint32_t slot);
/* N4 (SURVEY.md section 8f), OPT-IN because it changes admit / deny against the reference, which counts no tokens at request
 * time ("token is not caculated in request", pkg/gateway/check.go:124-126: a tenant over its TPM is only stopped once the
 * upstream has answered). With precharge on and a vocabulary loaded, every ADMITTED request adds its prompt's BPE count to
 * the tpm / tpd counters of its qos entry when its micro-batch commits (checks inside a micro-batch see the counters as of
 * the batch's start, as they do for token-type rules today), and the response phase reconciles: it adds total_tokens minus
 * arks_response_batch.precharged. A stream whose response never arrives keeps its estimate charged. Quotas are untouched
 * (they bill what the upstream reports). Off by default: decisions are the reference's. */
int arks_set_precharge(arks_ctx* ctx, int on);
/* N5, OPT-IN stream metering. The reference refuses every stream:true request without stream_options.include_usage:true
 * (ARKS_R_STREAM_OPTIONS, handle_request.go:156-171) because it cannot bill such a stream. With metering on such a request
 * is decided like any other (rate limits, then quota); if admitted its result row has ARKS_FLAG_METERED and the host must
 * set ARKS_RESP_METERED on every response chunk of that stream. Billing of a metered stream:
 *   - its prompt's BPE count when its micro-batch commits: count x (tpm entries) and x (tpd entries) on the rate counters,
 *     quota items prompt and total, gateway_token_usage{input};
 *   - every chunk answered ARKS_R_OK: its completion count on tpm / tpd, quota items response and total,
 *     gateway_token_usage{output}. An upstream `usage` in the chunk is still reported but NOT billed (counted = 0);
 *   - a count that is not available (ARKS_BPE_UNCOUNTED, no vocabulary) is replaced by the body's byte length, an upper
 *     bound of its byte-level BPE count;
 *   - the pre-charge (arks_set_precharge) skips metered rows and their `precharged` is ignored: billed exactly once.
 * Metered rows count every JSON string that is the value of a key named content, text, reasoning_content or arguments
 * (bpe_count reports that wider count for every stream:true request without include_usage while metering is on, admitted
 * or not, and for ARKS_RESP_METERED chunks; other rows keep the content-only count). Known under-counts: tool
 * definitions, chat-template tokens. Needs a vocabulary: ARKS_E_NOT_LOADED without one, and arks_load_bpe(NULL) is refused
 * while metering is on. Off by default: decisions are the reference's. */
int arks_set_stream_metering(arks_ctx* ctx, int on);

/* routing churn (BASELINE config 5): replace the weights of one endpoint's backends in place */
int arks_update_endpoint_weights(arks_ctx* ctx, uint32_t endpoint, uint32_t n, const int32_t* weights);

/* A2: HandleRequestHeaders bearer extraction (handle_request.go:38-46). Pure host function.
 * keys/values: n_headers (ptr,len) pairs. Returns token length (>0) and sets *token to point into
 * the value, 0 when no usable token (-> 401 ARKS_R_NO_TOKEN). */
size_t arks_extract_bearer(const uint8_t* const* keys, const size_t* key_lens,
                           const uint8_t* const* values, const size_t* value_lens, size_t n_headers,
                           const uint8_t** token);

/* request phase: H2D + scan_request + limit_admit (+ pick) + D2H */
int arks_submit_request_batch(arks_ctx* ctx, const arks_request_batch* b, arks_request_result* r);
/* response phase: H2D + scan_response + apply_usage + D2H */
int arks_submit_response_batch(arks_ctx* ctx, const arks_response_batch* b, arks_response_result* r);

/* split form of the two calls above (bench: kernel-only timing with inputs resident in HBM) */
int arks_stage_request_batch(arks_ctx* ctx, const arks_request_batch* b);  /* H2D only          */
int arks_run_request_batch(arks_ctx* ctx, int64_t now_unix);               /* kernels only      */
int arks_fetch_request_result(arks_ctx* ctx, arks_request_result* r);      /* D2H + stream sync */
int arks_stage_response_batch(arks_ctx* ctx, const arks_response_batch* b);
int arks_run_response_batch(arks_ctx* ctx, int64_t now_unix);
int arks_fetch_response_result(arks_ctx* ctx, arks_response_result* r);
/* asynchronous submits: H2D, kernels and D2H are queued on the library's stream and the call returns at once; results
 * land in `out` when arks_wait_* returns. One batch may be in flight per slot (select the slot first), which lets the
 * host overlap packing batch k+1 with the PCIe traffic and kernels of batch k. Batches still apply in call order.
 * Threads: all submit / stage / run / select calls of a context come from one thread at a time; arks_wait_* may run on
 * another thread for a slot whose submit call has returned (host/cpp's completion thread does exactly that). */
int arks_submit_request_async(arks_ctx* ctx, const arks_request_batch* b);
int arks_wait_request(arks_ctx* ctx, int slot, arks_request_result* out);
int arks_submit_response_async(arks_ctx* ctx, const arks_response_batch* b);
int arks_wait_response(arks_ctx* ctx, int slot, arks_response_result* out);
/* up to 4 staging slots so that several batches can be resident in HBM at once (bench: rotate batches so the
 * timed inputs exceed L2). stage_/run_ calls act on the selected slot (default 0); fetch_ returns the last run. */
int arks_select_slot(arks_ctx* ctx, int slot);
/* per-kernel device timing of the last run_* call: CUDA events around every launch on the library's stream.
 * arks_last_kernel_ms returns the number of intervals and fills ms[]: after a request batch {scan stage, rank_hot +
 * limit_admit, the fast-path kernel of the two-stage scan alone (0: fused kernel), the BPE kernels (0: no vocabulary)},
 * after a response batch {scan stage, fast-path kernel alone, BPE kernels}. */
int arks_set_profiling(arks_ctx* ctx, int on);
int arks_last_kernel_ms(arks_ctx* ctx, float* ms, int cap);
/* CUDA stream handle (cudaStream_t) the kernels are launched on, for event timing by the caller */
void* arks_stream(arks_ctx* ctx);
/* Large batches are scanned in two stages: a warp per document for everything plain (arks_b200/csrc/mask_scan.cuh), the
 * exact engine for the rows that path declines. Rows of the last run_* call left to the exact engine, or -1 if that call
 * used the fused kernels (small or mixed batches). Synchronises the stream: for tests and the bench. */
int64_t arks_last_declined(arks_ctx* ctx);
/* number of kernel launches issued by this context so far */
uint64_t arks_launch_count(const arks_ctx* ctx);
/* how the last arks_stage_* call (also inside the submit calls) placed its bodies in device memory: 0 in the metadata
 * upload (bodies_bytes <= 16 KiB), 1 behind the metadata on the compute stream (<= 256 KiB and, for requests, room left
 * behind the metadata and bearer tokens), 2 in the slot's own bodies buffer, uploaded on the copy stream; -1 when that
 * call staged no bodies (an empty or a refused batch). A diagnostic for tests: results never depend on the route. */
int arks_last_staging_route(const arks_ctx* ctx);

/* N3 (SURVEY.md §8f): the gateway's Prometheus series that are functions of the request stream
 * (pkg/gateway/metrics/metrics.go:24-98, collector.go:35-53), accumulated on the device next to the counters and read at
 * scrape time. One row of ARKS_METRIC_COLS int64 per qos entry == label set (namespace, user, model); durations stay on
 * the host (wall clock). Off by default; counters survive arks_load_tables by key like the rate windows.
 *   [0..3]   gateway_rate_limit_hits_total{rule_type=rpm,rpd,tpm,tpd}     check.go:145
 *   [4..5]   gateway_token_usage{type=input,output}                        handle_response.go:102-104
 *   [6..23]  gateway_token_distribution{type=input} buckets le=1,2,4..65536,+Inf (non-cumulative counts)
 *   [24..41] gateway_token_distribution{type=output}
 *   [42]     gateway_requests_total{status="200"}: one per response-body message (gateway.go:129)               */
#define ARKS_METRIC_COLS 44
#define ARKS_METRIC_HITS 0
#define ARKS_METRIC_USAGE 4
#define ARKS_METRIC_HIST_IN 6
#define ARKS_METRIC_HIST_OUT 24
#define ARKS_METRIC_HIST_BUCKETS 18
#define ARKS_METRIC_MESSAGES 42
int arks_enable_metrics(arks_ctx* ctx, int on);
int arks_snapshot_metrics(arks_ctx* ctx, int64_t* rows /* n_qos * ARKS_METRIC_COLS */);

/* page-locked host memory for batch staging (bodies / SoA arrays handed to arks_submit_*): makes the uploads real DMA
 * without making the caller link the CUDA runtime. NULL when the allocation fails. */
void* arks_alloc_pinned(size_t bytes);
void arks_free_pinned(void* p);

/* quota.QuotaService surface (quota/redis_impl.go:38-107) and A14 snapshot/restore (arks_impl.go:217-300) */
int arks_snapshot_quota(arks_ctx* ctx, int64_t* usage /* 3 * n_quotas: prompt,response,total */);
int arks_set_quota_usage(arks_ctx* ctx, uint32_t quota, const int64_t usage[3]); /* SetUsage */
/* syncQuotaUsage (arks_impl.go:217-300), all ArksQuotas in one pass, between batches. In/out per quota: status_present
 * (bit t: Status.QuotaStatus has type t) and status_used[3]; out: action[q] bit0 = update the CR status, bit1 = the store
 * was outdated. mode ARKS_SYNC_REFERENCE reproduces the reference (an outdated store is zeroed, because SetUsage is
 * called with Request == 0), ARKS_SYNC_RESTORE raises the store to the CR's value (the intended restore on start). */
#define ARKS_SYNC_REFERENCE 0
#define ARKS_SYNC_RESTORE 1
int arks_sync_quota_usage(arks_ctx* ctx, int mode, uint32_t* status_present /* n_quotas */, int64_t* status_used /* 3 * n_quotas */,
                          uint8_t* action /* n_quotas */);
int arks_incr_quota_usage(arks_ctx* ctx, uint32_t quota, const int64_t delta[3]); /* IncrUsage */
/* rate counters of the CURRENT windows (value 0 if the stored window is older than now_unix's) */
int arks_snapshot_rate(arks_ctx* ctx, int64_t now_unix, int64_t* counters /* 4 * n_qos */);

/* multi-GPU: ArksQuotas shared across GPUs (SURVEY §8e). Off by default (tenant-sharded, single-owner keys, exact).
 * When enabled (before arks_load_tables) every response-phase quota increment is also accumulated in a per-GPU delta
 * vector (3*n_quotas int64). A fold epoch: all-reduce(sum) the delta vectors (the caller's NCCL / torch.distributed
 * call), then on every GPU quota += reduced - own_delta and own_delta = 0. Host-buffer form: take (returns and zeroes
 * the delta) + apply (adds the sum of the OTHER GPUs' deltas). Device form: export (D2D copy of the delta into the
 * caller's buffer, e.g. a torch tensor handed to ncclAllReduce) + fold (reads the reduced vector from device memory).
 * The delta vector survives arks_load_tables by (namespace, quotaName) like the usage itself. */
int arks_enable_quota_sharing(arks_ctx* ctx, int on);
int arks_take_quota_delta(arks_ctx* ctx, int64_t* delta_out);
int arks_apply_quota_delta(arks_ctx* ctx, const int64_t* remote_delta);
void* arks_quota_delta_dev(arks_ctx* ctx);
int arks_export_quota_delta_dev(arks_ctx* ctx, void* dst_dev);
/* quota += reduced - own; delta -= own, where `own` is what arks_export_quota_delta_dev handed out (own_dev, or the
 * library's copy of the last export when own_dev is NULL): increments that arrived between export and fold stay in the
 * delta vector for the next epoch. */
int arks_fold_quota_delta_dev(arks_ctx* ctx, const void* reduced_dev, const void* own_dev);

/* ---- the fold done BY the library over NCCL (NVLink / NVSwitch), so a Go / C++ host needs no torch -------------------
 * One communicator per context (one context per GPU, one process per GPU or several GPUs in one process). libnccl.so.2
 * is dlopen()ed at arks_comm_init (ARKS_NCCL_LIB overrides the name); the library does not link against it.
 *   arks_comm_unique_id   rank 0: 128 opaque bytes (ncclGetUniqueId) to hand to every rank over any channel
 *   arks_comm_init        every rank: ncclCommInitRank. `shared` lists, in the SAME canonical order on every rank, the LOCAL
 *                         indices of the quotas that live on every GPU (local numbering may differ per rank); NULL / 0 =
 *                         every quota, identical numbering everywhere. Call arks_comm_set_shared again after every table
 *                         swap: the indices belong to the generation they were given for, and a fold against another
 *                         generation is refused (ARKS_E_INVALID_ARG) instead of touching rows that moved.
 *   arks_fold_quota_allreduce   one fold epoch, stream-ordered: snapshot this GPU's unfolded increments, gather the shared
 *                         rows, ncclAllReduce(sum, int64) in place, quota += reduced - own on the shared rows, delta -= the
 *                         snapshot. wait != 0 also waits for it (the epoch's duration is then the call's).
 * Replaces the Redis INCRBY every gateway replica does against the one shared store (quota/redis.go:74-100). */
#define ARKS_UNIQUE_ID_BYTES 128
int arks_comm_unique_id(arks_ctx* ctx, void* out /* ARKS_UNIQUE_ID_BYTES */);
int arks_comm_init(arks_ctx* ctx, int rank, int world, const void* unique_id, const uint32_t* shared, uint32_t n_shared);
int arks_comm_set_shared(arks_ctx* ctx, const uint32_t* shared, uint32_t n_shared);
int arks_fold_quota_allreduce(arks_ctx* ctx, int wait);
void arks_comm_destroy(arks_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* ARKS_GATEWAY_H */
