// arks_host.h — C++ host side above the C ABI (include/arks_gateway.h): what the reference's Go server does around the
// device path. The reference host is Go (pkg/gateway/*.go); no Go toolchain exists in the build image, so the compiled
// host lives here in C++, with the reference's names:
//
//   Batcher          micro-batches the concurrent ext_proc streams of one GPU: a stream reserves a row of the open
//                    pinned staging block and copies its own body; a dispatcher thread closes the block and queues it
//                    on the device (arks_submit_*_async, up to 4 batches in flight, no timer: the next block fills
//                    while earlier ones are on the GPU); a completion thread waits for the oldest batch and hands
//                    every row its decision (callback, or futex wake of a blocked caller); with one batch in flight
//                    (the default) the dispatcher does both, and a blocked caller that finds the batcher idle runs the
//                    cycle for its own row itself.
//   StreamProcessor  Server.Process's per-stream state machine (pkg/gateway/gateway.go:77-138) and the four handlers
//                    (handle_request.go:33-249, handle_response.go:37-268) over decoded ext_proc messages; the gRPC /
//                    protobuf transport stays with the embedding server
//
// Linearisation: dispatcher cycles in order (one device stream); inside a cycle the request batch, then the response
// batch; inside a batch rows in reservation order. Every decision carries (cycle, index, now_unix) so a test can replay the exact order.
#pragma once
#include <stdint.h>

#include <map>
#include <memory>
#include <mutex>

#include <string>
#include <string_view>
#include <vector>

#include "../../include/arks_gateway.h"

namespace arks_host {

struct RequestDecision {
  uint8_t reason, detail, flags;
  int32_t qos, token, pick;
  int64_t cur_usage, limit_max;
  uint64_t cycle;    // dispatcher cycle that carried the request
  uint32_t index;    // row inside that cycle's request batch
  int64_t now_unix;  // the batch's clock reading
  uint32_t gen;      // table generation qos / token refer to: hand it back with the stream's response chunks
  uint32_t model_off, model_len;  // raw span of the body's model string (bit 31 of model_len: contains escapes)
  uint32_t bpe_count;             // BPE tokens of the prompt (0 without a vocabulary)
  // rate-limit report (Batcher::SetRatelimitReport): [0] the requests figure, [1] the tokens figure; rl_entry is the index in
  // qos.RateLimits, ARKS_RL_NONE when there is no such figure (and for every row while the report is off)
  uint8_t rl_entry[2];
  int64_t rl_limit[2], rl_remaining[2];
  // sliding window with the report (Batcher::SetSlidingWindow): rl_sliding 1 when the batch ran with both; then rl_reset[t] is
  // the seconds until figure t's estimate reaches 0 and rl_retry the seconds until a rate-limit 429's entry admits again
  uint32_t rl_reset[2], rl_retry;
  uint8_t rl_sliding;
};
struct ResponseDecision {
  uint8_t reason, counted;
  int64_t usage[3];
  uint64_t cycle;
  uint32_t index;
  int64_t now_unix;
};

struct BatcherOptions {
  uint32_t max_batch = 4096;
  size_t max_bytes = 16u << 20;
  uint32_t linger_us = 0;  // after the first row of a cycle, wait this long for company before submitting (0: submit
                           // at once; under load the next block fills while the previous one is on the GPU)
  uint32_t max_inflight = 1;  // batches queued on the device at once (1..4). A small batch costs the GPU about the same
                              // time whatever its size, so queueing several tiny batches only adds waiting
                              // (tools/host_latency_sweep.py compares the depths); deeper queues help only bulk replay
};

struct BatcherStats {
  uint64_t cycles, request_batches, response_batches, requests, responses, max_request_batch, max_response_batch;
  // where a cycle's time goes (nanoseconds, summed over cycles): waiting for the rows' copies + staging + queueing the
  // device work; waiting for the device; handing the decisions to the rows
  uint64_t ns_submit, ns_device, ns_deliver;
  // the tail: per phase the longest single occurrence and how many took more than 100 us; `gap` is the time between the
  // end of one cycle and the start of the next while rows were waiting (dispatcher wake-up, lock hand-over)
  uint64_t max_ns_submit, max_ns_device, max_ns_deliver, max_ns_gap;
  uint64_t slow_submit, slow_device, slow_deliver, slow_gap;
  // the part of `submit` spent waiting for row owners that had reserved a row but not finished copying into it
  uint64_t ns_fill, max_ns_fill, slow_fill;
  uint64_t late_rows;  // rows that were not filled when their block was cut and went in a later cycle on their own
};

// names the routing headers and the error replies are built from (arks_impl.go: qos -> model, token -> namespace / user)
struct NameTables {
  std::vector<std::string> qos_model, token_namespace, token_user;
  std::vector<int32_t> qos_token;                               // owning ArksToken of each qos entry
  std::vector<std::vector<std::string>> qos_rule_names;         // RateLimit.Type of qos.RateLimits, in order ("rpm", ...)
  std::vector<std::string> qos_quota_name;                      // qos.Quota.Name, "" when none
  std::vector<std::vector<std::string>> qos_quota_item_types;   // QuotaItem.Type of the referenced ArksQuota, in order
};
// generation -> names. The qos / token indices of a decision are positional in the tables of the generation it was made
// on (RequestDecision::gen); while the config plane publishes new generations, a stream's headers and error replies are
// built from ITS generation's names. The last ARKS_GEN_HISTORY generations are kept (as many as the library re-maps
// response rows for).
class NameBook {
 public:
  void Publish(uint32_t gen, NameTables t);
  void Drop(uint32_t gen);                                    // a generation that was announced but not committed
  std::shared_ptr<const NameTables> Of(uint32_t gen) const;   // that generation's; the latest when it is not kept; never null
  std::shared_ptr<const NameTables> Latest() const;

 private:
  mutable std::mutex mu_;
  std::map<uint32_t, std::shared_ptr<const NameTables>> by_gen_;
};

typedef void (*RequestCallback)(void* user, const RequestDecision&);    // run on the batcher's completion thread
typedef void (*ResponseCallback)(void* user, const ResponseDecision&);

class Batcher {
 public:
  Batcher(arks_ctx* ctx, const BatcherOptions& opt);
  ~Batcher();
  Batcher(const Batcher&) = delete;
  Batcher& operator=(const Batcher&) = delete;

  // Blocking, callable from any number of threads. `pick_rand`: the stream's random draw for the weighted pick.
  // A row that can never fit (body larger than max_bytes) is answered with reason 255 without touching the device.
  RequestDecision HandleRequestBody(std::string_view token, std::string_view body, uint64_t pick_rand);
  // `gen`: RequestDecision::gen of the stream's request (the generation its qos index belongs to)
  // `precharged`: RequestDecision.bpe_count of the stream's request when SetPrecharge(true) is in force (N4), else 0
  ResponseDecision HandleResponseBody(int32_t qos, uint32_t gen, std::string_view body, uint8_t flags, uint32_t precharged = 0);
  // Asynchronous form for event-driven servers: returns once the row is staged (the body is copied, the caller's buffer
  // is free again); `cb(user, decision)` runs later on the completion thread, rows of a batch in order. false: the row
  // can never fit, cb is not called.
  bool SubmitRequest(std::string_view token, std::string_view body, uint64_t pick_rand, RequestCallback cb, void* user);
  bool SubmitResponse(int32_t qos, uint32_t gen, std::string_view body, uint8_t flags, ResponseCallback cb, void* user, uint32_t precharged = 0);
  // N4, opt-in (arks_set_precharge): the library charges every admitted request's prompt count to tpm / tpd; from then on the
  // response batches carry each stream's estimate back so that the accounting adds total_tokens - estimate
  int SetPrecharge(bool on);
  bool Precharge() const;
  // opt-in (arks_set_ratelimit_report): request decisions carry the rate-limit figures the StreamProcessor turns into the
  // x-ratelimit-* / retry-after headers. Batches already queued keep the setting they were queued with
  int SetRatelimitReport(bool on);
  bool RatelimitReport() const;
  // opt-in (arks_set_sliding_window): the limiter admits against the current window plus the previous window's remaining
  // share; with the report on, the reset / retry headers and expiresAt name the projected times. Queued batches keep theirs
  int SetSlidingWindow(bool on);
  bool SlidingWindow() const;

  // Config change while streams are in flight (qosconfig informer event): the next generation is built and uploaded on
  // the CALLING (config) thread with batches still running (arks_prepare_tables), then swapped in between two cycles
  // (arks_commit_tables: stream-ordered, counters carried by key on the device). Nothing waits for queued batches to
  // drain; the only exclusion is against the few microseconds in which a cycle submits. Requests decided before the
  // swap keep their (gen, qos); the library re-maps them by key when their response chunks arrive.
  // `names` (optional): the name tables of the generation being published; they enter Names() under the new generation's
  // number BEFORE the swap, so a decision of that generation never meets the previous generation's names.
  int LoadTables(const arks_tables* t, const NameTables* names = nullptr);
  // The same for the object-level plane: arks_upsert_* / arks_delete_* on Context() from the config thread, then
  // ApplyConfig() publishes the store (arks_config_prepare + commit).
  int ApplyConfig(const NameTables* names = nullptr);
  NameBook& Names();
  arks_ctx* Context() const;
  uint32_t Generation() const;  // arks_table_generation of the context

  void SetClock(int64_t (*clock)(void*), void* arg);  // default: time(nullptr)
  BatcherStats Stats() const;
  void ResetTailStats();  // the max_* / slow_* fields start over

 private:
  struct Impl;
  Impl* p_;
};

// ---- ext_proc per-stream state machine --------------------------------------------------------------------------
struct Header {
  std::string key, value;
};
// one table line per object: "T\t<namespace>\t<user>" / "Q\t<token index>\t<model>\t<quota name>\t<rule,rule,..>\t<type,type,..>"
bool ParseNameTables(std::string_view text, NameTables* out);
struct Action {
  enum Kind { kContinueRequestHeaders, kContinueRequestBody, kContinueResponseHeaders, kContinueResponseBody, kImmediate };
  Kind kind = kContinueRequestHeaders;
  int status = 0;                    // kImmediate: HTTP status
  std::vector<Header> set_headers;   // header mutation (continue) or response headers (immediate)
  std::string body;                  // kImmediate: JSON error body (util.go:40-77)
  bool clear_route_cache = false;
};

class StreamProcessor {
 public:
  StreamProcessor(Batcher* batcher, const NameTables* names) : b_(batcher), names_(names) {}  // one fixed configuration
  StreamProcessor(Batcher* batcher, const NameBook* book) : b_(batcher), book_(book) {}       // names follow the generations
  Action OnRequestHeaders(const std::vector<Header>& headers);              // handle_request.go:33-81
  Action OnRequestBody(std::string_view body, uint64_t pick_rand);          // handle_request.go:83-249
  Action OnResponseHeaders(const std::vector<Header>& headers);             // handle_response.go:37-78
  Action OnResponseBody(std::string_view body, bool end_of_stream);         // handle_response.go:80-268
  const RequestDecision& request_decision() const { return req_; }
  const ResponseDecision& response_decision() const { return resp_; }

 private:
  Batcher* b_;
  const NameTables* names_ = nullptr;
  const NameBook* book_ = nullptr;
  std::shared_ptr<const NameTables> NamesOf(uint32_t gen) const;
  std::string token_, buffered_;
  int32_t qos_ = -1;
  uint32_t gen_ = 0;
  bool stream_ = false;
  // the request was admitted with ARKS_FLAG_METERED (N5, arks_set_stream_metering on the Batcher's context): every chunk
  // carries ARKS_RESP_METERED
  bool metered_ = false;
  int status_ = 0;
  RequestDecision req_{};
  ResponseDecision resp_{};
  // what the request phase charged for this stream (N4), handed back with every response chunk: the library subtracts it
  // from the one chunk that carries the usage
  uint32_t Estimate() const { return b_->Precharge() && req_.bpe_count != 0xFFFFFFFFu ? req_.bpe_count : 0u; }
  std::vector<Header> rl_;  // the admitted request's rate-limit headers, for the response headers
};

// generateErrorResponse, util.go:40-77: status + headers + Content-Type + {"error":{"message":..,"code":..}}
Action ErrorResponse(int status, std::vector<Header> headers, const std::string& message);
int ReasonHttpStatus(uint8_t reason);
const char* ReasonHeader(uint8_t reason);
// What the reference puts on the wire for a failed request / response phase: status, x-error-* header with the VALUE the
// Go code sends, and the error message (handle_request.go:97-205, check.go:88-103,140-152, handle_response.go:125-181).
struct ErrorReply {
  int status;
  std::string header, header_value, message;
};
ErrorReply RequestErrorReply(const RequestDecision& d, const NameTables& names, std::string_view token, std::string_view body);
ErrorReply ResponseErrorReply(const ResponseDecision& d, const NameTables& names, int32_t qos, std::string_view last_chunk);
std::string DecodeJsonString(std::string_view raw);  // the model name out of its raw span (jsoniter ReadString semantics)
// end of the fixed window of `rule` ("rpm", ...) that holds now_unix: the 429 body's expiresAt, x-ratelimit-reset-*, retry-after
int64_t WindowEnd(int64_t now_unix, const std::string& rule);
std::string GoDuration(int64_t seconds);  // time.Duration.String() of whole seconds: "1s", "1m0s", "23h59m59s"
// the rate-limit report of a request decision as headers, in wire order: retry-after (a rate-limit 429 only), then limit /
// remaining / reset of the requests figure, then of the tokens figure; none when the decision carries no figure
std::vector<Header> RatelimitHeaders(const RequestDecision& d, const NameTables& names);

}  // namespace arks_host

// ---- flat C surface for tests / load generation (ctypes) ----------------------------------------------------------
extern "C" {
typedef struct arks_host_batcher arks_host_batcher;
int arks_host_create(arks_ctx* ctx, uint32_t max_batch, uint64_t max_bytes, uint32_t linger_us, uint32_t max_inflight,
                     arks_host_batcher** out);
void arks_host_destroy(arks_host_batcher* b);
void arks_host_set_fixed_clock(arks_host_batcher* b, int64_t now_unix);
int arks_host_request(arks_host_batcher* b, const uint8_t* token, uint32_t token_len, const uint8_t* body, uint32_t body_len,
                      uint64_t pick_rand, arks_host::RequestDecision* out);
int arks_host_response(arks_host_batcher* b, int32_t qos, uint32_t gen /* 0xffffffff: the current generation */, const uint8_t* body,
                       uint32_t body_len, uint8_t flags, arks_host::ResponseDecision* out);
int arks_host_load_tables(arks_host_batcher* b, const arks_tables* t);
/* the same with the generation's name tables (format: ParseNameTables), published under the new generation's number */
int arks_host_load_tables_named(arks_host_batcher* b, const arks_tables* t, const char* names, uint32_t names_len);
int arks_host_apply_config_named(arks_host_batcher* b, const char* names, uint32_t names_len);
void arks_host_reset_tail(arks_host_batcher* b);
void arks_host_open_loop_lateness(int64_t out[3]);
void arks_host_open_loop_call_latency(int64_t* buf); /* n entries filled by the next open-loop run: decision - time of the call */
int arks_host_apply_config(arks_host_batcher* b);
int arks_host_set_precharge(arks_host_batcher* b, int on);
int arks_host_set_ratelimit_report(arks_host_batcher* b, int on);
int arks_host_set_sliding_window(arks_host_batcher* b, int on);
/* RatelimitHeaders of a decision under the CURRENT names (arks_host_set_names) as "key: value\n" lines; returns the length, -1
 * if out_cap is too small */
int arks_host_ratelimit_headers(arks_host_batcher* b, const arks_host::RequestDecision* d, char* out, uint32_t out_cap);
int arks_host_response_pre(arks_host_batcher* b, int32_t qos, uint32_t gen, uint32_t precharged, const uint8_t* body, uint32_t body_len,
                           uint8_t flags, arks_host::ResponseDecision* out); /* publishes arks_upsert_* / arks_delete_* done on the context */
// names of the CURRENT generation for the reply shapes of arks_host_stream_transcript / arks_host_*_error_reply (format:
// ParseNameTables); arks_host_load_tables_named / arks_host_apply_config_named publish them together with a generation
int arks_host_set_names(arks_host_batcher* b, const char* text, uint32_t len);
// the reference-exact reply of a failed request / response decision as "status\nheader\nheader value\nmessage"
int arks_host_request_error_reply(arks_host_batcher* b, const arks_host::RequestDecision* d, const uint8_t* token, uint32_t token_len,
                                  const uint8_t* body, uint32_t body_len, char* out, uint32_t out_cap);
int arks_host_response_error_reply(arks_host_batcher* b, const arks_host::ResponseDecision* d, int32_t qos, const uint8_t* chunk,
                                   uint32_t chunk_len, char* out, uint32_t out_cap);
/* `gen`: the generation `qos` belongs to (RequestDecision.gen of the stream's request) */
int arks_host_response_error_reply_gen(arks_host_batcher* b, const arks_host::ResponseDecision* d, int32_t qos, uint32_t gen,
                                       const uint8_t* chunk, uint32_t chunk_len, char* out, uint32_t out_cap);
void arks_host_stats(arks_host_batcher* b, arks_host::BatcherStats* out);
// n requests issued by `threads` stream threads (thread t owns rows t, t+threads, ...; each row is one blocking
// HandleRequestBody). Decisions and per-call latencies (ns) come back in row order; returns wall nanoseconds.
int64_t arks_host_run_requests(arks_host_batcher* b, uint32_t n, uint32_t threads, const uint8_t* bodies, const uint32_t* body_off,
                               const uint32_t* body_len, const uint8_t* tokens, const uint32_t* token_off, const uint64_t* pick_rand,
                               arks_host::RequestDecision* out, int64_t* latency_ns);
int64_t arks_host_run_responses(arks_host_batcher* b, uint32_t n, uint32_t threads, const uint8_t* bodies, const uint32_t* body_off,
                                const uint32_t* body_len, const int32_t* qos, const uint32_t* gen /* or NULL: current */,
                                const uint8_t* flags, arks_host::ResponseDecision* out, int64_t* latency_ns);
// open-loop arrivals at rate_per_s (exponential gaps) from `producers` threads through SubmitRequest; latency_ns[i] =
// decision handed over - scheduled arrival of row i; returns wall nanoseconds
int64_t arks_host_open_loop_requests(arks_host_batcher* b, uint32_t n, double rate_per_s, uint32_t producers, const uint8_t* bodies,
                                     const uint32_t* body_off, const uint32_t* body_len, const uint8_t* tokens, const uint32_t* token_off,
                                     const uint64_t* pick_rand, arks_host::RequestDecision* out, int64_t* latency_ns);
// one ext_proc stream driven end to end; the transcript of actions is written as text (one action per block:
// "kind status clear\nkey: value\n...\n\nbody\n--\n") for comparison with the Python mirror
int arks_host_stream_transcript(arks_host_batcher* b, const char* const* req_hdr_keys,
                                const char* const* req_hdr_vals, uint32_t n_req_hdr, const uint8_t* req_body, uint32_t req_body_len,
                                const char* const* resp_hdr_keys, const char* const* resp_hdr_vals, uint32_t n_resp_hdr,
                                const uint8_t* const* resp_chunks, const uint32_t* resp_chunk_len, uint32_t n_resp_chunks,
                                uint64_t pick_rand, char* out, uint32_t out_cap);
}
