// arks_gateway.cu — libarksgw.so: the H100 (sm_90a) implementation behind include/arks_gateway.h.
//
// Data layout in HBM (DESIGN.md §2)
//   config (replaces the controller-runtime informer cache, pkg/gateway/qosconfig/arks_impl.go):
//     token hash table (open addressing, 64-bit FNV-1a of spec.token -> token index, bytes verified),
//     per token: namespace id, qos CSR; per qos entry: model-name span, quota index, endpoint index,
//     rate-limit CSR (rule, limit); per quota: item CSR (type, limit); per endpoint: backend-weight CSR.
//   state (replaces Redis, pkg/gateway/ratelimiter/redis_impl.go + pkg/gateway/quota/redis_impl.go):
//     rate[rule][qos]   int64   counter of the CURRENT fixed window of `rule` (cache_key.go:73-80); the host
//                               zeroes rate[rule][*] when floor(now/W) advances, which is what a new Redis key is
//     quota[quota][3]   int64   cumulative usage, never reset (quota/redis_impl.go:38-48)
//   per batch: bodies (16-byte aligned spans), tokens, a batch-local group table (qos -> arrivals), results.
//
// Kernels (DESIGN.md section 5; which scan kernel takes a batch depends on its size only)
//   fast_request_kernel /  batches >= 4 096: a lane per document (mask_scan.cuh): SWAR masks over 32-byte chunks read with one
//   fast_response_kernel   whole-sector read each, grammar walk over the tokens outside strings (tables staged by one TMA bulk copy),
//                          member extraction; then the same tail as the exact engine. Declined documents go on a slow list
//   warp_request_kernel /  batches <= 2 048 (the latency path, warp_scan.cuh): a warp per document, body by one TMA bulk copy
//   warp_response_kernel
//   scan_request_kernel    the exact engine (json_engine.cuh): one lane per request, table-driven JSON machine over the body,
//                          token lookup, qos / endpoint match, static decision, registration in the batch-local group table.
//                          <.., FROM_LIST>: over the slow list of the kernels above
//   limit_admit_kernel     one lane per request: closed-form fixed-window admission in arrival order
//                          (SURVEY.md section 8a A6), quota check, one commit per group, weighted pick (A12)
//   rank_hot_groups_kernel arrival ranks inside groups with more than 256 arrivals in one batch (a hot tenant)
//   scan_response_kernel   the exact engine for complete response bodies: usage extraction and the unconditional
//                          counter increments (check.go:47-72) as warp-aggregated 64-bit atomics
//   scan_sse_kernel        all-SSE batches: chunks cut into events (one lane per chunk), events parsed one per lane,
//                          verdicts folded per chunk
//   bpe_scan_kernel /      the token count of the north star (bpe.cuh): content strings -> pre-tokens -> merge loop per
//   bpe_merge_kernel       pre-token, hot merges staged into shared memory by TMA
//   carry_rows_kernel, fold_shared_kernel, gather_shared_kernel   generation swap / shared-quota fold (a few microseconds)
//
// Streams: uploads on `h2d`, everything that touches counters on `stream` (its order is the linearisation).
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <deque>
#include <dlfcn.h>
#include <nccl.h>  // types only: the entry points are looked up with dlsym at arks_comm_init
#include <mutex>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/arks_gateway.h"
#include "json_engine.cuh"
#include "mask_scan.cuh"
#include "warp_scan.cuh"
#include "bpe.cuh"
#include "config_store.h"

using namespace arks;

// ------------------------------------------------------------------------------------------------
// device-side views
// ------------------------------------------------------------------------------------------------
struct TokSlot {
  unsigned long long hash;
  int tok;  // -1 empty
  int pad;
};

struct DevTables {
  const uint8_t* pool;  // string bytes
  // tokens
  const TokSlot* tok_slots;
  uint32_t tok_mask;
  const uint32_t* tok_str_off;  // n_tokens: offset of spec.token in pool
  const uint32_t* tok_str_len;
  const uint32_t* tok_qos_off;  // n_tokens + 1
  // qos entries
  const uint32_t* qos_model_off;
  const uint32_t* qos_model_len;
  const int32_t* qos_quota;
  const int32_t* qos_ep;  // endpoint index for (token namespace, model) or -1
  const uint8_t* qos_vocab;  // BPE vocabulary slot of the entry's model (arks_bind_model_vocab; 0: the default)
  const uint32_t* qos_rl_off;
  const uint8_t* rl_rule;
  const int64_t* rl_value;
  // quotas
  const uint32_t* quota_item_off;
  const uint8_t* qitem_type;
  const int64_t* qitem_value;
  // endpoints
  const uint32_t* ep_backend_off;
  const int32_t* backend_weight;
  // state
  long long* rate;   // [4][n_qos]
  long long* quota;  // [n_quotas][3]
  long long* qdelta; // [n_quotas][3] increments not yet folded into the other GPUs' copies, or null (single-owner keys)
  long long* metrics; // [n_qos][ARKS_METRIC_COLS] Prometheus series (include/arks_gateway.h), or null when not enabled
  uint32_t n_qos;
};

struct ReqDev {  // request batch, device resident
  const uint8_t* bodies;
  const uint32_t* body_off;
  const uint32_t* body_len;
  const uint8_t* tokens;
  const uint32_t* token_off;
  const unsigned long long* pick_rand;  // may be null
  uint32_t n;
  const uint32_t* perm;  // lane -> body: bodies of one warp have (nearly) the same length; null = identity
  uint32_t bpw;          // bodies per warp (1..32): small batches are spread over more warps, see bodies_per_warp()
  // intermediates
  uint8_t* st_reason;  // static reason after scan (ARKS_R_OK == reached the limiter)
  uint8_t* st_flags;
  int32_t* st_qos;
  int32_t* st_tok;
  int32_t* gslot;  // group slot per request or -1
  int32_t* gnext;  // next (earlier-registered) member of the same group, -1 ends the list
  // two-stage scan (large batches): the requests the fast path (mask_scan.cuh) leaves to the exact engine
  uint32_t* slow_list;
  uint32_t* slow_n;  // [1]
  // group table (batch local): qos -> slot
  int32_t* gkey;
  int32_t* ghead;
  int32_t* gcnt;
  long long* gsnap;  // [slot][4] window counters as they were before this batch
  uint32_t gmask;
  // hot groups (> kHotGroup arrivals in this batch): arrival ranks computed by rank_hot_groups_kernel
  int32_t* hot_n;     // [1]
  int32_t* hot_list;  // slots
  int32_t* hotrank;   // per request, valid for members of hot groups
  // results (SoA, packed in one buffer for a single D2H)
  uint8_t* reason;
  uint8_t* detail;
  uint8_t* flags;
  int32_t* qos;
  int32_t* token;
  int32_t* pick;
  long long* cur_usage;
  long long* limit_max;
  uint32_t* model_off;  // raw span of the model string inside the body (host-side error shaping)
  uint32_t* model_len;  // bit 31: the span contains a backslash
  uint32_t* bpe;        // BPE tokens of the prompt text (0 without a vocabulary)
  int precharge;  // N4: admitted requests charge their BPE count to the token-type rules
  int meter;      // N5: stream requests without include_usage are decided and metered instead of refused
};

struct RespDev {
  const uint8_t* bodies;
  const uint32_t* body_off;
  const uint32_t* body_len;
  const int32_t* qos;
  const uint8_t* flags;
  uint32_t n;
  const uint32_t* perm;  // lane -> body (see ReqDev)
  uint32_t bpw;          // bodies per warp
  uint8_t* reason;
  uint8_t* counted;
  long long* usage;  // 3n
  uint32_t* slow_list;  // two-stage scan: the bodies left to the exact engine
  uint32_t* slow_n;
  uint32_t* bpe;        // BPE tokens of the completion text (0 without a vocabulary)
  const uint32_t* precharged;  // n or null: what the request phase charged the token-type rules for this stream (N4)
};

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
// automaton tables (generated header json_tables.h): global copies, staged into shared memory once per block so that the
// two lookups per byte are LDS (32 banks, random 2-byte reads) instead of constant-cache replays
__device__ __align__(16) const uint8_t g_json_cls[256] = ARKS_JSON_CLASS_TABLE;
__device__ __align__(16) const uint8_t g_json_tab_j[kJsonStatesJ * kJsonClasses] = ARKS_JSON_TABLE_J;
__device__ __align__(16) const uint8_t g_json_tab_e[kJsonStatesE * kJsonClasses] = ARKS_JSON_TABLE_E;

template <bool NEED_J, bool NEED_E>
struct JsonSmem {
  alignas(16) uint8_t tab_j[NEED_J ? kJsonStatesJ * kJsonClasses : 16];
  alignas(16) uint8_t tab_e[NEED_E ? kJsonStatesE * kJsonClasses : 16];
  alignas(16) uint8_t cls[256];
  // Issue the table copies as one cp.async group (all threads of the block). The caller overlaps them with other work,
  // then waits for the group and calls __syncthreads() before the first lookup.
  __device__ __forceinline__ JsonTables stage_async() {
    auto copy = [&](uint8_t* dst, const uint8_t* src, int bytes) {
      for (int o = threadIdx.x * 16; o < bytes; o += blockDim.x * 16)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(dst + o)), "l"(src + o));
    };
    copy(cls, g_json_cls, 256);
    if (NEED_J) copy(tab_j, g_json_tab_j, kJsonStatesJ * kJsonClasses);
    if (NEED_E) copy(tab_e, g_json_tab_e, kJsonStatesE * kJsonClasses);
    asm volatile("cp.async.commit_group;");
    return JsonTables{cls, tab_j, tab_e};
  }
};
static_assert((kJsonStatesJ * kJsonClasses) % 16 == 0 && (kJsonStatesE * kJsonClasses) % 16 == 0, "tables are copied in 16-byte pieces");

// ---- 1-D bulk copies (TMA: cp.async.bulk, SASS UBLKCP) completed on an mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(bar);
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(a), "r"(parity)
      : "memory");
}
// global -> shared, `bytes` a multiple of 16, both addresses 16-byte aligned; completes `bytes` transaction bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   (uint32_t)__cvta_generic_to_shared(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// parse state of a request (two-stage scan): what the body says, before any table lookup
constexpr uint8_t PS_STREAM = 1;     // "stream": true
constexpr uint8_t PS_STREAM_OK = 2;  // stream_options.include_usage == true
constexpr uint8_t PS_BAD = 0x40;     // the body does not decode (400 x-error-request-body-processing)

// one 32-byte chunk (one sector): sm_90 has no 256-bit load, so two 128-bit loads issued back to back, with no bound check
// between them. p must be 32-byte aligned
__device__ __forceinline__ void ld_nc_v8(const uint4* p, uint4& a, uint4& b) {
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w), "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w)
               : "l"(p));
}
__device__ __forceinline__ uint4 ld_nc_v4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// ------------------------------------------------------------------------------------------------
// Warp-tiled body feed.
//
// One warp owns 32 bodies, one per lane. The bodies are streamed through shared memory in windows of kWin bytes per
// body with a kStages-deep cp.async pipeline: in every stage the warp copies 32 x kWin bytes with 16-byte LDGSTS
// (8 lanes cover one 128-byte line of one body, so HBM sees full lines), and each lane then parses its own kWin
// bytes out of shared memory. Unit u of body b sits at 16-byte slot u*32 + ((b + u) & 31): the 8 lanes that store
// one body's line hit 8 different bank groups, and the 32 lanes that each read "their" unit u hit 32 different
// slots of one 512-byte row, so both sides of the transpose are conflict-free when lanes move in lock step.
// ------------------------------------------------------------------------------------------------
// A micro-batch whose bodies fit here travels as ONE upload (bodies appended to the offsets / tokens block) on the compute
// stream itself: one copy and one cross-stream event less on the path a lone request takes.
constexpr size_t kSmallBatchBytes = 256 << 10;
constexpr size_t kTinyBatchBytes = 16 << 10;  // below this the bodies ride in the meta block's upload

constexpr int kHotGroup = 256;  // above this many arrivals of one qos entry in a batch the member list is not walked
#ifndef ARKS_KWIN
#define ARKS_KWIN 128
#endif
#ifndef ARKS_KSTAGES
#define ARKS_KSTAGES 3
#endif
#ifndef ARKS_SSE_STAGES
#define ARKS_SSE_STAGES 2
#endif
#ifndef ARKS_MINBLK
#define ARKS_MINBLK 7
#endif
#ifndef ARKS_SSE_MINBLK
#define ARKS_SSE_MINBLK 7
#endif
constexpr int kWin = ARKS_KWIN;                  // bytes per body per stage
constexpr int kUnits = kWin / 16;                // 16-byte units per body per stage
constexpr int kStages = ARKS_KSTAGES;
constexpr int kStageBytes = 32 * kWin;           // per warp per stage
constexpr int kWarpsPerBlock = 2;
constexpr int kMinBlocks = ARKS_MINBLK;          // resident blocks per SM the scan kernels are compiled for
constexpr int kSmemPerBlock = kWarpsPerBlock * kStages * kStageBytes;
static_assert(kUnits == 8 || kUnits == 4, "window = 4 or 8 units");

__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gptr, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_addr), "l"(gptr), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

// issue the copies of window `w` (bytes [w*kWin, (w+1)*kWin) of all 32 bodies) into stage buffer `stage_smem`:
// kUnits neighbouring lanes copy one body's window, 32 / kUnits bodies per pass
__device__ __forceinline__ void issue_window(uint32_t stage_smem, const uint8_t* my_body, uint32_t my_padded, uint32_t w,
                                             uint32_t lane) {
  const uint32_t u = lane & (kUnits - 1);   // unit within the window handled by this lane
  const uint32_t off = w * kWin + u * 16;   // byte offset inside the body
#pragma unroll
  for (int k = 0; k < kUnits; k++) {
    const uint32_t b = lane / kUnits + (32 / kUnits) * k;  // body (== owning lane) this copy belongs to
    const uint8_t* base = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, (unsigned long long)my_body, b));
    const uint32_t plen = __shfl_sync(0xffffffffu, my_padded, b);
    const uint32_t slot = u * 32 + ((b + u) & 31);
    const bool in = off < plen;
    cp_async16(stage_smem + slot * 16, in ? base + off : base, in ? 16u : 0u);
  }
}


// Stream bytes [0, end) of 32 spans, one per lane (lanes without work pass end == 0), through a STAGES-deep window
// pipeline. start() issues the first STAGES-1 windows (one cp.async group each) and returns, so the caller can do
// unrelated long-latency work before run(); run() calls per_window(wbeg, lim, load) on every lane for every window,
// load(u) returns the lane's own 16-byte unit u (absolute unit index inside the span).
template <int STAGES>
struct WindowPipe {
  const uint8_t* body;
  uint8_t* warp_smem;
  uint32_t end, padded, n_win, lane, smem0;
  __device__ __forceinline__ void start(const uint8_t* body_, uint32_t end_, uint8_t* warp_smem_) {
    body = body_; end = end_; warp_smem = warp_smem_;
    lane = threadIdx.x & 31;
    padded = (end + 15u) & ~15u;
    uint32_t maxlen = end;
#pragma unroll
    for (int d = 16; d; d >>= 1) maxlen = max(maxlen, __shfl_xor_sync(0xffffffffu, maxlen, d));
    n_win = (maxlen + kWin - 1) / kWin;
    smem0 = (uint32_t)__cvta_generic_to_shared(warp_smem);
#pragma unroll
    for (int s = 0; s < STAGES - 1; s++) {
      if ((uint32_t)s < n_win) issue_window(smem0 + s * kStageBytes, body, padded, s, lane);
      cp_async_commit();
    }
  }
  template <class F>
  __device__ __forceinline__ void run(F&& per_window) {
    for (uint32_t w = 0; w < n_win; w++) {
      const uint32_t nxt = w + STAGES - 1;
      if (nxt < n_win) issue_window(smem0 + (nxt % STAGES) * kStageBytes, body, padded, nxt, lane);
      cp_async_commit();
      cp_async_wait<STAGES - 1>();
      __syncwarp();
      const uint8_t* st = warp_smem + (w % STAGES) * kStageBytes;
      const uint32_t wbeg = w * kWin;
      const uint32_t ln = lane;
      per_window(wbeg, min(end, wbeg + kWin), [st, wbeg, ln](uint32_t u) {
        const uint32_t ul = u - (wbeg >> 4);
        const uint4 v = *reinterpret_cast<const uint4*>(st + (ul * 32 + ((ln + ul) & 31)) * 16);
        Unit16 q;
        q.w[0] = v.x; q.w[1] = v.y; q.w[2] = v.z; q.w[3] = v.w;
        return q;
      });
      __syncwarp();  // everyone is done with this stage before it is overwritten
    }
    cp_async_wait<0>();
  }
};
// Parse bytes [begin, end) (begin < 16) of 32 spans with machine `m`, one span per lane.
// SCHED: 0 = consume_t (any machine), 1 = consume_evsync, 8 = consume_rounds<8> (JsonT; all lanes must call)
template <int SCHED, int STAGES, class M>
__device__ __forceinline__ void feed_pipe(M& m, WindowPipe<STAGES>& pipe, uint32_t begin) {
  uint32_t pos = begin;
  const uint32_t end = pipe.end;
  pipe.run([&](uint32_t wbeg, uint32_t lim, auto&& load) {
    if constexpr (SCHED != 0) {
      // special-byte masks of this window's units, computed up front with the warp converged (inside the parse loop the
      // lanes cross unit boundaries at different iterations, so the same code would run ~7 lanes wide)
      uint32_t mk[kUnits / 2];
#pragma unroll
      for (int j = 0; j < kUnits / 2; j++) mk[j] = 0;
#pragma unroll
      for (int j = 0; j < kUnits; j++) {
        if (wbeg + 16u * j < lim) {
          const Unit16 q = load((wbeg >> 4) + j);
          mk[j >> 1] |= special_mask16(q.w[0], q.w[1], q.w[2], q.w[3]) << (16 * (j & 1));
        }
      }
      auto mask_of = [&](uint32_t u, uint32_t, uint32_t, uint32_t, uint32_t) {
        const uint32_t ul = u - (wbeg >> 4);
        uint32_t w;
        if constexpr (kUnits == 8) w = (ul & 4) ? ((ul & 2) ? mk[3] : mk[2]) : ((ul & 2) ? mk[1] : mk[0]);
        else w = (ul & 2) ? mk[1] : mk[0];
        return (w >> (16 * (ul & 1))) & 0xffffu;
      };
      if constexpr (SCHED == 1) consume_evsync(m, pos, lim, load, mask_of);
      else consume_rounds<SCHED>(m, pos, lim, load, mask_of);
    } else {
      consume_t(m, pos, lim, load);
    }
    if (m.dead()) pos = end;  // nothing further can change the verdict
  });
}
template <int STAGES = kStages, int SCHED = 0, class M>
__device__ __forceinline__ void feed_tiled(M& m, const uint8_t* body, uint32_t begin, uint32_t end, uint8_t* warp_smem) {
  WindowPipe<STAGES> pipe;
  pipe.start(body, end, warp_smem);
  feed_pipe<SCHED>(m, pipe, begin);
}

__device__ __forceinline__ unsigned long long fnv1a64(const uint8_t* p, uint32_t n) {
  unsigned long long h = 0xcbf29ce484222325ull;
#pragma unroll 8
  for (uint32_t i = 0; i < n; i++) h = (h ^ p[i]) * 0x100000001b3ull;  // the loads of a round go out together
  return h;
}

// compare the (possibly escaped) model span of a body with a pool string
__device__ bool model_equals(const uint8_t* body, uint32_t m_start, uint32_t m_rawlen, uint32_t m_esc, const uint8_t* name, uint32_t nlen) {
  const uint8_t* p = body + m_start;
  if (!m_esc) {
    if (m_rawlen != nlen) return false;
    uint32_t diff = 0;  // no early exit: the loads of all bytes are in flight together
    for (uint32_t i = 0; i < nlen; i++) diff |= (uint32_t)(p[i] ^ name[i]);
    return diff == 0;
  }
  uint32_t k = 0;
  bool ok = true;
  decode_span(p, m_rawlen, [&](uint8_t b) {
    if (k >= nlen || name[k] != b) ok = false;
    k++;
  });
  return ok && k == nlen;
}

// GetQosByToken's first half: the first ArksToken whose spec.token equals the bearer (arks_impl.go:303-317), or -1.
// A chain of dependent global loads (token bytes -> hash slot -> token string).
__device__ __forceinline__ int32_t lookup_token(const DevTables& T, const ReqDev& B, uint32_t i) {
  const uint8_t* tk = B.tokens + B.token_off[i];
  const uint32_t tkl = B.token_off[i + 1] - B.token_off[i];
  const unsigned long long h = fnv1a64(tk, tkl);
  uint32_t s = (uint32_t)h & T.tok_mask;
  for (;;) {
    TokSlot e = T.tok_slots[s];
    if (e.tok < 0) return -1;
    if (e.hash == h && T.tok_str_len[e.tok] == tkl) {
      const uint8_t* q = T.pool + T.tok_str_off[e.tok];
      uint32_t diff = 0;
      for (uint32_t k = 0; k < tkl; k++) diff |= (uint32_t)(q[k] ^ tk[k]);
      if (diff == 0) return e.tok;
    }
    s = (s + 1) & T.tok_mask;
  }
}

// The same lookup in two halves for kernels that have other work to put in between (the fast path: hash and first probe before
// pass A, the string compare after pass C — the two dependent round trips to L2 then run under the scan instead of after it).
struct TokProbe {
  unsigned long long h;
  uint32_t s;
  TokSlot e;
};
__device__ __forceinline__ TokProbe lookup_token_begin(const DevTables& T, const ReqDev& B, uint32_t i) {
  const uint8_t* tk = B.tokens + B.token_off[i];
  const uint32_t tkl = B.token_off[i + 1] - B.token_off[i];
  TokProbe p;
  p.h = fnv1a64(tk, tkl);
  p.s = (uint32_t)p.h & T.tok_mask;
  p.e = T.tok_slots[p.s];
  return p;
}
__device__ __forceinline__ int32_t lookup_token_end(const DevTables& T, const ReqDev& B, uint32_t i, TokProbe p) {
  const uint8_t* tk = B.tokens + B.token_off[i];
  const uint32_t tkl = B.token_off[i + 1] - B.token_off[i];
  for (;;) {
    if (p.e.tok < 0) return -1;
    if (p.e.hash == p.h && T.tok_str_len[p.e.tok] == tkl) {
      const uint8_t* q = T.pool + T.tok_str_off[p.e.tok];
      uint32_t diff = 0;
#pragma unroll 8
      for (uint32_t k = 0; k < tkl; k++) diff |= (uint32_t)(q[k] ^ tk[k]);  // eight pairs of loads in flight per round
      if (diff == 0) return p.e.tok;
    }
    p.s = (p.s + 1) & T.tok_mask;
    p.e = T.tok_slots[p.s];
  }
}

// Everything HandleRequestBody decides after the body is decoded and before the limiter (handle_request.go:106-171):
// model present, token known, model in the token's qos list, model an endpoint of the namespace, stream options; then the
// registration in the batch-local group table. `pstate`: PS_* of the body, (m_start, m_rawlen, m_esc): its model span.
__device__ __forceinline__ void resolve_request(const DevTables& T, const ReqDev& B, uint32_t i, const uint8_t* body, int32_t tok,
                                                uint8_t pstate, uint32_t m_start, uint32_t m_rawlen, uint32_t m_esc) {
  uint8_t reason = ARKS_R_OK, flags = 0, claimer = 0;
  int32_t qos = -1, slot = -1, tok_seen = -1;  // the token is only reported once the decision reached GetQosByToken
  // N5: a stream without include_usage is metered. The bit is set whatever the decision (the BPE scan counts the wide key
  // set for it); limit_admit reports it only on admitted rows
  const uint8_t metered = B.meter && (pstate & (PS_BAD | PS_STREAM | PS_STREAM_OK)) == PS_STREAM ? ARKS_FLAG_METERED : 0;
  do {
    if (pstate & PS_BAD) { reason = ARKS_R_REQUEST_BODY; break; }            // handle_request.go:97-104
    if (m_rawlen == 0) { reason = ARKS_R_NO_MODEL; break; }                  // :106-115
    tok_seen = tok;
    if (tok < 0) { reason = ARKS_R_TOKEN_NOT_FOUND; break; }
    for (uint32_t q = T.tok_qos_off[tok]; q < T.tok_qos_off[tok + 1]; q++)
      if (model_equals(body, m_start, m_rawlen, m_esc, T.pool + T.qos_model_off[q], T.qos_model_len[q])) { qos = (int32_t)q; break; }
    if (qos < 0) { reason = ARKS_R_MODEL_NOT_IN_TOKEN; break; }
    if (T.qos_ep[qos] < 0) { reason = ARKS_R_NO_MODEL_BACKENDS; break; }   // handle_request.go:137-154
    const bool stream = pstate & PS_STREAM;
    if (stream && !(pstate & PS_STREAM_OK) && !metered) { reason = ARKS_R_STREAM_OPTIONS; break; }  // :156-171
    flags = stream ? 1 : 0;
    // register in the batch-local group table: qos -> dense slot, arrival count, member list
    uint32_t g = ((uint32_t)qos * 2654435761u) & B.gmask;
    for (;;) {
      int32_t prev = atomicCAS(&B.gkey[g], -1, qos);
      if (prev == -1) {
        // the claimer snapshots the group's window counters: limit_admit reads only the snapshot, so the one lane
        // that later writes the counters back races with nobody
        claimer = 1;
#pragma unroll
        for (int r = 0; r < 4; r++) B.gsnap[(size_t)g * 4 + r] = T.rate[(size_t)r * T.n_qos + qos];
        break;
      }
      if (prev == qos) break;
      g = (g + 1) & B.gmask;
    }
    // the table is memset to 0xff: counts start at -1. The arrival that takes a group past the hot threshold lists it.
    if (atomicAdd(&B.gcnt[g], 1) + 2 == kHotGroup + 1) B.hot_list[atomicAdd(B.hot_n, 1) + 1] = (int32_t)g;
    B.gnext[i] = atomicExch(&B.ghead[g], (int32_t)i);
    slot = (int32_t)g;
  } while (0);
  B.st_reason[i] = reason;
  B.st_flags[i] = flags | metered | (claimer << 7);
  B.st_qos[i] = qos;
  B.st_tok[i] = tok_seen;
  B.gslot[i] = slot;
}

// ------------------------------------------------------------------------------------------------
// Lane assignment: bodies are handed to lanes in order of length (counting sort, arbitrary order inside a bucket). Lanes of a warp run in lock step window by window, so a warp is as slow as its longest / densest
// body; with equal lengths, bodies that share a shape (the completions of one serving stack, the requests of one
// application) also reach their structure-dense regions in the same windows. Decisions do not depend on the
// assignment: every output is indexed by the body, and arrival order enters only through limit_admit's ranks.
// ------------------------------------------------------------------------------------------------
constexpr int kLenBuckets = 4096;  // byte-exact below 2 KiB (a one-byte offset already misaligns two bodies), 32-byte steps above
__device__ __forceinline__ uint32_t len_bucket(uint32_t len) {
  return len < 2048u ? len : min(2048u + ((len - 2048u) >> 5), (uint32_t)kLenBuckets - 1u);
}

__global__ void len_hist_kernel(const uint32_t* body_len, uint32_t n, uint32_t* hist) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < n;
  const uint32_t b = live ? len_bucket(body_len[i]) : 0xffffffffu;
  const unsigned peers = __match_any_sync(0xffffffffu, b);  // one atomic per distinct bucket in the warp
  if (live && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[b], (uint32_t)__popc(peers));
}
static_assert(kLenBuckets == 4096, "len_scan_kernel: one block of 1024 threads, 4 counters each");
// exclusive scan of the kLenBuckets counters in place (one block of 1024 threads, 4 counters each)
__global__ void __launch_bounds__(1024) len_scan_kernel(uint32_t* hist) {
  __shared__ uint32_t warp_tot[32];
  const uint32_t t = threadIdx.x;
  uint32_t v[4], sum = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { v[k] = hist[4 * t + k]; sum += v[k]; }
  uint32_t incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
    if ((t & 31) >= (uint32_t)d) incl += o;
  }
  if ((t & 31) == 31) warp_tot[t >> 5] = incl;
  __syncthreads();
  if (t < 32) {
    uint32_t w = warp_tot[t], wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(0xffffffffu, wi, d);
      if (t >= (uint32_t)d) wi += o;
    }
    warp_tot[t] = wi - w;
  }
  __syncthreads();
  uint32_t base = warp_tot[t >> 5] + incl - sum;
#pragma unroll
  for (int k = 0; k < 4; k++) { hist[4 * t + k] = base; base += v[k]; }
}
__global__ void len_scatter_kernel(const uint32_t* body_len, uint32_t n, uint32_t* offs, uint32_t* perm) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < n;
  const uint32_t b = live ? len_bucket(body_len[i]) : 0xffffffffu;
  const unsigned peers = __match_any_sync(0xffffffffu, b);
  const int leader = __ffs(peers) - 1;
  const uint32_t lane = threadIdx.x & 31;
  uint32_t base = 0;
  if (live && (int)lane == leader) base = atomicAdd(&offs[b], (uint32_t)__popc(peers));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (live) perm[base + __popc(peers & ((1u << lane) - 1u))] = i;
}

// ------------------------------------------------------------------------------------------------
// kernel 1: scan_request — A3 (body parse), A4 (GetQosByToken), A5 (GetModelList) of SURVEY.md §8a
// ------------------------------------------------------------------------------------------------
// FROM_LIST: second stage of the two-stage scan — the requests the fast path left to the exact engine (B.slow_list).
template <int SCHED, bool FROM_LIST>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, kMinBlocks) scan_request_kernel(DevTables T, ReqDev B) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t n = FROM_LIST ? *B.slow_n + 1u : B.n;  // the counter starts at -1 (it is cleared together with the 0xff tables)
  const uint32_t lane_id = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * B.bpw + (threadIdx.x & 31);
  if (FROM_LIST && ((blockIdx.x * blockDim.x) >> 5) * B.bpw >= n) return;  // nothing left for this block
  const bool live = (threadIdx.x & 31) < B.bpw && lane_id < n;
  const uint32_t i = live ? (FROM_LIST ? B.slow_list[lane_id] : B.perm ? B.perm[lane_id] : lane_id) : 0;  // the body this lane parses
  const uint8_t* body = B.bodies + (live ? B.body_off[i] : 0);
  const uint32_t len = live ? B.body_len[i] : 0;

  uint32_t stack_words[kStackWords];  // local memory, touched only beyond 32 levels of nesting
  __shared__ __align__(16) JsonSmem<true, false> json_smem;
  const JsonTables tabs = json_smem.stage_async();
  WindowPipe<kStages> pipe;
  pipe.start(body, len, smem + (threadIdx.x >> 5) * (kStages * kStageBytes));

  // GetQosByToken does not need the body, so it runs here, while the automaton tables and the first body windows are
  // still in flight.
  int32_t tok = -1;
  if (live) tok = lookup_token(T, B, i);
  cp_async_wait<kStages - 1>();  // the table group is the oldest one
  __syncthreads();

  JsonCold cold;  // rarely touched parse state: local memory on purpose (json_engine.cuh)
  JsonT m;
  m.init(K_REQ, body, stack_words, &cold, tabs);
  feed_pipe<SCHED>(m, pipe, 0);
  if (!live) return;

  const bool parsed = m.ok_at_end();
  const uint8_t pstate = !parsed ? PS_BAD
                                 : (uint8_t)((cold.stream3 == 2 ? PS_STREAM : 0) | (cold.so_present && cold.iu3 == 2 ? PS_STREAM_OK : 0));
  const uint32_t m_rawlen = parsed ? cold.m_rawlen : 0;
  B.model_off[i] = m_rawlen ? cold.m_start : 0u;
  B.model_len[i] = m_rawlen ? (m_rawlen | (cold.m_esc ? 0x80000000u : 0u)) : 0u;
  B.bpe[i] = 0;
  resolve_request(T, B, i, body, tok, pstate, cold.m_start, m_rawlen, cold.m_esc);
}

// ------------------------------------------------------------------------------------------------
// kernel 1': the fast path (mask_scan.cuh) — first stage of the two-stage scan of large batches. One lane per body, three
// convergent passes; a body it accepts is decided here (same tail as the exact kernel), a body it declines is appended
// to B.slow_list for scan_*_kernel<.., FROM_LIST>.
// ------------------------------------------------------------------------------------------------
__device__ __align__(16) const FastTablesInit g_fast_tables{};
static_assert(sizeof(FastTables) % 16 == 0, "staged with one bulk copy");
constexpr int kFastThreads = 128;
struct FastBlockSmem;

// the grammar tables of mask_scan.cuh into shared memory: ONE 1-D bulk copy (TMA) per block, completion on an mbarrier
__device__ __forceinline__ void stage_fast_tables(FastTables* dst, uint64_t* bar) {
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(bar, (uint32_t)sizeof(FastTables));
    bulk_g2s(dst, &g_fast_tables.t, (uint32_t)sizeof(FastTables), bar);
  }
  __syncthreads();        // the barrier is initialised before anybody polls it
  mbar_wait(bar, 0);
}

// Shared memory of a fast-path block: the grammar tables and the per-document scratch of mask_scan.cuh, interleaved by slot.
struct __align__(128) FastBlockSmem {
  FastTables tabs;
  uint64_t bar;
  uint32_t tb[kFastChunks * kFastThreads];
  uint32_t mem[2 * kFastMaxMembers * kFastThreads];
  uint32_t ring[16 * kFastThreads];  // the current and the next chunk of every lane (dynamic byte access for escapes)
  // hand-over between pass A (thread t scans the document of slot t) and passes B/C (thread t walks slot order[t]):
  uint32_t hand[5 * kFastThreads];   // bs_lo, bs_hi, nz_lo, nz_hi, tokens + 1 (0: pass A declined)
  uint32_t hist[64];
  uint32_t order[kFastThreads];
  uint32_t slot[kFastThreads];       // which of the block's documents column t holds (pass A takes them in order of length)
};

// Pass A for the body of slot threadIdx.x; its result goes to sm.hand. Streams the body through a 4-deep register queue of
// 32-byte chunks (the loads of chunks j+1..j+4 are in flight while chunk j is processed): a lane-per-document kernel has one
// partial wave of warps per SM, so memory latency has to be covered inside the lane, not by other warps. One copy of the
// chunk code (the instruction cache is small).
__device__ __forceinline__ void fast_pass_a(const uint8_t* body, uint32_t len, FastBlockSmem& sm) {
  const uint32_t t = threadIdx.x;
  uint32_t ntok1 = 0;
  FastScratch s{sm.tb + t, sm.mem + t, (uint32_t)kFastThreads, 0u, 0u, 0u, 0u};
  if (len != 0 && len <= kFastMaxLen) {
    const FastRing ring{sm.ring + t, (uint32_t)kFastThreads};
    const uint32_t nch = (len + 31) >> 5, plen = (len + 15u) & ~15u;
    FastCarry c{0, 0, 0, 0};
    const uint4* p = reinterpret_cast<const uint4*>(body);
    const uint4 z = make_uint4(0, 0, 0, 0);
    // A body that starts on a 32-byte boundary (every packer of this repository does that; the ABI asks for 16) is read a
    // whole sector at a time (ld_nc_v8), without a bound check between its halves. Reading 16 bytes past a body's padded
    // end stays inside the staging buffer (allocated with slack) and is masked off by the chunk's valid count.
    const bool a32 = (reinterpret_cast<uintptr_t>(body) & 31u) == 0;
    auto ld = [&](uint32_t j, uint4& a, uint4& b) {
      a = z; b = z;
      if (j < nch) {
        if (a32) ld_nc_v8(p + 2 * j, a, b);
        else {
          a = ld_nc_v4(p + 2 * j);
          if (32 * j + 16 < plen) b = ld_nc_v4(p + 2 * j + 1);  // never past the 16-byte padding
        }
      }
    };
    uint4 a0, b0, a1, b1, a2, b2, a3, b3;
    ld(0, a0, b0); ld(1, a1, b1); ld(2, a2, b2); ld(3, a3, b3);
    {
      const uint32_t w0[8] = {a0.x, a0.y, a0.z, a0.w, b0.x, b0.y, b0.z, b0.w};
      ring.put(0, w0);
    }
    uint32_t ntok = 0;
    // (Four copies of this step with the queue rotating by name instead of by 24 register moves made pass A faster and the
    // whole kernel slower: the code the later passes share the instruction cache with grew by a third.)
#pragma unroll 1
    for (uint32_t j = 0; j < nch; j++) {
      const uint32_t w[8] = {a0.x, a0.y, a0.z, a0.w, b0.x, b0.y, b0.z, b0.w};
      a0 = a1; b0 = b1; a1 = a2; b1 = b2; a2 = a3; b2 = b3;
      ld(j + 4, a3, b3);
      {
        const uint32_t wn[8] = {a0.x, a0.y, a0.z, a0.w, b0.x, b0.y, b0.z, b0.w};
        ring.put(j + 1, wn);  // the chunk after the current one is at hand too (a \uXXXX may straddle the boundary)
      }
      uint32_t bm, tbw;
      fast_chunk(w, min(len - 32 * j, 32u), ring, len, 32 * j, c, &tbw, &bm);
      s.tb(j) = tbw;
      ntok += __popc(tbw);
      const uint32_t bit = 1u << (j & 31);
      if (j < 32) { s.bs_lo |= bm ? bit : 0u; s.nz_lo |= tbw ? bit : 0u; }
      else { s.bs_hi |= bm ? bit : 0u; s.nz_hi |= tbw ? bit : 0u; }
    }
    if (!(c.bad || c.in_str)) ntok1 = ntok + 1;
  }
  sm.hand[0 * kFastThreads + t] = s.bs_lo;
  sm.hand[1 * kFastThreads + t] = s.bs_hi;
  sm.hand[2 * kFastThreads + t] = s.nz_lo;
  sm.hand[3 * kFastThreads + t] = s.nz_hi;
  sm.hand[4 * kFastThreads + t] = ntok1;
}

// A block's 128 documents are taken in two different orders, both found with a counting sort in shared memory (64 buckets):
//   pass A in order of LENGTH (chunks): its loop runs as long as the longest document of the warp. The batch itself stays in
//     arrival order — every block holds the same mix of lengths and all blocks finish together; a globally length-sorted batch
//     put all the long documents into the last blocks, which then ran on alone, and the sort
//     kernels cost time of their own;
//   passes B / C in order of the number of bytes outside strings: one table step per such byte, and documents of one length
//     still differ 2x in structure.
// Returns the position thread t takes in that order. All threads of the block call it.
__device__ __forceinline__ uint32_t fast_block_order(FastBlockSmem& sm, uint32_t bucket, bool on) {
  const uint32_t t = threadIdx.x;
  if (!on) return t;
  if (t < 64) sm.hist[t] = 0;
  __syncthreads();
  const uint32_t mine = atomicAdd(&sm.hist[bucket], 1u);
  __syncthreads();
  uint32_t before = 0;
  for (uint32_t k = 0; k < bucket; k++) before += sm.hist[k];
  sm.order[before + mine] = t;
  __syncthreads();
  const uint32_t r = sm.order[t];
  __syncthreads();  // hist / order are reused by the next call
  return r;
}

// passes B and C over the scratch in column u; false: declined
// All 32 lanes of the warp call this (live: the lane has a document). The lanes leave pass A, the walk and the member pass
// at different times; without a __syncwarp() each goes on alone and the code behind runs once per straggler (the request
// tail ran a handful of lanes wide). The kernel is bound by the warp instructions it issues, so for requests the lanes wait
// here to issue the next pass together; for completions, whose tail is the warp-wide accounting anyway,
// waiting costs more than it saves and the lanes run on.
template <int KIND, int WALK>
__device__ __forceinline__ bool fast_pass_bc(bool live, const uint8_t* body, uint32_t len, FastBlockSmem& sm, uint32_t u, FastOut& o) {
  if (KIND == K_REQ) __syncwarp();
  live = live && sm.hand[4 * kFastThreads + u] != 0;
  const FastScratch s{sm.tb + u, sm.mem + u, (uint32_t)kFastThreads, sm.hand[0 * kFastThreads + u], sm.hand[1 * kFastThreads + u],
                      sm.hand[2 * kFastThreads + u], sm.hand[3 * kFastThreads + u]};
  const uint32_t nch = (len + 31) >> 5;
  int nmem = -1;
  if (live) nmem = fast_walk<WALK>(body, sm.tabs, s, nch, KIND == K_REQ ? kFastKeyLensReq : kFastKeyLensResp);
  if (KIND == K_REQ) __syncwarp();
  bool ok = false;
  if (nmem >= 0) ok = fast_members<KIND>(body, s, nch, nmem, o);
  if (KIND == K_REQ) __syncwarp();
  return ok;
}

template <int WALK>
__global__ void __launch_bounds__(kFastThreads) fast_request_kernel(DevTables T, ReqDev B, int regroup) {
  extern __shared__ __align__(1024) uint8_t smem[];
  FastBlockSmem& sm = *reinterpret_cast<FastBlockSmem*>(smem);
  stage_fast_tables(&sm.tabs, &sm.bar);
  const uint32_t base = blockIdx.x * blockDim.x;
  TokProbe probe{};
  {
    const uint32_t own = base + threadIdx.x;
    const uint32_t len0 = own < B.n ? B.body_len[B.perm ? B.perm[own] : own] : 0u;
    const uint32_t a = fast_block_order(sm, min((len0 + 31) >> 5, 63u), regroup != 0);  // the document pass A scans here
    const bool in = base + a < B.n;
    const uint32_t i = in ? (B.perm ? B.perm[base + a] : base + a) : 0;
    if (in && (regroup & 127) < 2) probe = lookup_token_begin(T, B, i);  // consumed after pass C (same thread, same document)
    fast_pass_a(B.bodies + (in ? B.body_off[i] : 0), in && !(regroup & 512) ? B.body_len[i] : 0u, sm);
    sm.slot[threadIdx.x] = a;
  }
  if (regroup & 256) return;  // timing experiments only (ARKS_REGROUP=257): pass A alone, no results
  regroup &= 255;
  const int notail = regroup & 128;
  regroup &= 127;
  // With the length order alone every thread goes on with the document it scanned — no barrier: the warps with the short
  // documents are in pass B while the long ones still scan. Regrouping by structure (2) needs everybody's pass A first.
  uint32_t u = threadIdx.x;
  if (regroup > 1) {
    __syncthreads();
    u = fast_block_order(sm, min(sm.hand[4 * kFastThreads + threadIdx.x] >> 2, 63u), true);  // column
  }
  const uint32_t lane_id = base + sm.slot[u];
  const bool live = lane_id < B.n;
  const uint32_t i = live ? (B.perm ? B.perm[lane_id] : lane_id) : 0;
  const uint8_t* body = B.bodies + (live ? B.body_off[i] : 0);
  const uint32_t len = live ? B.body_len[i] : 0u;
  FastOut o;
  const bool accepted = fast_pass_bc<K_REQ, WALK>(live, body, len, sm, u, o);
  if (!live) return;
  if (!accepted) {
    B.slow_list[atomicAdd(B.slow_n, 1u) + 1u] = i;
    return;
  }
  if (notail) { B.model_off[i] = o.m_start + o.stream3 + o.iu3; return; }  // timing experiments only: no tail
  B.model_off[i] = o.m_rawlen ? o.m_start : 0u;
  B.model_len[i] = o.m_rawlen ? (o.m_rawlen | (o.m_esc ? 0x80000000u : 0u)) : 0u;
  B.bpe[i] = 0;
  const uint8_t pstate = (uint8_t)((o.stream3 == 2 ? PS_STREAM : 0) | (o.so_present && o.iu3 == 2 ? PS_STREAM_OK : 0));
  // with regrouping by structure (2) another thread scanned this document: look the token up from scratch
  const int32_t tok = !o.m_rawlen ? -1 : regroup < 2 ? lookup_token_end(T, B, i, probe) : lookup_token(T, B, i);
  resolve_request(T, B, i, body, tok, pstate, o.m_start, o.m_rawlen, o.m_esc);
}

// ------------------------------------------------------------------------------------------------
// kernel 1' with TWO lanes per document in pass A (mask_scan.cuh "one document, two lanes"): 64 documents per block of 128
// threads, 4 096 warps per 64 Ki-document wave instead of 2 048, and each lane's pass-A chain half as long. Lanes 2k / 2k+1
// share document k of the block; the even lane goes on alone through passes B / C and the tail.
// ------------------------------------------------------------------------------------------------
constexpr int kSplitDocs = kFastThreads / 2;
struct __align__(128) FastSplitSmem {
  FastTables tabs;
  uint64_t bar;
  uint32_t tb[kFastChunks * kSplitDocs];
  uint32_t mem[2 * kFastMaxMembers * kSplitDocs];
  uint32_t ring[16 * kFastThreads];  // per LANE: each half validates its own escapes
  uint32_t hist[64];
  uint32_t order[kSplitDocs];
};
static_assert(sizeof(FastSplitSmem) <= 31 * 1024, "seven blocks per SM: a 64 Ki wave (1 024 blocks) is resident at once");

// which of the block's 64 documents pair `pair` scans: the documents in order of length (counting sort, see fast_block_order)
__device__ __forceinline__ uint32_t split_block_order(FastSplitSmem& sm, uint32_t len0, bool on) {
  const uint32_t t = threadIdx.x, pair = t >> 1;
  if (!on) return pair;
  if (t < 64) sm.hist[t] = 0;
  __syncthreads();
  const uint32_t bucket = min((len0 + 31) >> 5, 63u);
  uint32_t mine = 0;
  if (!(t & 1)) mine = atomicAdd(&sm.hist[bucket], 1u);
  __syncthreads();
  if (!(t & 1)) {
    uint32_t before = 0;
    for (uint32_t k = 0; k < bucket; k++) before += sm.hist[k];
    sm.order[before + mine] = pair;
  }
  __syncthreads();
  return sm.order[pair];
}

// pass A of one lane over chunks [j0, j1) of the document in column `col`; everything it learns goes into `acc` and `c`
__device__ __forceinline__ void split_pass_a(const uint8_t* body, uint32_t len, uint32_t j0, uint32_t j1, FastSplitSmem& sm, uint32_t col,
                                             FastCarry& c, FastHalf& acc) {
  const FastScratch s{sm.tb + col, sm.mem + col, (uint32_t)kSplitDocs, 0u, 0u, 0u, 0u};
  const FastRing ring{sm.ring + threadIdx.x, (uint32_t)kFastThreads};
  const uint32_t nch = (len + 31) >> 5, plen = (len + 15u) & ~15u;
  const uint32_t jload = min(j1 + 1, nch);  // one chunk beyond the range: an escape may reach into it
  const uint4* p = reinterpret_cast<const uint4*>(body);
  const uint4 z = make_uint4(0, 0, 0, 0);
  const bool a32 = (reinterpret_cast<uintptr_t>(body) & 31u) == 0;
  auto ld = [&](uint32_t j, uint4& a, uint4& b) {
    a = z; b = z;
    if (j < jload) {
      if (a32) ld_nc_v8(p + 2 * j, a, b);
      else {
        a = ld_nc_v4(p + 2 * j);
        if (32 * j + 16 < plen) b = ld_nc_v4(p + 2 * j + 1);
      }
    }
  };
  uint4 a0, b0, a1, b1, a2, b2, a3, b3;
  ld(j0, a0, b0); ld(j0 + 1, a1, b1); ld(j0 + 2, a2, b2); ld(j0 + 3, a3, b3);
  {
    const uint32_t w0[8] = {a0.x, a0.y, a0.z, a0.w, b0.x, b0.y, b0.z, b0.w};
    ring.put(j0, w0);
  }
#pragma unroll 1
  for (uint32_t j = j0; j < j1; j++) {
    const uint32_t w[8] = {a0.x, a0.y, a0.z, a0.w, b0.x, b0.y, b0.z, b0.w};
    a0 = a1; b0 = b1; a1 = a2; b1 = b2; a2 = a3; b2 = b3;
    ld(j + 4, a3, b3);
    {
      const uint32_t wn[8] = {a0.x, a0.y, a0.z, a0.w, b0.x, b0.y, b0.z, b0.w};
      ring.put(j + 1, wn);
    }
    const uint32_t nv = min(len - 32 * j, 32u);
    uint32_t bm, tbw;
    fast_chunk(w, nv, ring, len, 32 * j, c, &tbw, &bm);
    s.tb(j) = tbw;
    fast_half_note(acc, j, tbw, bm, nv >= 32 ? 0xffffffffu : ((1u << nv) - 1u));
  }
}

// Pass A of the pair's document by both lanes, the hand-over, and the scratch view the even lane walks. Returns false in the
// odd lane and for documents off this path. All 32 lanes of a warp run this together (shuffles inside).
__device__ __forceinline__ bool split_scan(const uint8_t* body, uint32_t len, FastSplitSmem& sm, uint32_t col, FastScratch& s, uint32_t* nch_out) {
  const bool odd = threadIdx.x & 1;
  const bool elig = len != 0 && len <= kFastMaxLen;
  const uint32_t nch = elig ? (len + 31) >> 5 : 0, h = fast_split_point(nch);
  FastCarry c{0, 0, 0, 0};
  FastHalf acc{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (elig && !odd) {
    split_pass_a(body, len, 0, h, sm, col, c, acc);
  } else if (elig && h < nch) {
    // the escape carry into chunk h is a function of the backslashes at the end of chunk h - 1 alone
    const uint4* p = reinterpret_cast<const uint4*>(body) + 2 * (h - 1);
    const uint4 a = ld_nc_v4(p), b = ld_nc_v4(p + 1);
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    c.esc = fast_esc_after(fast_backslash_mask(w, 32), &c.bad);
    c.bad_flip = c.bad;
    split_pass_a(body, len, h, nch, sm, col, c, acc);
  }
  acc.bad0 = c.bad; acc.bad1 = c.bad_flip; acc.parity = c.in_str;
  // the odd lane's findings to the even lane
  FastHalf H;
  H.bs_lo = __shfl_xor_sync(0xffffffffu, acc.bs_lo, 1); H.bs_hi = __shfl_xor_sync(0xffffffffu, acc.bs_hi, 1);
  H.nz0_lo = __shfl_xor_sync(0xffffffffu, acc.nz0_lo, 1); H.nz0_hi = __shfl_xor_sync(0xffffffffu, acc.nz0_hi, 1);
  H.nz1_lo = __shfl_xor_sync(0xffffffffu, acc.nz1_lo, 1); H.nz1_hi = __shfl_xor_sync(0xffffffffu, acc.nz1_hi, 1);
  H.ntok0 = __shfl_xor_sync(0xffffffffu, acc.ntok0, 1); H.ntok1 = __shfl_xor_sync(0xffffffffu, acc.ntok1, 1);
  H.bad0 = __shfl_xor_sync(0xffffffffu, acc.bad0, 1); H.bad1 = __shfl_xor_sync(0xffffffffu, acc.bad1, 1);
  H.parity = __shfl_xor_sync(0xffffffffu, acc.parity, 1);
  __syncwarp();  // the odd lane's words of the bitmap are in shared memory before the even lane reads them
  if (odd || !elig) return false;
  s = FastScratch{sm.tb + col, sm.mem + col, (uint32_t)kSplitDocs, acc.bs_lo, acc.bs_hi, acc.nz0_lo, acc.nz0_hi};
  uint32_t ntok = acc.ntok0;
  *nch_out = nch;
  return fast_split_merge(s, len, h, c, H, &ntok);
}

template <int WALK>
__global__ void __launch_bounds__(kFastThreads, 7) fast_request_kernel2(DevTables T, ReqDev B, int regroup) {
  extern __shared__ __align__(1024) uint8_t smem[];
  FastSplitSmem& sm = *reinterpret_cast<FastSplitSmem*>(smem);
  stage_fast_tables(&sm.tabs, &sm.bar);
  const uint32_t base = blockIdx.x * kSplitDocs, pair = threadIdx.x >> 1;
  const uint32_t own = base + pair;
  const uint32_t len0 = own < B.n ? B.body_len[B.perm ? B.perm[own] : own] : 0u;
  const uint32_t slot = split_block_order(sm, len0, (regroup & 127) != 0);
  const bool in = base + slot < B.n;
  const uint32_t i = in ? (B.perm ? B.perm[base + slot] : base + slot) : 0;
  const uint8_t* body = B.bodies + (in ? B.body_off[i] : 0);
  const uint32_t len = in ? B.body_len[i] : 0u;
  TokProbe probe{};
  if (in && !(threadIdx.x & 1)) probe = lookup_token_begin(T, B, i);  // consumed after pass C
  FastScratch s{nullptr, nullptr, 0, 0, 0, 0, 0};
  uint32_t nch = 0;
  const bool ok = split_scan(body, len, sm, pair, s, &nch);
  if ((threadIdx.x & 1) || !in) return;
  if (regroup & 256) return;  // timing experiments only: pass A alone
  FastOut o;
  bool accepted = ok;
  if (accepted) {
    const int nmem = fast_walk<WALK>(body, sm.tabs, s, nch, kFastKeyLensReq);
    accepted = nmem >= 0 && fast_members<K_REQ>(body, s, nch, nmem, o);
  }
  if (!accepted) {
    B.slow_list[atomicAdd(B.slow_n, 1u) + 1u] = i;
    return;
  }
  B.model_off[i] = o.m_rawlen ? o.m_start : 0u;
  B.model_len[i] = o.m_rawlen ? (o.m_rawlen | (o.m_esc ? 0x80000000u : 0u)) : 0u;
  B.bpe[i] = 0;
  const uint8_t pstate = (uint8_t)((o.stream3 == 2 ? PS_STREAM : 0) | (o.so_present && o.iu3 == 2 ? PS_STREAM_OK : 0));
  const int32_t tok = !o.m_rawlen ? -1 : lookup_token_end(T, B, i, probe);
  resolve_request(T, B, i, body, tok, pstate, o.m_start, o.m_rawlen, o.m_esc);
}

// ------------------------------------------------------------------------------------------------
// kernel 1'': the latency path (warp_scan.cuh) — micro-batches. One WARP per body: the body arrives in shared memory by one
// 1-D bulk copy (TMA), the 32 lanes scan it together, lane 0 decides it (same tail as the other scan kernels). A body the
// path declines is appended to B.slow_list for scan_*_kernel<.., FROM_LIST>.
// ------------------------------------------------------------------------------------------------
constexpr int kWdWarps = 4;  // warps per block
struct __align__(128) WdWarpSmem {
  uint8_t doc[wd::kFastMaxLen];  // bulk-copy destination
  uint32_t tok[wd::kFastMaxTok + 32];
  uint32_t bmap[wd::kFastMaxLen / 32];
  uint64_t bar;
};
constexpr int kWdSmemPerBlock = kWdWarps * (int)sizeof(WdWarpSmem);

// exclusive prefix of the lanes' stack effects (Hillis-Steele over effect_compose)
__device__ __forceinline__ wd::FastEffect wd_effect_prefix(const wd::FastEffect& own, uint32_t lane, uint32_t* total_bad) {
  wd::FastEffect inc = own;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    wd::FastEffect o;
    o.npop = __shfl_up_sync(0xffffffffu, inc.npop, d);
    o.npush = __shfl_up_sync(0xffffffffu, inc.npush, d);
    o.pword = __shfl_up_sync(0xffffffffu, inc.pword, d);
    o.bad = __shfl_up_sync(0xffffffffu, inc.bad, d);
    o.ptypes = 0;
    if (lane >= (uint32_t)d) inc = wd::effect_compose(o, inc);
  }
  *total_bad = __shfl_sync(0xffffffffu, inc.bad, 31);
  wd::FastEffect pre;
  pre.npop = __shfl_up_sync(0xffffffffu, inc.npop, 1);
  pre.npush = __shfl_up_sync(0xffffffffu, inc.npush, 1);
  pre.pword = __shfl_up_sync(0xffffffffu, inc.pword, 1);
  pre.bad = 0;
  pre.ptypes = 0;
  if (lane == 0) pre.npop = pre.npush = pre.pword = 0;
  return pre;
}

// one document, whole warp; true = accepted, `out` valid on every lane
template <int KIND>
__device__ __forceinline__ bool wd_scan_doc(const uint8_t* doc, uint32_t len, WdWarpSmem& sm, wd::FastOut& out) {
  using namespace wd;
  const uint32_t lane = threadIdx.x & 31;
  uint32_t ntok = 0, carry_esc = 0, carry_str = 0;
  bool bad = false;
  for (uint32_t seg = 0; seg * kFastSeg < len; seg++) {
    const uint32_t base = seg * kFastSeg + 32u * lane;
    FastMasks m;
    {
      const uint4* p = reinterpret_cast<const uint4*>(doc + base);
      uint4 a = make_uint4(0, 0, 0, 0), b = a;
      if (base < len) { a = p[0]; b = p[1]; }
      m.w[0] = a.x; m.w[1] = a.y; m.w[2] = a.z; m.w[3] = a.w;
      m.w[4] = b.x; m.w[5] = b.y; m.w[6] = b.z; m.w[7] = b.w;
    }
    fast_masks(m, base < len ? min(len - base, 32u) : 0u);
    const bool allbs = m.B == 0xffffffffu;  // 32 backslashes in a row: exact engine
    const uint32_t co = odd_tail(m.B);
    uint32_t prev = __shfl_up_sync(0xffffffffu, co, 1);
    if (lane == 0) prev = carry_esc;
    carry_esc = __shfl_sync(0xffffffffu, co, 31);
    const uint32_t E = wd::find_escaped(m.B, prev);
    const uint32_t Qu = m.Q & ~E;
    const uint32_t pm = __ballot_sync(0xffffffffu, __popc(Qu) & 1);
    const uint32_t inside = ((uint32_t)__popc(pm & ((1u << lane) - 1u)) & 1u) ^ carry_str;
    carry_str ^= (uint32_t)__popc(pm) & 1u;
    const uint32_t R = wd::prefix_xor32(Qu) ^ (inside ? 0xffffffffu : 0u);
    sm.bmap[seg * 32 + lane] = m.B;
    const bool ok = !allbs && fast_string_checks(doc, len, base, m, E, R);
    const uint32_t TB = m.V & ~(R & ~Qu);
    const uint32_t cnt = (uint32_t)__popc(TB);
    uint32_t incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= (uint32_t)d) incl += o;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    if (__any_sync(0xffffffffu, !ok) || ntok + total > kFastMaxTok) { bad = true; break; }
    fast_emit(doc, base, TB, Qu, R, sm.tok, ntok + incl - cnt);
    ntok += total;
  }
  __syncwarp();
  if (bad || carry_str || ntok == 0) return false;
  const int c = (int)((ntok + 31) / 32);
  const int k0 = min((int)lane * c, (int)ntok), k1 = min(k0 + c, (int)ntok);
  FastEffect eff{0, 0, 0, 0, 0};
  for (int k = k0; k < k1; k++) effect_token(eff, sm.tok[k]);
  uint32_t total_bad;
  const FastEffect pre = wd_effect_prefix(eff, lane, &total_bad);
  FastFound f;
  f.n_model = f.n_stream = f.n_so = f.n_iu = f.n_usage = f.n_u[0] = f.n_u[1] = f.n_u[2] = f.bad = 0;
  f.o.m_start = f.o.m_rawlen = f.o.m_esc = f.o.stream3 = f.o.so_present = f.o.iu3 = 0;
  f.o.usage[0] = f.o.usage[1] = f.o.usage[2] = 0;
  bool ok = !total_bad;
  if (ok && k0 < k1) ok = pre.npop == 0 && fast_walk_chunk<KIND>(doc, sm.bmap, sm.tok, k0, k1, (int)ntok, pre.npush, pre.pword, eff, f);
  ok = ok && f.n_model <= 1 && f.n_stream <= 1 && f.n_so <= 1 && f.n_iu <= 1 && f.n_usage <= 1 && f.n_u[0] <= 1 && f.n_u[1] <= 1 && f.n_u[2] <= 1;
  if (__any_sync(0xffffffffu, !ok)) return false;
  // every member at most once in the whole document; its finder hands the value to everybody
  const uint32_t bm = __ballot_sync(0xffffffffu, f.n_model), bs = __ballot_sync(0xffffffffu, f.n_stream),
                 bo = __ballot_sync(0xffffffffu, f.n_so), bu = __ballot_sync(0xffffffffu, f.n_usage);
  if (__popc(bm) > 1 || __popc(bs) > 1 || __popc(bo) > 1 || __popc(bu) > 1) return false;
  const int lm = bm ? __ffs(bm) - 1 : 0, ls = bs ? __ffs(bs) - 1 : 0, lo = bo ? __ffs(bo) - 1 : 0, lu = bu ? __ffs(bu) - 1 : 0;
  out.m_start = __shfl_sync(0xffffffffu, f.o.m_start, lm);
  out.m_rawlen = __shfl_sync(0xffffffffu, f.o.m_rawlen, lm);
  out.m_esc = __shfl_sync(0xffffffffu, f.o.m_esc, lm);
  if (KIND == K_REQ) {
    out.stream3 = __shfl_sync(0xffffffffu, f.o.stream3, ls);
    out.so_present = __shfl_sync(0xffffffffu, f.o.so_present, lo);
    out.iu3 = __shfl_sync(0xffffffffu, f.o.iu3, lo);
  } else {
#pragma unroll
    for (int q = 0; q < 3; q++) out.usage[q] = __shfl_sync(0xffffffffu, f.o.usage[q], lu);
  }
  return true;
}
// the body of this warp into its shared-memory window; false: not eligible (empty or longer than the window)
__device__ __forceinline__ bool wd_fetch(WdWarpSmem& sm, const uint8_t* src, uint32_t len) {
  const uint32_t lane = threadIdx.x & 31;
  const bool elig = len > 0 && len <= wd::kFastMaxLen;
  if (lane == 0) {
    mbar_init(&sm.bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (elig) {
      const uint32_t bytes = (len + 15u) & ~15u;
      mbar_expect_tx(&sm.bar, bytes);
      bulk_g2s(sm.doc, src, bytes, &sm.bar);
    }
  }
  __syncwarp();
  if (elig) mbar_wait(&sm.bar, 0);
  return elig;
}

__global__ void __launch_bounds__(kWdWarps * 32) warp_request_kernel(DevTables T, ReqDev B) {
  extern __shared__ __align__(1024) uint8_t smem[];
  WdWarpSmem& sm = reinterpret_cast<WdWarpSmem*>(smem)[threadIdx.x >> 5];
  const uint32_t i = blockIdx.x * kWdWarps + (threadIdx.x >> 5);
  if (i >= B.n) return;
  const uint8_t* body = B.bodies + B.body_off[i];
  const uint32_t len = B.body_len[i];
  // GetQosByToken's chain of dependent loads runs in lane 0 while the body is on its way
  const bool elig = wd_fetch(sm, body, len);
  int32_t tok = -1;
  if ((threadIdx.x & 31) == 0) tok = lookup_token(T, B, i);
  wd::FastOut o;
  const bool ok = elig && wd_scan_doc<K_REQ>(sm.doc, len, sm, o);
  if ((threadIdx.x & 31) != 0) return;
  if (!ok) {
    B.slow_list[atomicAdd(B.slow_n, 1u) + 1u] = i;
    return;
  }
  B.model_off[i] = o.m_rawlen ? o.m_start : 0u;
  B.model_len[i] = o.m_rawlen ? (o.m_rawlen | (o.m_esc ? 0x80000000u : 0u)) : 0u;
  B.bpe[i] = 0;
  const uint8_t pstate = (uint8_t)((o.stream3 == 2 ? PS_STREAM : 0) | (o.so_present && o.iu3 == 2 ? PS_STREAM_OK : 0));
  resolve_request(T, B, i, body, tok, pstate, o.m_start, o.m_rawlen, o.m_esc);
}

// ------------------------------------------------------------------------------------------------
// kernel 2: limit_admit — A6 (checkRateLimit + doRequestRateLimit), A8 (checkTokenQuotaLimit), A12 (pick)
//
// Serial semantics being reproduced (oracle/ork_core.c handle_request): requests are applied in index order;
// a request is denied by the first over-limit entry of qos.RateLimits, then by the first over-limit quota item;
// an admitted request adds 1 to every request-type entry's counter. Within one batch only request-type counters
// of the request's own qos entry change, so for the n_g arrivals of a group the first
//     k = min over request-type entries j of  max(0, floor((limit_j - cur_rule(j) - 1) / cnt_rule(j)) + 1)
// are admitted (k = 0 if any token-type entry or quota item is already over) and every later one is denied by
// the first entry that is over with `k` admissions applied.
// ------------------------------------------------------------------------------------------------
// kernel 2b: one block per hot group sweeps the slot column once, front to back, and hands every member its arrival
// rank (members with a smaller request index). n / 256 coalesced tile loads per hot group.
__global__ void __launch_bounds__(256) rank_hot_groups_kernel(ReqDev B) {
  __shared__ uint32_t warp_tot[8];
  const int n_hot = *B.hot_n + 1;  // the counter starts at -1 (it is part of the group-table memset)
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int h = blockIdx.x; h < n_hot; h += gridDim.x) {
    const int32_t s = B.hot_list[h];
    uint32_t base = 0;
    for (uint32_t t0 = 0; t0 < B.n; t0 += 1024) {  // 4 consecutive entries per thread, 1024 per tile
      const uint32_t j = t0 + threadIdx.x * 4;
      int4 v = make_int4(-1, -1, -1, -1);
      if (j + 3 < B.n) v = *reinterpret_cast<const int4*>(B.gslot + j);
      else {
        if (j < B.n) v.x = B.gslot[j];
        if (j + 1 < B.n) v.y = B.gslot[j + 1];
        if (j + 2 < B.n) v.z = B.gslot[j + 2];
      }
      const uint32_t f0 = v.x == s, f1 = v.y == s, f2 = v.z == s, f3 = v.w == s;
      const uint32_t mine = f0 + f1 + f2 + f3;
      uint32_t incl = mine;  // inclusive scan of the per-thread counts over the warp
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= (uint32_t)d) incl += t;
      }
      if (lane == 31) warp_tot[wid] = incl;
      __syncthreads();
      uint32_t before = 0, total = 0;
#pragma unroll
      for (int w = 0; w < 8; w++) {
        const uint32_t t = warp_tot[w];
        before += (uint32_t)w < wid ? t : 0;
        total += t;
      }
      uint32_t r = base + before + incl - mine;
      if (f0) B.hotrank[j] = (int32_t)r;
      r += f0;
      if (f1) B.hotrank[j + 1] = (int32_t)r;
      r += f1;
      if (f2) B.hotrank[j + 2] = (int32_t)r;
      r += f2;
      if (f3) B.hotrank[j + 3] = (int32_t)r;
      base += total;
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(128) limit_admit_kernel(DevTables T, ReqDev B) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = i < B.n;
  uint8_t reason = live ? B.st_reason[i] : 0, detail = 0;
  const int32_t qos = live ? B.st_qos[i] : -1, slot = live ? B.gslot[i] : -1;
  int32_t pick = -1;
  long long cur_out = 0, lim_out = 0;
  // ---- phase A (per lane): how many arrivals of my group can be admitted
  uint32_t rl0 = 0, rl1 = 0;
  long long n_g = 0, k = 0, cur[4] = {0, 0, 0, 0}, cnt[4] = {0, 0, 0, 0}, q_cur = 0, q_lim = 0;
  int32_t qt = ARKS_QUOTA_NONE;
  int quota_fail = -1;  // first over-limit item
  // Everything a decision may need is fetched in three rounds of independent loads (the kernel is a chain of dependent
  // global round trips, nothing else): round 1 the qos row, round 2 what the row points at, round 3 their contents.
  uint32_t i0 = 0, i1 = 0, b0 = 0, b1 = 0;
  int32_t ep = -1;
  unsigned long long prand = 0;
  if (slot >= 0) {
    rl0 = T.qos_rl_off[qos];
    rl1 = T.qos_rl_off[qos + 1];
    qt = T.qos_quota[qos];
    ep = T.qos_ep[qos];
    prand = B.pick_rand ? B.pick_rand[i] : 0ull;
    n_g = (long long)B.gcnt[slot] + 1;  // counts start at -1 (single memset of the group table)
#pragma unroll
    for (int r = 0; r < 4; r++) cur[r] = B.gsnap[(size_t)slot * 4 + r];  // pre-batch values (claimer's snapshot)
    const uint32_t qs = qt >= 0 ? (uint32_t)qt : 0u, es = ep >= 0 ? (uint32_t)ep : 0u;  // safe rows for the prefetch
    i0 = T.quota_item_off[qs]; i1 = T.quota_item_off[qs + 1];
    b0 = T.ep_backend_off[es]; b1 = T.ep_backend_off[es + 1];
    const long long qu0 = T.quota[(size_t)qs * 3], qu1 = T.quota[(size_t)qs * 3 + 1], qu2 = T.quota[(size_t)qs * 3 + 2];
    for (uint32_t j = rl0; j < rl1; j++) cnt[T.rl_rule[j]]++;
    k = n_g;
    for (uint32_t j = rl0; j < rl1; j++) {
      int rule = T.rl_rule[j];
      long long lim = T.rl_value[j];
      if (rule < 2) {
        long long room = lim - cur[rule] - 1;  // cur + a*cnt + 1 <= lim  <=>  a <= room / cnt
        long long kj = room < 0 ? 0 : room / cnt[rule] + 1;
        k = kj < k ? kj : k;
      } else if (cur[rule] > lim) {
        k = 0;  // "token is not caculated in request": cur + 0 > limit (check.go:124-126)
      }
    }
    if (qt >= 0) {
      for (uint32_t j = i0; j < i1; j++) {
        const int ty = T.qitem_type[j];
        const long long c = ty == 0 ? qu0 : ty == 1 ? qu1 : qu2;
        if (c > T.qitem_value[j]) { quota_fail = (int)(j - i0); q_cur = c; q_lim = T.qitem_value[j]; break; }
      }
    }
    if (qt == ARKS_QUOTA_MISSING || quota_fail >= 0) k = 0;
  }
  // ---- phase B: arrival rank inside the group, only for groups that straddle their limit (0 < k < n_g)
  const bool need_rank = slot >= 0 && k > 0 && k < n_g;
  long long rank = 0;
  if (need_rank && n_g <= kHotGroup) {  // small group: walk its member list
    for (int32_t j = B.ghead[slot]; j >= 0; j = B.gnext[j]) rank += (uint32_t)j < i;
  }
  if (need_rank && n_g > kHotGroup) rank = B.hotrank[i];  // hot tenant: ranked by rank_hot_groups_kernel
  // ---- phase C: decision, commit, pick
  if (slot >= 0) {
    const bool admitted = k >= n_g ? true : k <= 0 ? false : rank < k;
    if (!admitted) {
      // first entry over its limit once k admissions are applied (RateLimitResponse.currentUsage = cur + k*cnt)
      reason = 0;
      for (uint32_t j = rl0; j < rl1 && !reason; j++) {
        int rule = T.rl_rule[j];
        long long lim = T.rl_value[j];
        long long c = rule < 2 ? cur[rule] + k * cnt[rule] : cur[rule];
        long long req = rule < 2 ? 1 : 0;
        if (c + req > lim) {
          reason = ARKS_R_RATE_LIMIT; detail = (uint8_t)(j - rl0); cur_out = c; lim_out = lim;
          if (T.metrics)  // RecordRateLimitHit(ns, user, model, RuleName), check.go:145
            atomicAdd(reinterpret_cast<unsigned long long*>(T.metrics + (size_t)qos * ARKS_METRIC_COLS + ARKS_METRIC_HITS + rule), 1ull);
        }
      }
      if (!reason) {
        if (qt == ARKS_QUOTA_MISSING) reason = ARKS_R_QUOTA_CONFIG;
        else { reason = ARKS_R_QUOTA; detail = (uint8_t)quota_fail; cur_out = q_cur; lim_out = q_lim; }
      }
    }
    // N4 (opt-in): the estimate is charged when the micro-batch commits; nobody reads T.rate here. Metered rows (N5) are
    // charged by meter_charge_kernel instead
    if (admitted && B.precharge && !(B.st_flags[i] & ARKS_FLAG_METERED)) {
      const uint32_t est = B.bpe[i] == kBpeUncounted ? 0u : B.bpe[i];
      if (est && cnt[2]) atomicAdd(reinterpret_cast<unsigned long long*>(T.rate + (size_t)2 * T.n_qos + qos), (unsigned long long)est * (unsigned long long)cnt[2]);
      if (est && cnt[3]) atomicAdd(reinterpret_cast<unsigned long long*>(T.rate + (size_t)3 * T.n_qos + qos), (unsigned long long)est * (unsigned long long)cnt[3]);
    }
    if (admitted && B.pick_rand) {
      // Envoy's weighted choice over the HTTPRoute backendRefs order (arksendpoint_controller.go:283-347)
      unsigned long long sum = 0;
      for (uint32_t b = b0; b < b1; b++) sum += (unsigned long long)max(T.backend_weight[b], 0);
      if (sum) {
        unsigned long long x = prand % sum, acc = 0;
        for (uint32_t b = b0; b < b1; b++) {
          acc += (unsigned long long)max(T.backend_weight[b], 0);
          if (x < acc) { pick = (int32_t)(b - b0); break; }
        }
      }
    }
    // the group's claimer commits the increments (DoLimit INCRBY 1 x admitted); nobody reads T.rate in this kernel
    if (B.st_flags[i] & 0x80) {
      long long adm = k < n_g ? (k < 0 ? 0 : k) : n_g;
      if (adm > 0) {
        if (cnt[0]) T.rate[(size_t)0 * T.n_qos + qos] = cur[0] + adm * cnt[0];
        if (cnt[1]) T.rate[(size_t)1 * T.n_qos + qos] = cur[1] + adm * cnt[1];
      }
    }
  }
  if (!live) return;
  B.reason[i] = reason;
  B.detail[i] = detail;
  B.flags[i] = reason == ARKS_R_OK ? (B.st_flags[i] & 0x7f) : 0;
  B.qos[i] = qos;
  B.token[i] = B.st_tok[i];
  B.pick[i] = pick;
  B.cur_usage[i] = cur_out;
  B.limit_max[i] = lim_out;
}

// ------------------------------------------------------------------------------------------------
// kernel 3: scan_response — A10 (HandleResponseBody) + A11 (doTokenRateLimit / doTokenQuotaLimit)
// ------------------------------------------------------------------------------------------------
// 64-bit add aggregated over the lanes of a warp that target the same address
__device__ __forceinline__ void warp_agg_add(long long* addr, long long v, bool active) {
  unsigned mask = __ballot_sync(0xffffffffu, active);
  if (!active) return;
  unsigned peers = __match_any_sync(mask, (unsigned long long)addr);
  int leader = __ffs(peers) - 1;
  unsigned long long sum = 0;  // counters wrap like the reference's int64 INCRBY: add modulo 2^64
  // reduce over the peer set (peers differ per lane group; iterate set bits)
  for (unsigned p = peers; p; p &= p - 1) {
    int src = __ffs(p) - 1;
    sum += (unsigned long long)__shfl_sync(peers, v, src);
  }
  if ((int)(threadIdx.x & 31) == leader) atomicAdd(reinterpret_cast<unsigned long long*>(addr), sum);
}

// What A11 needs to know about a qos entry: how many of its rate-limit rules are tpm / tpd and how many items of each
// type its quota has. Two levels of dependent global loads, fetched while the first body windows are in flight.
struct QosAcct {
  int32_t qt;        // quota index, ARKS_QUOTA_NONE or ARKS_QUOTA_MISSING
  uint32_t nt[2];    // rules of type tpm, tpd
  uint32_t nq[3];    // quota items of type prompt, response, total
};
__device__ __forceinline__ QosAcct load_qos_acct(const DevTables& T, int32_t qos, bool live) {
  QosAcct a;
  a.qt = ARKS_QUOTA_NONE;
  a.nt[0] = a.nt[1] = 0;
  a.nq[0] = a.nq[1] = a.nq[2] = 0;
  if (!live) return a;
  for (uint32_t j = T.qos_rl_off[qos]; j < T.qos_rl_off[qos + 1]; j++) {
    const int rule = T.rl_rule[j];
    if (rule >= 2) a.nt[rule - 2]++;
  }
  a.qt = T.qos_quota[qos];
  if (a.qt >= 0)
    for (uint32_t j = T.quota_item_off[a.qt]; j < T.quota_item_off[a.qt + 1]; j++) {
      const int ty = T.qitem_type[j];
      a.nq[0] += ty == 0; a.nq[1] += ty == 1; a.nq[2] += ty == 2;
    }
  return a;
}

// A11 for one response per lane (all 32 lanes must call): doTokenRateLimit / doTokenQuotaLimit and the result row.
// bucket of gateway_token_distribution (ExponentialBuckets(1, 2, 17) + Inf): the first upper bound >= v
__device__ __forceinline__ int token_bucket(long long v) {
  if (v <= 1) return 0;
  if (v > 65536) return ARKS_METRIC_HIST_BUCKETS - 1;
  return 64 - __clzll(v - 1);
}

__device__ __forceinline__ void account_usage(const DevTables& T, const RespDev& B, uint32_t i, bool live, int32_t qos, const QosAcct& acct,
                                              uint8_t reason, uint8_t counted, long long u0, long long u1, long long u2) {
  if (live && qos < 0) {  // the row's qos entry does not exist in these tables: nothing to bill (ARKS_R_QOS_GONE)
    reason = ARKS_R_QOS_GONE; counted = 0; u0 = u1 = u2 = 0;
  }
  // N5: a metered stream is billed by meter_charge_kernel; its upstream usage is reported, not billed
  if (live && (B.flags[i] & (ARKS_RESP_STREAM | ARKS_RESP_METERED)) == (ARKS_RESP_STREAM | ARKS_RESP_METERED)) counted = 0;
  if (T.metrics && live && qos >= 0) {  // N3: the series the reference updates per response-body message
    unsigned long long* row = reinterpret_cast<unsigned long long*>(T.metrics + (size_t)qos * ARKS_METRIC_COLS);
    const uint8_t fl = B.flags[i];
    atomicAdd(row + ARKS_METRIC_MESSAGES, 1ull);  // RecordRequest(..., "200"), gateway.go:129
    // RecordTokenUsage: `!hasCompleted && complete && EndOfStream`, handle_response.go:102-104
    if (counted && (fl & ARKS_RESP_END_OF_STREAM) && !(fl & ARKS_RESP_COMPLETED)) {
      atomicAdd(row + ARKS_METRIC_USAGE + 0, (unsigned long long)u0);
      atomicAdd(row + ARKS_METRIC_USAGE + 1, (unsigned long long)u1);
      atomicAdd(row + ARKS_METRIC_HIST_IN + token_bucket(u0), 1ull);
      atomicAdd(row + ARKS_METRIC_HIST_OUT + token_bucket(u1), 1ull);
    }
  }
  // doTokenRateLimit: += total on every token-type entry (check.go:47-59). Warp-aggregated per address.
  const int32_t qt = counted ? acct.qt : ARKS_QUOTA_NONE;
  // N4: the request phase's estimate is reconciled. Modulo 2^64 like every counter: u2 may be INT64_MIN
  const unsigned long long pre = B.precharged && live ? B.precharged[i] : 0u;
#pragma unroll
  for (int r = 0; r < 2; r++)
    warp_agg_add(T.rate + (size_t)(2 + r) * T.n_qos + qos, (long long)(((unsigned long long)u2 - pre) * (unsigned long long)acct.nt[r]),
                 counted && acct.nt[r]);
  // doTokenQuotaLimit: QosToQuotaRequests + IncrUsage (check.go:62-72, qosconfig/types.go:45-72)
  long long add[3] = {0, 0, 0};
  if (counted && qt == ARKS_QUOTA_MISSING) reason = ARKS_R_QUOTA_CONFIG_RESP;
  if (counted && qt >= 0) {
    add[0] = (long long)((unsigned long long)u0 * (unsigned long long)acct.nq[0]);
    add[1] = (long long)((unsigned long long)u1 * (unsigned long long)acct.nq[1]);
    add[2] = (long long)((unsigned long long)u2 * (unsigned long long)acct.nq[2]);
  }
#pragma unroll
  for (int ty = 0; ty < 3; ty++)
    warp_agg_add(T.quota + (size_t)(qt >= 0 ? qt : 0) * 3 + ty, add[ty], counted && qt >= 0 && add[ty] != 0);
  if (T.qdelta) {  // quota shared across GPUs: remember what the other replicas have not seen yet (SURVEY.md §8e)
#pragma unroll
    for (int ty = 0; ty < 3; ty++)
      warp_agg_add(T.qdelta + (size_t)(qt >= 0 ? qt : 0) * 3 + ty, add[ty], counted && qt >= 0 && add[ty] != 0);
  }
  if (live) {
    B.reason[i] = reason;
    B.counted[i] = counted;
    B.usage[3 * (size_t)i + 0] = u0;
    B.usage[3 * (size_t)i + 1] = u1;
    B.usage[3 * (size_t)i + 2] = u2;
  }
}

// complete (non-stream) response bodies: one JSON document per lane.
// FROM_LIST: second stage of the two-stage scan (the bodies in B.slow_list).
template <int SCHED, bool FROM_LIST>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, kMinBlocks) scan_response_kernel(DevTables T, RespDev B) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t n = FROM_LIST ? *B.slow_n + 1u : B.n;  // the counter starts at -1 (it is cleared together with the 0xff tables)
  const uint32_t lane_id = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * B.bpw + (threadIdx.x & 31);
  if (FROM_LIST && ((blockIdx.x * blockDim.x) >> 5) * B.bpw >= n) return;
  const bool live = (threadIdx.x & 31) < B.bpw && lane_id < n;
  const uint32_t i = live ? (FROM_LIST ? B.slow_list[lane_id] : B.perm ? B.perm[lane_id] : lane_id) : 0;  // the body this lane parses
  uint8_t reason = ARKS_R_OK, counted = 0;
  long long u0 = 0, u1 = 0, u2 = 0;
  int32_t qos = 0;
  QosAcct acct;
  {
    const uint8_t* body = B.bodies + (live ? B.body_off[i] : 0);
    const uint8_t fl = live ? B.flags[i] : ARKS_RESP_END_OF_STREAM;
    const bool pending = !(fl & ARKS_RESP_END_OF_STREAM);  // more of the body is still to come: handle_response.go:141-149
    qos = live ? B.qos[i] : 0;
    const uint32_t len = live && !pending && qos >= 0 ? B.body_len[i] : 0;
    uint32_t stack_words[kStackWords];  // local memory, touched only beyond 32 levels of nesting
    __shared__ __align__(16) JsonSmem<true, false> json_smem;
    const JsonTables tabs = json_smem.stage_async();
    WindowPipe<kStages> pipe;
    pipe.start(body, len, smem + (threadIdx.x >> 5) * (kStages * kStageBytes));
    acct = load_qos_acct(T, qos, live && qos >= 0);  // global latency chain, hidden behind the copies issued above
    cp_async_wait<kStages - 1>();        // the table group is the oldest one
    __syncthreads();
    JsonCold cold;  // rarely touched parse state: local memory on purpose (json_engine.cuh)
    JsonT ev;
    ev.init(K_RESP, body, stack_words, &cold, tabs);
    feed_pipe<SCHED>(ev, pipe, 0);
    if (live) {
      if (pending) reason = ARKS_R_PENDING;
      else if (!ev.ok_at_end()) reason = ARKS_R_RESPONSE_UNMARSHAL;   // :157-166
      else if (cold.m_rawlen == 0) reason = ARKS_R_RESPONSE_UNKNOWN;  // :167-181
      else { u0 = cold.usage[0]; u1 = cold.usage[1]; u2 = cold.usage[2]; }
      counted = reason == ARKS_R_OK && u2 != 0;  // :186
    }
  }
  account_usage(T, B, i, live, qos, acct, reason, counted, u0, u1, u2);
}

// the fast path for complete response bodies: first stage of the two-stage scan (see fast_request_kernel)
template <int WALK>
__global__ void __launch_bounds__(kFastThreads) fast_response_kernel(DevTables T, RespDev B, int regroup) {
  extern __shared__ __align__(1024) uint8_t smem[];
  FastBlockSmem& sm = *reinterpret_cast<FastBlockSmem*>(smem);
  stage_fast_tables(&sm.tabs, &sm.bar);
  const uint32_t base = blockIdx.x * blockDim.x;
  {
    const uint32_t own = base + threadIdx.x;
    uint32_t len0 = 0;
    if (own < B.n) {
      const uint32_t i0 = B.perm ? B.perm[own] : own;
      if ((B.flags[i0] & ARKS_RESP_END_OF_STREAM) && B.qos[i0] >= 0) len0 = B.body_len[i0];
    }
    const uint32_t a = fast_block_order(sm, min((len0 + 31) >> 5, 63u), regroup != 0);
    const bool in = base + a < B.n;
    const uint32_t i = in ? (B.perm ? B.perm[base + a] : base + a) : 0;
    const bool scan = in && (B.flags[i] & ARKS_RESP_END_OF_STREAM) && B.qos[i] >= 0;
    fast_pass_a(B.bodies + (scan ? B.body_off[i] : 0), scan ? B.body_len[i] : 0u, sm);
    sm.slot[threadIdx.x] = a;
  }
  if (regroup & 256) return;  // timing experiments only: pass A alone
  regroup &= 255;
  uint32_t u = threadIdx.x;
  if (regroup > 1) {
    __syncthreads();
    u = fast_block_order(sm, min(sm.hand[4 * kFastThreads + threadIdx.x] >> 2, 63u), true);
  }
  const uint32_t lane_id = base + sm.slot[u];
  const bool in = lane_id < B.n;
  const uint32_t i = in ? (B.perm ? B.perm[lane_id] : lane_id) : 0;
  const int32_t qos = in ? B.qos[i] : 0;
  const uint8_t fl = in ? B.flags[i] : ARKS_RESP_END_OF_STREAM;
  const bool pending = !(fl & ARKS_RESP_END_OF_STREAM);
  uint8_t reason = ARKS_R_OK, counted = 0;
  long long u0 = 0, u1 = 0, u2 = 0;
  bool live = in;
  const bool scan2 = in && !pending && qos >= 0;
  FastOut o;
  const bool accepted = fast_pass_bc<K_RESP, WALK>(scan2, B.bodies + (scan2 ? B.body_off[i] : 0), scan2 ? B.body_len[i] : 0u, sm, u, o);
  if (scan2) {
    if (accepted) {
      if (o.m_rawlen == 0) reason = ARKS_R_RESPONSE_UNKNOWN;  // handle_response.go:167-181
      else { u0 = o.usage[0]; u1 = o.usage[1]; u2 = o.usage[2]; }
      counted = reason == ARKS_R_OK && u2 != 0;               // :186
    } else {
      B.slow_list[atomicAdd(B.slow_n, 1u) + 1u] = i;  // the exact engine decides (and accounts) this one
      live = false;
    }
  } else if (in && pending) {
    reason = ARKS_R_PENDING;  // :141-149 (a row without a qos entry: account_usage answers ARKS_R_QOS_GONE)
  }
  const QosAcct acct = load_qos_acct(T, qos, live && qos >= 0);
  account_usage(T, B, i, live, qos, acct, reason, counted, u0, u1, u2);  // all 32 lanes: warp-aggregated atomics inside
}

// two lanes per document in pass A (see fast_request_kernel2)
template <int WALK>
__global__ void __launch_bounds__(kFastThreads, 7) fast_response_kernel2(DevTables T, RespDev B, int regroup) {
  extern __shared__ __align__(1024) uint8_t smem[];
  FastSplitSmem& sm = *reinterpret_cast<FastSplitSmem*>(smem);
  stage_fast_tables(&sm.tabs, &sm.bar);
  const uint32_t base = blockIdx.x * kSplitDocs, pair = threadIdx.x >> 1;
  const uint32_t own = base + pair;
  uint32_t len0 = 0;
  if (own < B.n) {
    const uint32_t i0 = B.perm ? B.perm[own] : own;
    if ((B.flags[i0] & ARKS_RESP_END_OF_STREAM) && B.qos[i0] >= 0) len0 = B.body_len[i0];
  }
  const uint32_t slot = split_block_order(sm, len0, (regroup & 127) != 0);
  const bool odd = threadIdx.x & 1;
  const bool in = base + slot < B.n;
  const uint32_t i = in ? (B.perm ? B.perm[base + slot] : base + slot) : 0;
  const int32_t qos = in ? B.qos[i] : 0;
  const uint8_t fl = in ? B.flags[i] : ARKS_RESP_END_OF_STREAM;
  const bool pending = !(fl & ARKS_RESP_END_OF_STREAM);
  const bool scan = in && !pending && qos >= 0;
  const uint8_t* body = B.bodies + (scan ? B.body_off[i] : 0);
  const uint32_t len = scan ? B.body_len[i] : 0u;
  FastScratch s{nullptr, nullptr, 0, 0, 0, 0, 0};
  uint32_t nch = 0;
  const bool ok = split_scan(body, len, sm, pair, s, &nch);
  if (regroup & 256) return;  // timing experiments only: pass A alone
  uint8_t reason = ARKS_R_OK, counted = 0;
  long long u0 = 0, u1 = 0, u2 = 0;
  bool live = in && !odd;  // the even lane carries the row; the odd one only keeps the warp-wide calls below complete
  if (live && scan) {
    FastOut o;
    bool accepted = ok;
    if (accepted) {
      const int nmem = fast_walk<WALK>(body, sm.tabs, s, nch, kFastKeyLensResp);
      accepted = nmem >= 0 && fast_members<K_RESP>(body, s, nch, nmem, o);
    }
    if (accepted) {
      if (o.m_rawlen == 0) reason = ARKS_R_RESPONSE_UNKNOWN;  // handle_response.go:167-181
      else { u0 = o.usage[0]; u1 = o.usage[1]; u2 = o.usage[2]; }
      counted = reason == ARKS_R_OK && u2 != 0;               // :186
    } else {
      B.slow_list[atomicAdd(B.slow_n, 1u) + 1u] = i;  // the exact engine decides (and accounts) this one
      live = false;
    }
  } else if (live && pending) {
    reason = ARKS_R_PENDING;  // :141-149 (a row without a qos entry: account_usage answers ARKS_R_QOS_GONE)
  }
  const QosAcct acct = load_qos_acct(T, qos, live && qos >= 0);
  account_usage(T, B, i, live, qos, acct, reason, counted, u0, u1, u2);  // all 32 lanes: warp-aggregated atomics inside
}

// the latency path for complete response bodies: one warp per body (see warp_request_kernel)
__global__ void __launch_bounds__(kWdWarps * 32) warp_response_kernel(DevTables T, RespDev B) {
  extern __shared__ __align__(1024) uint8_t smem[];
  WdWarpSmem& sm = reinterpret_cast<WdWarpSmem*>(smem)[threadIdx.x >> 5];
  const uint32_t i = blockIdx.x * kWdWarps + (threadIdx.x >> 5);
  if (i >= B.n) return;
  const uint32_t lane = threadIdx.x & 31;
  const int32_t qos = B.qos[i];
  const bool pending = !(B.flags[i] & ARKS_RESP_END_OF_STREAM);
  uint8_t reason = ARKS_R_OK, counted = 0;
  long long u0 = 0, u1 = 0, u2 = 0;
  bool live = lane == 0;
  const uint32_t len = B.body_len[i];
  const bool scan = !pending && qos >= 0;
  const bool elig = wd_fetch(sm, B.bodies + B.body_off[i], scan ? len : 0u);
  const QosAcct acct = load_qos_acct(T, qos, live && qos >= 0);  // behind the bulk copy
  if (scan) {
    wd::FastOut o;
    if (elig && wd_scan_doc<K_RESP>(sm.doc, len, sm, o)) {
      if (o.m_rawlen == 0) reason = ARKS_R_RESPONSE_UNKNOWN;  // handle_response.go:167-181
      else { u0 = o.usage[0]; u1 = o.usage[1]; u2 = o.usage[2]; }
      counted = reason == ARKS_R_OK && u2 != 0;               // :186
    } else {
      if (lane == 0) B.slow_list[atomicAdd(B.slow_n, 1u) + 1u] = i;  // the exact engine decides (and accounts) this one
      live = false;
    }
  } else if (pending) {
    reason = ARKS_R_PENDING;  // :141-149 (a row without a qos entry: account_usage answers ARKS_R_QOS_GONE)
  }
  account_usage(T, B, i, live, qos, acct, reason, counted, u0, u1, u2);  // lane 0 carries the row
}

// ------------------------------------------------------------------------------------------------
// kernel 3b: scan_sse — SSE chunks (BASELINE config 3). Same verdicts as the sequential machine SseT, different
// work split. A lane that walks a whole chunk sits at an arbitrary phase of the frame structure, so a warp of 32
// chunks runs ~9 lanes wide. Here a warp first cuts its 32 chunks into events (SseSplit, 16 bytes per step, one lane
// per chunk), then parses the events one per lane — every lane starts on the '{' of a frame and frames of one server
// look alike, so the lanes stay together — and finally every chunk's lane folds its events' verdicts in order.
// Irregular chunks (anything SseSplit does not understand) run the sequential SseT machine in their own lane.
// ------------------------------------------------------------------------------------------------
constexpr int kSseStages = ARKS_SSE_STAGES;
constexpr int kSseEvCap = 320;  // events per warp tile (32 chunks); a chunk that does not fit is parsed sequentially
constexpr int kSseSmemPerBlock = kWarpsPerBlock * kSseStages * kStageBytes;

template <int SCHED>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, ARKS_SSE_MINBLK) scan_sse_kernel(DevTables T, RespDev B) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(16) JsonSmem<false, true> json_smem;
  __shared__ uint2 s_desc[kWarpsPerBlock][kSseEvCap];  // x: byte offset of the payload in B.bodies; y: len | owner<<16 | seq<<21
  __shared__ long long s_usage[kWarpsPerBlock][32][3];
  __shared__ uint32_t s_best[kWarpsPerBlock][32], s_fail[kWarpsPerBlock][32], s_n[kWarpsPerBlock];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lane_id = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * B.bpw + lane;
  const bool live = lane < B.bpw && lane_id < B.n;
  const uint32_t i = live ? (B.perm ? B.perm[lane_id] : lane_id) : 0;  // the chunk this lane cuts and accounts
  uint8_t* wsmem = smem + warp * (kSseStages * kStageBytes);
  const JsonTables tabs = json_smem.stage_async();
  const uint32_t chunk_off = live ? B.body_off[i] : 0;
  const int32_t qos = live ? B.qos[i] : 0;
  const uint32_t len = live && qos >= 0 ? B.body_len[i] : 0;
  const uint8_t* body = B.bodies + chunk_off;
  WindowPipe<kSseStages> pipe1;
  pipe1.start(body, len, wsmem);
  const QosAcct acct = load_qos_acct(T, qos, live && qos >= 0);  // global latency chain, hidden behind the copies issued above
  cp_async_wait<kSseStages - 1>();                   // the table group is the oldest one
  __syncthreads();
  uint32_t stack_words[kStackWords];
  JsonCold cold;
  s_best[warp][lane] = 0;
  s_fail[warp][lane] = 0;
  if (lane == 0) s_n[warp] = 0;
  __syncwarp();

  // phase 1: lines -> events
  SseSplit sp;
  sp.init();
  {
    uint32_t seq = 0;
    auto emit = [&](uint32_t off, uint32_t l) {
      const uint32_t slot = atomicAdd(&s_n[warp], 1u);
      if (slot < (uint32_t)kSseEvCap) s_desc[warp][slot] = make_uint2(chunk_off + off, l | lane << 16 | seq << 21);
      else sp.flags |= SseSplit::F_IRREGULAR;
      seq++;
    };
    pipe1.run([&](uint32_t wbeg, uint32_t lim, auto&& load) {
      for (uint32_t ub = wbeg; ub < lim; ub += 16) {
        const Unit16 q = load(ub >> 4);
        sp.unit(ub, lim - ub, q.w[0], q.w[1], q.w[2], q.w[3], emit);
      }
    });
    sp.finish(len);
  }
  __syncwarp();
  const uint32_t n_ev = min(s_n[warp], (uint32_t)kSseEvCap);

  // phase 2: one event per lane
  for (uint32_t r0 = 0; r0 < n_ev; r0 += 32) {
    const uint32_t slot = r0 + lane;
    const bool has = slot < n_ev;
    const uint2 d = has ? s_desc[warp][slot] : make_uint2(0u, 0u);
    const uint32_t owner = (d.y >> 16) & 31u, seq1 = (d.y >> 21) + 1u;
    const uint8_t* base = B.bodies + (d.x & ~15u);
    const uint32_t begin = d.x & 15u, end = has ? begin + (d.y & 0xffffu) : 0u;
    JsonT ev;
    ev.init(K_EVT, base, stack_words, &cold, tabs);
    feed_tiled<kSseStages, SCHED>(ev, base, begin, end, wsmem);
    bool wins = false;
    if (has) {
      const SseEventVerdict v = sse_event_verdict(ev, end);
      if (v.fail) s_fail[warp][owner] = 1;
      else if (v.no_choices) { atomicMax(&s_best[warp][owner], seq1); wins = true; }
    }
    __syncwarp();
    if (wins && s_best[warp][owner] == seq1) {  // the last usage-bearing event of its chunk so far (handle_response.go:119-123)
      s_usage[warp][owner][0] = cold.usage[0];
      s_usage[warp][owner][1] = cold.usage[1];
      s_usage[warp][owner][2] = cold.usage[2];
    }
    __syncwarp();
  }

  // phase 3: the chunk's verdict
  uint8_t reason = ARKS_R_OK, counted = 0;
  long long u0 = 0, u1 = 0, u2 = 0;
  if (live) {
    if (!sp.irregular()) {
      if (s_fail[warp][lane]) reason = ARKS_R_STREAMING;
      else if (s_best[warp][lane]) { u0 = s_usage[warp][lane][0]; u1 = s_usage[warp][lane][1]; u2 = s_usage[warp][lane][2]; }
    } else {
      SseT st;
      st.init(body, stack_words, &cold, tabs);
      uint32_t pos = 0;
      const uint4* units = reinterpret_cast<const uint4*>(body);
      consume_t(st, pos, len, [&](uint32_t u) {
        const uint4 v = ld_nc_v4(units + u);
        Unit16 q;
        q.w[0] = v.x; q.w[1] = v.y; q.w[2] = v.z; q.w[3] = v.w;
        return q;
      });
      if (!st.finish(len)) reason = ARKS_R_STREAMING;
      else { u0 = st.usage[0]; u1 = st.usage[1]; u2 = st.usage[2]; }
    }
    counted = reason == ARKS_R_OK && u2 != 0;  // handle_response.go:186
  }
  __syncwarp();
  account_usage(T, B, i, live, qos, acct, reason, counted, u0, u1, u2);
}

// ------------------------------------------------------------------------------------------------
// BPE token counting (bpe.cuh): a side output of both phases, two kernels behind the scan stage.
// ------------------------------------------------------------------------------------------------
// pass 1: one lane per body. Decoded `content` strings go to `text` (same offsets as the bodies), every pre-token becomes
// a work-list entry: text offset | (length - 1) << 32 | body << 40. Entries are handed out 32 at a time (one atomic per flush).
constexpr int kBpeFlush = 32;
// Rows whose `row_flags` contain every bit of `wide_mask` count the wide key set (N5 metered rows); row_flags may be null.
// kDigits: the pre-tokenizer family (bpe_pretokenize). kRows: lane k scans row rows[k] of the first *rows_n (one vocabulary's
// rows, bpe_split_kernel) instead of row k of n.
template <uint32_t kDigits, bool kRows>
__global__ void __launch_bounds__(128) bpe_scan_kernel(const uint8_t* bodies, const uint32_t* body_off, const uint32_t* body_len, uint32_t n,
                                                       BpeTablesDev T, uint8_t* text, unsigned long long* list, uint32_t* list_n,
                                                       uint32_t list_cap, uint32_t* bpe_out, const uint8_t* row_flags, uint32_t wide_mask,
                                                       const uint32_t* rows, const uint32_t* rows_n) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (kRows ? *rows_n : n)) return;
  const uint32_t i = kRows ? rows[k] : k;
  const uint32_t off = body_off[i];
  const uint32_t keys = row_flags && (row_flags[i] & wide_mask) == wide_mask ? kBpeKeysWide : kBpeKeysContent;
  unsigned long long buf[kBpeFlush];
  uint32_t nb = 0, overflow = 0;
  // The counter may run past the capacity (the merge kernel clamps it). A flush that straddles the end still writes the
  // entries that fit: the merge kernel reads every index below the clamped counter, and a slot this launch left unwritten
  // would hold an entry of an earlier batch or vocabulary slot, counted against the row it names. The row's own entries
  // are skipped there (it is reported uncounted).
  auto flush = [&]() {
    if (!nb) return;
    const uint32_t at = atomicAdd(list_n, nb);
    // (the overflow flag is set apart from the two loops: with it inside the second branch the digits3 instantiations spill)
    if (at + nb > list_cap) overflow = 1;
    if (at + nb <= list_cap)
      for (uint32_t k = 0; k < nb; k++) list[at + k] = buf[k];
    else
      for (uint32_t k = 0; at + k < list_cap; k++) list[at + k] = buf[k];  // at + nb > list_cap: k stays below nb
    nb = 0;
  };
  const BpeScanOut o = bpe_scan_body<kDigits>(bodies + off, body_len[i], text + off, T, keys, [&](uint32_t s, uint32_t len) {
    buf[nb++] = (unsigned long long)(off + s) | (unsigned long long)(len - 1) << 32 | (unsigned long long)i << 40;
    if (nb == kBpeFlush) flush();
  });
  flush();
  bpe_out[i] = (o.bad || overflow) ? kBpeUncounted : 0u;
}
// pass 2: one lane per pre-token (grid-stride over the work list). The hot merges come from shared memory, staged by one
// bulk copy (TMA) per block; the rest of the merge table is read through L2. kIgnoreMerges: the vocabulary's whole-piece
// lookup comes first (bpe_piece_tokens).
constexpr int kBpeMergeThreads = 256;
template <bool kIgnoreMerges>
__global__ void __launch_bounds__(kBpeMergeThreads) bpe_merge_kernel(const unsigned long long* list, const uint32_t* list_n, uint32_t list_cap,
                                                                    BpeTablesDev T, const uint8_t* text, uint32_t* bpe_out) {
  __shared__ __align__(128) BpeSlot hot[kBpeHotSlots];
  __shared__ uint64_t bar;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(&bar, (uint32_t)sizeof(hot));
    bulk_g2s(hot, T.hot, (uint32_t)sizeof(hot), &bar);
  }
  __syncthreads();
  mbar_wait(&bar, 0);
  const uint32_t total = min(*list_n, list_cap);
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
    const unsigned long long e = list[k];
    const uint32_t off = (uint32_t)e, len = ((uint32_t)(e >> 32) & 0xffu) + 1u, body = (uint32_t)(e >> 40);
    if (bpe_out[body] == kBpeUncounted) continue;  // written by pass 1, never by this kernel
    const uint32_t ntok = bpe_piece_tokens<kIgnoreMerges>(text + off, len, hot, T);
    atomicAdd(&bpe_out[body], ntok);
  }
}

// Several vocabularies (arks_bind_model_vocab): every row goes to the list of its qos entry's vocabulary slot (rows without
// an entry, qos < 0, and rows whose slot is not loaded to slot 0). rows: kBpeMaxVocabs lists of `stride` entries, rows_n:
// their lengths (zeroed before). One atomic per distinct slot per warp.
__global__ void __launch_bounds__(128) bpe_split_kernel(const uint8_t* qos_vocab, const int32_t* qos_of, uint32_t n, uint32_t loaded,
                                                        uint32_t* rows, uint32_t stride, uint32_t* rows_n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t q = qos_of[i];
  uint32_t v = q >= 0 ? qos_vocab[q] : 0u;
  if (v >= kBpeMaxVocabs || !((loaded >> v) & 1u)) v = 0;
  const uint32_t lane = threadIdx.x & 31u;
  const unsigned peers = __match_any_sync(__activemask(), v);
  const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
  uint32_t at = 0;
  if (lane == leader) at = atomicAdd(&rows_n[v], (uint32_t)__popc(peers));
  at = __shfl_sync(peers, at, leader) + (uint32_t)__popc(peers & ((1u << lane) - 1u));
  rows[(size_t)v * stride + at] = i;
}

// N5 (arks_set_stream_metering): bills the metered rows of a batch, one lane per row, after the BPE kernels. A row is metered
// when it was answered ARKS_R_OK and its flags contain every bit of `mask`; it is billed its BPE count, or its body length
// when there is no count (bpe null: no vocabulary; or ARKS_BPE_UNCOUNTED). qos: the current generation's index (response
// rows were re-mapped at staging; -1 bills nothing). `side` 0: prompts (quota item prompt, gateway_token_usage{input}),
// 1: completion chunks (quota item response, gateway_token_usage{output}); tpm / tpd and quota item total on both.
__global__ void __launch_bounds__(128) meter_charge_kernel(DevTables T, uint32_t n, const uint8_t* reason, const uint8_t* flags, uint32_t mask,
                                                           const int32_t* qos_of, const uint32_t* bpe, const uint32_t* body_len, int side) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool on = i < n && reason[i] == ARKS_R_OK && (flags[i] & mask) == mask;
  const int32_t qos = on ? qos_of[i] : -1;
  on = on && qos >= 0;
  long long c = 0;
  if (on) {
    const uint32_t b = bpe ? bpe[i] : kBpeUncounted;
    c = b == kBpeUncounted ? (long long)body_len[i] : (long long)b;
  }
  on = on && c != 0;
  const QosAcct a = load_qos_acct(T, qos, on);
  const uint32_t row = on ? (uint32_t)qos : 0u;
#pragma unroll
  for (int r = 0; r < 2; r++) warp_agg_add(T.rate + (size_t)(2 + r) * T.n_qos + row, c * (long long)a.nt[r], on && a.nt[r]);
  const bool q_on = on && a.qt >= 0;
  const size_t qrow = (size_t)(q_on ? a.qt : 0) * 3;
  const long long add_side = c * (long long)a.nq[side], add_total = c * (long long)a.nq[2];
  warp_agg_add(T.quota + qrow + side, add_side, q_on && add_side != 0);
  warp_agg_add(T.quota + qrow + 2, add_total, q_on && add_total != 0);
  if (T.qdelta) {  // quota shared across GPUs, as in account_usage
    warp_agg_add(T.qdelta + qrow + side, add_side, q_on && add_side != 0);
    warp_agg_add(T.qdelta + qrow + 2, add_total, q_on && add_total != 0);
  }
  if (T.metrics) warp_agg_add(T.metrics + (size_t)row * ARKS_METRIC_COLS + ARKS_METRIC_USAGE + side, c, on);
}

// syncQuotaUsage (arks_impl.go:226-296): one lane per ArksQuota, in place on the device copies of the CR status
__global__ void sync_quota_kernel(const uint32_t* item_off, const uint8_t* item_type, long long* quota, uint32_t n_quotas, int restore,
                                  uint32_t* present, long long* used, uint8_t* action) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_quotas) return;
  uint32_t pres = present[q];
  long long u[3] = {used[3 * (size_t)q], used[3 * (size_t)q + 1], used[3 * (size_t)q + 2]};
  long long* cur = quota + 3 * (size_t)q;
  int update_cr = 0, update_quota = 0;
  for (uint32_t j = item_off[q]; j < item_off[q + 1]; j++) {
    const int ty = item_type[j];
    if (pres & (1u << ty)) {
      if (u[ty] < cur[ty]) { update_cr = 1; u[ty] = cur[ty]; }
      else if (u[ty] > cur[ty]) update_quota = 1;
    } else {
      update_cr = 1; pres |= 1u << ty; u[ty] = cur[ty];
    }
  }
  if (update_quota)
    for (uint32_t j = item_off[q]; j < item_off[q + 1]; j++) {
      const int ty = item_type[j];
      if (!restore) cur[ty] = 0;  // SetUsage(QosToQuotaRequests(conf, nil)): Request == 0
      else if (u[ty] > cur[ty]) cur[ty] = u[ty];
    }
  present[q] = pres;
  used[3 * (size_t)q] = u[0]; used[3 * (size_t)q + 1] = u[1]; used[3 * (size_t)q + 2] = u[2];
  action[q] = (uint8_t)(update_cr | update_quota << 1);
}

// quota[i] += reduced[i] - exported[i]; delta[i] -= exported[i] — applies what the OTHER GPUs added up to their export;
// increments this GPU made after ITS export stay in the delta vector for the next epoch
__global__ void fold_quota_delta_kernel(long long* quota, long long* delta, const long long* reduced, const long long* exported, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    quota[i] += reduced[i] - exported[i];
    delta[i] -= exported[i];
  }
}
// the same with only the shared rows on the wire: gather them into the message ...
__global__ void gather_shared_kernel(long long* msg, const long long* exported, const uint32_t* idx, uint32_t n_shared) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n_shared * 3u) msg[k] = exported[(size_t)idx[k / 3] * 3 + k % 3];
}
// ... and after the all-reduce: quota[shared] += reduced - exported; every row's delta gives up what was exported
__global__ void fold_shared_kernel(long long* quota, long long* delta, const long long* msg, const long long* exported, const uint32_t* idx,
                                   uint32_t n_shared, size_t n_all) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n_all) delta[k] -= exported[k];
  if (k < (size_t)n_shared * 3u) {
    const size_t q = (size_t)idx[k / 3] * 3 + k % 3;
    quota[q] += msg[k] - exported[q];
  }
}
__global__ void add_quota_kernel(long long* quota, const long long* add, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) quota[i] += add[i];
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct HostTables {  // what we need to remember for reloads, snapshots and validation
  std::vector<std::string> qos_key;    // namespace \0 user \0 model
  std::vector<std::string> quota_key;  // namespace \0 name
  std::vector<uint32_t> ep_backend_off;
  uint32_t n_tokens = 0, n_qos = 0, n_quotas = 0, n_endpoints = 0, n_backends = 0;
};

// from this size on requests / complete response bodies go through the two-stage scan (mask_scan.cuh first); below it the
// exact kernel alone is one launch and spreads the few bodies over more warps (bodies_per_warp). ARKS_FAST_MIN overrides.
constexpr uint32_t kFastMinBatchDefault = 4096;
// up to this size a batch takes the latency path (warp_scan.cuh: a warp per body): the GPU is mostly idle and what the
// streams wait for is the time ONE body takes. ARKS_WARP_MAX overrides (0: off).
constexpr uint32_t kWarpMaxBatchDefault = 2048;

struct arks_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;  // kernels, counter memsets, result D2H: the order of this stream IS the linearisation
  cudaStream_t h2d = nullptr;     // batch uploads (overlap the kernels of earlier batches)
  cudaStream_t cfg_stream = nullptr;  // config plane: the next generation's tables are uploaded here, off the data path
  std::mutex cfg_mu;                  // prepare (config thread) vs commit (batch thread)
  bool precharge = false;              // N4 (arks_set_precharge)
  bool meter = false;                  // N5 (arks_set_stream_metering)
  bool split = false;                  // fast path: two lanes per document in pass A (fast_*_kernel2), ARKS_SPLIT=1; measured slower
  bool walk8 = true;                   // fast path, pass B: the step inlined eight times (true) or one copy in a loop
  int regroup = 1;                     // fast path: regroup a block's documents by structure between passes A and B
  struct NcclApi* nccl = nullptr;      // dlopen()ed libnccl + this context's communicator (arks_comm_init)
  arks::ConfigStore* store = nullptr;  // objects behind arks_upsert_* / arks_delete_*
  int32_t *d_qos_from = nullptr, *d_quota_from = nullptr;  // row maps of the current generation (kept alive for the carry kernels)
  char err[512] = {0};
  uint32_t max_batch = 0;
  uint64_t max_bytes = 0;
  uint64_t launches = 0;
  bool loaded = false;
  HostTables ht;
  std::vector<void*> table_allocs;
  DevTables dt{};
  long long* d_rate = nullptr;
  long long* d_metrics = nullptr;  // [n_qos][ARKS_METRIC_COLS] when metrics are enabled
  bool metrics_on = false;
  long long* d_quota = nullptr;
  long long* d_qdelta = nullptr;   // allocated when quota sharing is enabled
  long long* d_qtmp = nullptr;
  long long* d_qexp = nullptr;     // what the last arks_export_quota_delta_dev handed out
  bool qexp_valid = false;
  bool share_quota = false;
  // BPE side output (arks_load_bpe): tables + per-batch scratch
  bool bpe_on = false;                      // slot 0 (the default vocabulary) is loaded
  BpeTablesDev bpe[kBpeMaxVocabs]{};        // per vocabulary slot (arks_load_bpe_vocab); slot 0: arks_load_bpe
  std::vector<void*> bpe_allocs[kBpeMaxVocabs];
  uint8_t* d_bpe_cls = nullptr;             // the Unicode class table every slot reads (uploaded with slot 0)
  uint32_t vocab_loaded = 0;                // bit s: slot s holds a vocabulary (bit 0 == bpe_on); written under cfg_mu
  uint32_t vocab_used = 0;                  // slots other than 0 the current generation's qos entries use (under cfg_mu)
  bool vocab_multi = false;                 // vocab_used != 0: queue_bpe splits the rows by vocabulary
  std::unordered_map<std::string, uint32_t> vocab_bind;  // model name -> slot (arks_bind_model_vocab), under cfg_mu
  uint32_t* d_bpe_rows = nullptr;           // kBpeMaxVocabs row lists of max_batch entries (bpe_split_kernel)
  uint8_t* d_bpe_text = nullptr;            // decoded `content` strings, laid out like the bodies
  unsigned long long* d_bpe_list = nullptr; // work list of pre-tokens
  uint32_t* d_bpe_n = nullptr;
  uint32_t bpe_list_cap = 0;
  uint32_t generation = 0;                  // bumped by every successful arks_load_tables
  std::deque<std::vector<int32_t>> remap;   // remap[k]: qos index of generation (generation - remap.size() + k) -> the next one, or -1
  int32_t* d_backend_weight = nullptr;
  int64_t last_win[4];
  // batch buffers: kSlots independent staging slots so several batches can be resident in HBM at once
  struct Slot {
    uint8_t* d_req_bodies = nullptr;   // max_bytes
    uint8_t* d_req_meta = nullptr;     // offsets/lens/token_off/pick_rand/tokens packed
    uint8_t* d_resp_bodies = nullptr;
    uint8_t* d_resp_meta = nullptr;    // offsets/lens/qos/flags packed
    uint8_t* h_req_meta = nullptr;     // pinned staging for the meta blocks
    uint8_t* h_resp_meta = nullptr;
    cudaEvent_t req_copied = nullptr, resp_copied = nullptr;
    uint8_t* h_req_result = nullptr;   // pinned, per slot: asynchronous submits keep several batches in flight
    uint8_t* h_resp_result = nullptr;
    cudaEvent_t req_done = nullptr, resp_done = nullptr;
    cudaEvent_t req_ran = nullptr, resp_ran = nullptr;  // the slot's device buffers are free again (kernels done)
    uint32_t req_fetch_n = 0, resp_fetch_n = 0;
    ReqDev rq{};
    RespDev rp{};
    uint32_t req_n = 0, resp_n = 0;
    int resp_mode = 0;  // 1 all JSON documents, 2 all SSE chunks, 0 mixed
    bool resp_metered = false;  // the staged response batch has a metered chunk (N5): the meter kernel runs after the BPE kernels
    uint32_t resp_n_sse = 0;
    const uint32_t* d_resp_kind = nullptr;  // mixed batch: row indices, complete bodies first then SSE chunks
    bool req_staged = false, resp_staged = false;
    bool req_zc = false, resp_zc = false;  // this batch's result rows are written into the pinned host block by the kernels
  };
  static constexpr int kSlots = 4;
  Slot slots[kSlots];
  int cur = 0;
  size_t meta_cap = 0;
  uint32_t fetch_n = 0;          // batch size of the last run_* call (what fetch_* copies back)
  // optional per-kernel timing (bench roofline): events around each launch of the last run_* call
  bool prof = false;
  int sched[3] = {8, 8, 1};  // parse schedule of the request scan, the JSON response scan, the SSE event phase: 0 consume_t,
                             // 1 consume_evsync, 8 consume_rounds<8> (json_engine.cuh). ARKS_SCHED="r,p,s" overrides (A/B runs)
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  int ev_n = 0;
  cudaEvent_t ev_fast[2] = {nullptr, nullptr};  // around the fast-path kernel alone (roofline of the dominant kernel)
  bool ev_fast_set = false;
  cudaEvent_t ev_bpe[2] = {nullptr, nullptr};   // around the two BPE kernels
  bool ev_bpe_set = false;
  cudaEvent_t ev_admit0 = nullptr;              // start of rank_hot + limit_admit (after the BPE kernels)
  cudaEvent_t ev_meter[2] = {nullptr, nullptr}; // around meter_charge_kernel (N5)
  bool ev_meter_set = false;
  bool is_req_timing = false;
  bool last_two_stage = false;
  int last_route = -1;           // staging route of the last stage_* call (arks_last_staging_route)
  const uint32_t* last_slow_n = nullptr;
  uint8_t* d_inter = nullptr;    // intermediates + group table
  uint32_t* d_perm = nullptr;    // lane -> body permutation of the batch being scanned (length order)
  uint32_t* d_lenhist = nullptr; // kLenBuckets counters / offsets
  bool sort_lanes = true;        // ARKS_SORT=0 scans in arrival order (A/B runs)
  bool sort_fast = false;        // ARKS_SORT=2: global length order in front of the fast path too (A/B runs)
  bool fast_scan = true;         // ARKS_FAST=0: large batches also take the fused lane-per-document kernels (A/B runs)
  uint32_t fast_min = kFastMinBatchDefault;  // ARKS_FAST_MIN=n: batches of n rows and more take the two-stage scan
  uint32_t warp_max = kWarpMaxBatchDefault;  // ARKS_WARP_MAX=n: batches of up to n rows take the warp-per-document latency path
  int n_sm = 132;
  uint32_t* d_slow = nullptr;    // [0] counter, [64..] the rows left to the exact engine by the fast path (mask_scan.cuh)
  uint8_t* d_result = nullptr;   // packed results
  size_t result_cap = 0;
  uint32_t gsize = 0;
};

static int fail(arks_ctx* c, int code, const char* fmt, ...) {
  if (c) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(c->err, sizeof c->err, fmt, ap);
    va_end(ap);
  }
  return code;
}
#define CK(call)                                                                                      \
  do {                                                                                                \
    cudaError_t e_ = (call);                                                                          \
    if (e_ != cudaSuccess) return fail(ctx, ARKS_E_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

static const int64_t kRuleWindow[4] = {60, 86400, 60, 86400};  // ratelimiter/rate_limiter.go:31-68
static int64_t window_start(int64_t now, int rule) {            // ratelimiter/cache_key.go:73-80
  int64_t w = kRuleWindow[rule];
  int64_t r = (now + 62135596800LL) % w;
  if (r < 0) r += w;
  return now - r;
}

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

extern "C" {

int arks_abi_version(void) { return ARKS_ABI_VERSION; }

const char* arks_last_error(const arks_ctx* ctx) { return ctx ? ctx->err : "null context"; }

size_t arks_extract_bearer(const uint8_t* const* keys, const size_t* key_lens, const uint8_t* const* values,
                           const size_t* value_lens, size_t n_headers, const uint8_t** token) {
  // handle_request.go:38-46 — strings.ToLower(key) == "authorization" && HasPrefix(value, "Bearer ")
  static const char A[] = "authorization";
  *token = nullptr;
  for (size_t i = 0; i < n_headers; i++) {
    if (key_lens[i] != 13) continue;
    bool ok = true;
    for (int k = 0; k < 13; k++) {
      uint8_t c = keys[i][k];
      if (c >= 'A' && c <= 'Z') c += 32;
      ok &= c == (uint8_t)A[k];
    }
    if (!ok) continue;
    if (value_lens[i] >= 7 && memcmp(values[i], "Bearer ", 7) == 0) {
      *token = values[i] + 7;
      return value_lens[i] - 7;
    }
  }
  return 0;
}

int arks_create(int device, uint32_t max_batch, uint64_t max_batch_bytes, arks_ctx** out) {
  if (!out || max_batch == 0) return ARKS_E_INVALID_ARG;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device >= ndev) return ARKS_E_NO_DEVICE;
  arks_ctx* ctx = new arks_ctx();
  ctx->device = device;
  if (const char* e = getenv("ARKS_SORT")) { ctx->sort_lanes = e[0] != '0'; ctx->sort_fast = e[0] == '2'; }
  if (const char* e = getenv("ARKS_SCHED")) {
    int a = 8, b = 8, c = 8;
    if (sscanf(e, "%d,%d,%d", &a, &b, &c) == 3) {
      auto ok = [](int v) { return v == 0 || v == 1 || v == 8; };
      if (ok(a) && ok(b) && ok(c)) { ctx->sched[0] = a; ctx->sched[1] = b; ctx->sched[2] = c; }
    }
  }
  ctx->max_batch = max_batch;
  ctx->max_bytes = align_up(max_batch_bytes + 16, 256);
  for (int r = 0; r < 4; r++) ctx->last_win[r] = INT64_MIN;
  *out = ctx;
  CK(cudaSetDevice(device));
  CK(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&ctx->h2d, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&ctx->cfg_stream, cudaStreamNonBlocking));
  size_t n = max_batch;
  // meta: body_off, body_len, token_off(n+1), pick_rand, qos, flags + token bytes (256 B per request budget)
  ctx->meta_cap = align_up(n * 4, 256) * 4 + align_up(n * 8, 256) + align_up(n, 256) + align_up(n * 256, 256) + kSmallBatchBytes + 256;
  for (int k = 0; k < 4; k++) CK(cudaEventCreate(&ctx->ev[k]));
  for (int k = 0; k < 2; k++) CK(cudaEventCreate(&ctx->ev_fast[k]));
  for (int k = 0; k < 2; k++) CK(cudaEventCreate(&ctx->ev_bpe[k]));
  for (int k = 0; k < 2; k++) CK(cudaEventCreate(&ctx->ev_meter[k]));
  CK(cudaEventCreate(&ctx->ev_admit0));
#define ARKS_FOR_SCHED(X) X(0) X(1) X(8)
#define ARKS_SET(S)                                                                                                        \
  CK(cudaFuncSetAttribute(scan_request_kernel<S, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemPerBlock));     \
  CK(cudaFuncSetAttribute(scan_request_kernel<S, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemPerBlock));      \
  CK(cudaFuncSetAttribute(scan_response_kernel<S, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemPerBlock));    \
  CK(cudaFuncSetAttribute(scan_response_kernel<S, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemPerBlock));     \
  CK(cudaFuncSetAttribute(scan_sse_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSseSmemPerBlock));
  ARKS_FOR_SCHED(ARKS_SET)
#undef ARKS_SET
  CK(cudaFuncSetAttribute(warp_request_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWdSmemPerBlock));
  CK(cudaFuncSetAttribute(warp_response_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWdSmemPerBlock));
  if (const char* e = getenv("ARKS_WARP_MAX")) ctx->warp_max = (uint32_t)strtoul(e, nullptr, 10);
  CK(cudaFuncSetAttribute(fast_request_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastBlockSmem)));
  CK(cudaFuncSetAttribute(fast_response_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastBlockSmem)));
  CK(cudaFuncSetAttribute(fast_request_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastBlockSmem)));
  CK(cudaFuncSetAttribute(fast_response_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastBlockSmem)));
  CK(cudaFuncSetAttribute(fast_request_kernel2<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastSplitSmem)));
  CK(cudaFuncSetAttribute(fast_response_kernel2<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastSplitSmem)));
  if (const char* e = getenv("ARKS_SPLIT")) ctx->split = e[0] != '0';
  // a 64 Ki-document wave is 512 blocks: with four of them resident per SM (4 x ~50 KB) the whole wave runs at once
  static_assert(sizeof(FastBlockSmem) <= 56 * 1024, "four fast-path blocks per SM");
  {
    const char* cv = getenv("ARKS_CARVEOUT");  // percent of the SM's L1/shared array given to shared memory; default: the driver's choice
    if (cv && *cv) {
      CK(cudaFuncSetAttribute(fast_request_kernel<0>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(cv)));
      CK(cudaFuncSetAttribute(fast_response_kernel<0>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(cv)));
      CK(cudaFuncSetAttribute(fast_request_kernel<8>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(cv)));
      CK(cudaFuncSetAttribute(fast_response_kernel<8>, cudaFuncAttributePreferredSharedMemoryCarveout, atoi(cv)));
    }
    const char* wk = getenv("ARKS_WALK");
    ctx->walk8 = wk && *wk ? atoi(wk) == 8 : true;
    const char* rg = getenv("ARKS_REGROUP");
    ctx->regroup = rg && *rg ? atoi(rg) : 1;
  }
  if (const char* e = getenv("ARKS_FAST")) ctx->fast_scan = e[0] != '0';
  if (const char* e = getenv("ARKS_FAST_MIN")) ctx->fast_min = (uint32_t)strtoul(e, nullptr, 10);
  {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    ctx->n_sm = prop.multiProcessorCount;
  }
  uint32_t g = 64;
  while (g < 2 * n) g <<= 1;
  ctx->gsize = g;
  size_t inter = align_up(n, 256) * 2 + align_up(n * 4, 256) * 5 + align_up((size_t)g * 4, 256) * 3 + (size_t)g * 32 + 2048 +
                 align_up((n / kHotGroup + 2) * 4, 256);
  CK(cudaMalloc(&ctx->d_inter, inter));
  CK(cudaMalloc(&ctx->d_perm, (size_t)4 * max_batch + 256));
  CK(cudaMalloc(&ctx->d_slow, (size_t)4 * max_batch + 256));

  CK(cudaMalloc(&ctx->d_lenhist, (size_t)4 * kLenBuckets));
  ctx->result_cap = align_up(n, 256) * 3 + align_up(n * 4, 256) * 6 + align_up(n * 8, 256) * 3;
  CK(cudaMalloc(&ctx->d_result, ctx->result_cap));
  CK(cudaMemset(ctx->d_result, 0, ctx->result_cap));  // the packed block has alignment gaps that the D2H copies too
  return 0;
}

static void free_tables(arks_ctx* ctx) {
  for (void* p : ctx->table_allocs) cudaFree(p);
  ctx->table_allocs.clear();
}

static void free_store(arks::ConfigStore* s);
void arks_destroy(arks_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  free_store(ctx->store);
  arks_comm_destroy(ctx);
  if (ctx->h2d) cudaStreamSynchronize(ctx->h2d);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  free_tables(ctx);  // one arena per generation: tables, counters and row maps are interior pointers
  for (auto& sl : ctx->slots) {
    cudaFree(sl.d_req_bodies);
    cudaFree(sl.d_req_meta);
    cudaFree(sl.d_resp_bodies);
    cudaFree(sl.d_resp_meta);
    cudaFreeHost(sl.h_req_meta);
    cudaFreeHost(sl.h_resp_meta);
    cudaFreeHost(sl.h_req_result);
    cudaFreeHost(sl.h_resp_result);
    if (sl.req_done) cudaEventDestroy(sl.req_done);
    if (sl.req_ran) cudaEventDestroy(sl.req_ran);
    if (sl.resp_ran) cudaEventDestroy(sl.resp_ran);
    if (sl.resp_done) cudaEventDestroy(sl.resp_done);
    if (sl.req_copied) cudaEventDestroy(sl.req_copied);
    if (sl.resp_copied) cudaEventDestroy(sl.resp_copied);
  }
  for (int k = 0; k < 4; k++)
    if (ctx->ev[k]) cudaEventDestroy(ctx->ev[k]);
  for (int k = 0; k < 2; k++) {
    if (ctx->ev_fast[k]) cudaEventDestroy(ctx->ev_fast[k]);
    if (ctx->ev_bpe[k]) cudaEventDestroy(ctx->ev_bpe[k]);
    if (ctx->ev_meter[k]) cudaEventDestroy(ctx->ev_meter[k]);
  }
  if (ctx->ev_admit0) cudaEventDestroy(ctx->ev_admit0);
  cudaFree(ctx->d_inter);
  cudaFree(ctx->d_perm);
  cudaFree(ctx->d_slow);
  for (auto& v : ctx->bpe_allocs)
    for (void* p : v) cudaFree(p);
  cudaFree(ctx->d_bpe_cls);
  cudaFree(ctx->d_bpe_rows);
  cudaFree(ctx->d_bpe_text);
  cudaFree(ctx->d_bpe_list);
  cudaFree(ctx->d_bpe_n);

  cudaFree(ctx->d_lenhist);
  cudaFree(ctx->d_result);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->h2d) cudaStreamDestroy(ctx->h2d);
  if (ctx->cfg_stream) cudaStreamDestroy(ctx->cfg_stream);
  delete ctx;
}

void* arks_stream(arks_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
// how many rows of the last batch that took the two-stage scan were left to the exact engine; -1 if the last run_* call
// used the fused kernels. Synchronises the stream: for tests and the bench, not for the data path.
int64_t arks_last_declined(arks_ctx* ctx) {
  if (!ctx || !ctx->last_two_stage) return -1;
  if (cudaSetDevice(ctx->device) != cudaSuccess || cudaStreamSynchronize(ctx->stream) != cudaSuccess) return -1;
  uint32_t v = 0;
  if (!ctx->last_slow_n || cudaMemcpy(&v, ctx->last_slow_n, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return (int64_t)(v + 1u);  // the counter starts at -1
}
uint64_t arks_launch_count(const arks_ctx* ctx) { return ctx ? ctx->launches : 0; }
int arks_last_staging_route(const arks_ctx* ctx) { return ctx ? ctx->last_route : -1; }

int arks_sync_quota_usage(arks_ctx* ctx, int mode, uint32_t* status_present, int64_t* status_used, uint8_t* action) {
  if (!ctx || !ctx->loaded) return ARKS_E_NOT_LOADED;
  if (!status_present || !status_used || !action || (mode != ARKS_SYNC_REFERENCE && mode != ARKS_SYNC_RESTORE)) return ARKS_E_INVALID_ARG;
  const uint32_t n = ctx->ht.n_quotas;
  if (n == 0) return 0;
  CK(cudaSetDevice(ctx->device));
  uint32_t* d_pres = nullptr;
  long long* d_used = nullptr;
  uint8_t* d_act = nullptr;
  CK(cudaMalloc(&d_pres, (size_t)4 * n));
  CK(cudaMalloc(&d_used, (size_t)24 * n));
  CK(cudaMalloc(&d_act, n));
  CK(cudaMemcpyAsync(d_pres, status_present, (size_t)4 * n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(d_used, status_used, (size_t)24 * n, cudaMemcpyHostToDevice, ctx->stream));
  sync_quota_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(ctx->dt.quota_item_off, ctx->dt.qitem_type, ctx->d_quota, n,
                                                            mode == ARKS_SYNC_RESTORE, d_pres, d_used, d_act);
  CK(cudaMemcpyAsync(status_present, d_pres, (size_t)4 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(status_used, d_used, (size_t)24 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(action, d_act, n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  cudaFree(d_pres); cudaFree(d_used); cudaFree(d_act);
  ctx->launches += 1;
  return 0;
}

int arks_enable_metrics(arks_ctx* ctx, int on) {
  if (!ctx) return ARKS_E_INVALID_ARG;
  ctx->metrics_on = on != 0;
  if (ctx->loaded) ctx->dt.metrics = ctx->metrics_on ? ctx->d_metrics : nullptr;
  return 0;
}
int arks_snapshot_metrics(arks_ctx* ctx, int64_t* rows) {
  if (!ctx || !ctx->loaded) return ARKS_E_NOT_LOADED;
  if (!rows) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (ctx->ht.n_qos) CK(cudaMemcpy(rows, ctx->d_metrics, (size_t)8 * ARKS_METRIC_COLS * ctx->ht.n_qos, cudaMemcpyDeviceToHost));
  return 0;
}

void* arks_alloc_pinned(size_t bytes) {
  void* p = nullptr;
  return cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) == cudaSuccess ? p : nullptr;
}
void arks_free_pinned(void* p) {
  if (p) cudaFreeHost(p);
}

// ---- BPE side output ------------------------------------------------------------------------------
static_assert(kBpeMaxVocabs == ARKS_BPE_MAX_VOCABS && kBpeFlagNfc == ARKS_BPE_NFC && kBpeFlagDigits3 == ARKS_BPE_DIGITS3 &&
                  kBpeFlagIgnoreMerges == ARKS_BPE_IGNORE_MERGES, "include/arks_gateway.h and bpe.cuh disagree");
// Slot 0 is the default vocabulary (arks_load_bpe); slots 1.. are bound to models by name (arks_bind_model_vocab). Every
// slot has its own merge / hot / byte-id tables and flags; the Unicode class table is one, uploaded with slot 0.
int arks_load_bpe_vocab(arks_ctx* ctx, uint32_t slot, const arks_bpe_tables* t, const uint8_t* tok_bytes, const uint32_t* tok_off,
                        uint32_t n_tok) {
  if (!ctx || slot >= kBpeMaxVocabs) return ARKS_E_INVALID_ARG;
  if (!t && slot == 0 && ctx->meter) return fail(ctx, ARKS_E_INVALID_ARG, "stream metering needs the vocabulary: switch it off first");
  if (!t && slot == 0 && (ctx->vocab_loaded & ~1u)) return fail(ctx, ARKS_E_INVALID_ARG, "other vocabulary slots are loaded: empty them first");
  if (t && slot != 0 && !ctx->bpe_on) return fail(ctx, ARKS_E_NOT_LOADED, "vocabulary slot %u needs slot 0 (arks_load_bpe) first", slot);
  if (t && (t->flags & ARKS_BPE_IGNORE_MERGES) && (!tok_off || (n_tok && !tok_bytes)))
    return fail(ctx, ARKS_E_INVALID_ARG, "ARKS_BPE_IGNORE_MERGES needs the vocabulary's token strings");
  if (!t) {
    {
      // the check and the clearing in one section: a binding that comes after it finds the slot empty (ARKS_E_NOT_LOADED)
      std::lock_guard<std::mutex> g(ctx->cfg_mu);
      bool bound = slot != 0 && ((ctx->vocab_used >> slot) & 1u);
      for (const auto& kv : ctx->vocab_bind) bound |= slot != 0 && kv.second == slot;
      if (bound)
        return fail(ctx, ARKS_E_INVALID_ARG, "vocabulary slot %u: a model is bound to it (bind it to slot 0 and publish a generation first)", slot);
      ctx->vocab_loaded &= ~(1u << slot);
    }
    if (slot == 0) ctx->bpe_on = false;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));  // batches queued before this call still read the tables
    for (void* p : ctx->bpe_allocs[slot]) cudaFree(p);
    ctx->bpe_allocs[slot].clear();
    return 0;
  }
  // A replacement is built completely before the slot's current tables are touched: a refused or failed load leaves the
  // slot (and the bindings and generations that use it) as they were.
  if (!t->byte_id || (slot == 0 && !t->cp_class) || (t->n_merges && (!t->left || !t->right || !t->merged)))
    return fail(ctx, ARKS_E_INVALID_ARG, "incomplete BPE tables");
  CK(cudaSetDevice(ctx->device));
  std::vector<BpeSlot> table, hot;
  const uint32_t slots = bpe_table_slots(t->n_merges);
  bpe_fill_table(table, slots, t->left, t->right, t->merged, t->n_merges);
  bpe_fill_table(hot, kBpeHotSlots, t->left, t->right, t->merged, t->n_merges < kBpeHotMerges ? t->n_merges : kBpeHotMerges);
  std::vector<void*> fresh;
  auto up = [&](const void* src, size_t bytes, const void** out) -> cudaError_t {
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes + 64);
    if (e != cudaSuccess) return e;
    fresh.push_back(p);
    *out = p;
    return cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice);
  };
  auto drop = [&](cudaError_t e) {
    for (void* p : fresh) cudaFree(p);
    return fail(ctx, ARKS_E_CUDA, "arks_load_bpe_vocab: %s (slot %u unchanged)", cudaGetErrorString(e), slot);
  };
  BpeTablesDev d{};
  cudaError_t e = up(t->byte_id, 256 * 4, (const void**)&d.byte_id);
  if (e == cudaSuccess) e = up(table.data(), table.size() * sizeof(BpeSlot), (const void**)&d.table);
  if (e == cudaSuccess) e = up(hot.data(), hot.size() * sizeof(BpeSlot), (const void**)&d.hot);
  d.table_mask = slots - 1;
  d.flags = t->flags;
  if (e == cudaSuccess && (t->flags & ARKS_BPE_IGNORE_MERGES)) {
    std::vector<BpeWholeSlot> whole;
    d.whole_mask = bpe_fill_whole(whole, tok_bytes, tok_off, n_tok) - 1;
    e = up(whole.data(), whole.size() * sizeof(BpeWholeSlot), (const void**)&d.whole);
    if (e == cudaSuccess) e = up(tok_off, ((size_t)n_tok + 1) * 4, (const void**)&d.whole_off);
    if (e == cudaSuccess)
      e = up(n_tok ? (const void*)tok_bytes : (const void*)tok_off, n_tok ? tok_off[n_tok] : 0, (const void**)&d.whole_pool);
  }
  // per-context buffers, allocated once and kept
  if (e == cudaSuccess && !ctx->d_bpe_text) {
    // The work list holds max_bytes / 3 + 1024 entries (one per pre-token) per batch and vocabulary slot: a pre-token is
    // rarely shorter than three bytes on average, but digits and "1 2 3" style text make about one per byte. A row whose
    // entries do not all fit is reported ARKS_BPE_UNCOUNTED (which rows: the order lanes reach the list). Such a row
    // gets no N4 pre-charge and, when metered (N5), is billed its body length.
    const uint32_t cap = (uint32_t)std::min<uint64_t>(ctx->max_bytes / 3 + 1024, 0xfffffff0ull);
    uint8_t* text = nullptr;
    unsigned long long* list = nullptr;
    uint32_t* cnt = nullptr;
    e = cudaMalloc(&text, ctx->max_bytes + 64);
    if (e == cudaSuccess) e = cudaMalloc(&list, (size_t)cap * 8);
    if (e == cudaSuccess) e = cudaMalloc(&cnt, 256);
    if (e == cudaSuccess) {
      ctx->d_bpe_text = text; ctx->d_bpe_list = list; ctx->d_bpe_n = cnt; ctx->bpe_list_cap = cap;
    } else {
      cudaFree(text); cudaFree(list); cudaFree(cnt);
    }
  }
  if (e == cudaSuccess && slot != 0 && !ctx->d_bpe_rows) e = cudaMalloc(&ctx->d_bpe_rows, (size_t)kBpeMaxVocabs * ctx->max_batch * 4 + 64);
  if (e == cudaSuccess && slot == 0 && !ctx->d_bpe_cls) e = cudaMalloc(&ctx->d_bpe_cls, 0x110000 / 2 + 64);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);  // batches queued before this call still read the old tables
  if (e == cudaSuccess && slot == 0) e = cudaMemcpy(ctx->d_bpe_cls, t->cp_class, 0x110000 / 2, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return drop(e);
  d.cp_class = ctx->d_bpe_cls;
  for (void* p : ctx->bpe_allocs[slot]) cudaFree(p);
  ctx->bpe_allocs[slot] = std::move(fresh);
  ctx->bpe[slot] = d;
  if (slot == 0) ctx->bpe_on = true;
  std::lock_guard<std::mutex> g(ctx->cfg_mu);
  ctx->vocab_loaded |= 1u << slot;
  return 0;
}
int arks_load_bpe(arks_ctx* ctx, const arks_bpe_tables* t) {
  if (!ctx) return ARKS_E_INVALID_ARG;
  if (t && (t->flags & ARKS_BPE_IGNORE_MERGES))
    return fail(ctx, ARKS_E_INVALID_ARG, "ARKS_BPE_IGNORE_MERGES needs the token strings: use arks_load_bpe_vocab");
  return arks_load_bpe_vocab(ctx, 0, t, nullptr, nullptr, 0);
}
int arks_bind_model_vocab(arks_ctx* ctx, const char* model, uint32_t model_len, uint32_t slot) {
  if (!ctx || (!model && model_len) || slot >= kBpeMaxVocabs) return ARKS_E_INVALID_ARG;
  std::lock_guard<std::mutex> g(ctx->cfg_mu);
  const std::string m(model ? model : "", model_len);
  if (slot == 0) { ctx->vocab_bind.erase(m); return 0; }
  if (!((ctx->vocab_loaded >> slot) & 1u)) return fail(ctx, ARKS_E_NOT_LOADED, "vocabulary slot %u is not loaded", slot);
  ctx->vocab_bind[m] = slot;
  return 0;
}
// queue the two BPE kernels for `n` bodies on the compute stream; counts land in bpe_out. Rows whose row_flags (may be null)
// contain every bit of wide_mask count the wide key set of metered rows
// row_qos: each row's qos index in the current generation (-1: none), which picks its vocabulary when the generation binds
// a model to a slot other than 0. Otherwise (one vocabulary) exactly the two kernels over all rows.
static int queue_bpe(arks_ctx* ctx, const uint8_t* bodies, const uint32_t* body_off, const uint32_t* body_len, uint32_t n, uint32_t* bpe_out,
                     const uint8_t* row_flags, uint32_t wide_mask, const int32_t* row_qos) {
  if (!ctx->vocab_multi) {
    // one vocabulary (slot 0), with its own pre-tokenizer family and ignore_merges flag; flags 0 is the Qwen2 pair
    const BpeTablesDev& T = ctx->bpe[0];
    CK(cudaMemsetAsync(ctx->d_bpe_n, 0, 4, ctx->stream));
    if (T.flags & ARKS_BPE_DIGITS3)
      bpe_scan_kernel<3, false><<<(n + 127) / 128, 128, 0, ctx->stream>>>(bodies, body_off, body_len, n, T, ctx->d_bpe_text, ctx->d_bpe_list,
                                                                          ctx->d_bpe_n, ctx->bpe_list_cap, bpe_out, row_flags, wide_mask,
                                                                          nullptr, nullptr);
    else
      bpe_scan_kernel<1, false><<<(n + 127) / 128, 128, 0, ctx->stream>>>(bodies, body_off, body_len, n, T, ctx->d_bpe_text, ctx->d_bpe_list,
                                                                          ctx->d_bpe_n, ctx->bpe_list_cap, bpe_out, row_flags, wide_mask,
                                                                          nullptr, nullptr);
    if (T.flags & ARKS_BPE_IGNORE_MERGES)
      bpe_merge_kernel<true><<<ctx->n_sm * 4, kBpeMergeThreads, 0, ctx->stream>>>(ctx->d_bpe_list, ctx->d_bpe_n, ctx->bpe_list_cap, T,
                                                                                  ctx->d_bpe_text, bpe_out);
    else
      bpe_merge_kernel<false><<<ctx->n_sm * 4, kBpeMergeThreads, 0, ctx->stream>>>(ctx->d_bpe_list, ctx->d_bpe_n, ctx->bpe_list_cap, T,
                                                                                   ctx->d_bpe_text, bpe_out);
    ctx->launches += 2;
    return 0;
  }
  // Several vocabularies: the rows are split into one list per slot, then every slot in use runs the two kernels over its
  // own rows with its own tables. The text buffer and the work list are reused in stream order (a row's decoded text sits
  // at its body's offset, so the slots never overlap); each slot has its own counters in d_bpe_n: [16 + s] work-list
  // entries, [32 + s] rows.
  uint32_t* list_n = ctx->d_bpe_n + 16;
  uint32_t* rows_n = ctx->d_bpe_n + 32;
  const uint32_t use = (ctx->vocab_used | 1u) & ctx->vocab_loaded;
  CK(cudaMemsetAsync(list_n, 0, 32 * 4, ctx->stream));
  bpe_split_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(ctx->dt.qos_vocab, row_qos, n, use, ctx->d_bpe_rows, ctx->max_batch, rows_n);
  ctx->launches += 1;
  for (uint32_t v = 0; v < kBpeMaxVocabs; v++) {
    if (!((use >> v) & 1u)) continue;
    const BpeTablesDev& T = ctx->bpe[v];
    const uint32_t* rows = ctx->d_bpe_rows + (size_t)v * ctx->max_batch;
    if (T.flags & ARKS_BPE_DIGITS3)
      bpe_scan_kernel<3, true><<<(n + 127) / 128, 128, 0, ctx->stream>>>(bodies, body_off, body_len, n, T, ctx->d_bpe_text, ctx->d_bpe_list,
                                                                         list_n + v, ctx->bpe_list_cap, bpe_out, row_flags, wide_mask, rows,
                                                                         rows_n + v);
    else
      bpe_scan_kernel<1, true><<<(n + 127) / 128, 128, 0, ctx->stream>>>(bodies, body_off, body_len, n, T, ctx->d_bpe_text, ctx->d_bpe_list,
                                                                         list_n + v, ctx->bpe_list_cap, bpe_out, row_flags, wide_mask, rows,
                                                                         rows_n + v);
    if (T.flags & ARKS_BPE_IGNORE_MERGES)
      bpe_merge_kernel<true><<<ctx->n_sm * 4, kBpeMergeThreads, 0, ctx->stream>>>(ctx->d_bpe_list, list_n + v, ctx->bpe_list_cap, T,
                                                                                  ctx->d_bpe_text, bpe_out);
    else
      bpe_merge_kernel<false><<<ctx->n_sm * 4, kBpeMergeThreads, 0, ctx->stream>>>(ctx->d_bpe_list, list_n + v, ctx->bpe_list_cap, T,
                                                                                   ctx->d_bpe_text, bpe_out);
    ctx->launches += 2;
  }
  return 0;
}
// queue meter_charge_kernel (N5) on the compute stream, timed on its own when profiling
static int queue_meter(arks_ctx* ctx, uint32_t n, const uint8_t* reason, const uint8_t* flags, uint32_t mask, const int32_t* qos,
                       const uint32_t* bpe, const uint32_t* body_len, int side) {
  if (ctx->prof) CK(cudaEventRecord(ctx->ev_meter[0], ctx->stream));
  meter_charge_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(ctx->dt, n, reason, flags, mask, qos, bpe, body_len, side);
  if (ctx->prof) { CK(cudaEventRecord(ctx->ev_meter[1], ctx->stream)); ctx->ev_meter_set = true; }
  ctx->launches += 1;
  return 0;
}

// ---- config plane -------------------------------------------------------------------------------
// Counters of the outgoing generation carried into the incoming one ON THE DEVICE, stream-ordered between two batches:
// row q of the new arrays is row map[q] of the old ones (or zero). No host round trip, no stream synchronisation.
__global__ void carry_rows_kernel(long long* dst, const long long* src, const int32_t* map, uint32_t n_new, uint32_t cols, uint32_t dst_stride,
                                  uint32_t src_stride, int col_major) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_new * cols) return;
  const uint32_t q = col_major ? k % n_new : k / cols, c = col_major ? k / n_new : k % cols;
  const int32_t o = map[q];
  // rate counters are [rule][qos] (col_major: the "column" index c selects the rule plane), the others [row][col]
  const size_t di = col_major ? (size_t)c * dst_stride + q : (size_t)q * cols + c;
  const size_t si = col_major ? (size_t)c * src_stride + (o < 0 ? 0 : o) : (size_t)(o < 0 ? 0 : o) * cols + c;
  dst[di] = o < 0 ? 0 : src[si];
}

// a generation built off the data path (arks_prepare_tables), waiting for arks_commit_tables
struct arks_prepared {
  HostTables ht;
  std::vector<void*> allocs;  // tables; freed when the generation is retired
  DevTables d{};
  long long *rate = nullptr, *quota = nullptr, *metrics = nullptr, *qdelta = nullptr, *qtmp = nullptr, *qexp = nullptr;
  int32_t *d_qos_from = nullptr, *d_quota_from = nullptr;  // new row -> old row, on the device
  std::vector<int32_t> old_to_new;                          // qos index of the outgoing generation -> this one
  uint32_t base_generation = 0;
  uint32_t n_qos = 0, n_quotas = 0;
  uint32_t vocab_used = 0;  // vocabulary slots other than 0 its qos entries use (arks_bind_model_vocab at prepare time)
};

static void free_prepared(arks_ctx* ctx, arks_prepared* p) {
  if (!p) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->cfg_stream);
  for (void* q : p->allocs) cudaFree(q);
  delete p;
}
void arks_discard_prepared(arks_ctx* ctx, arks_prepared* p) {
  if (ctx) free_prepared(ctx, p);
}

int arks_prepare_tables(arks_ctx* ctx, const arks_tables* t, arks_prepared** out) {
  if (!ctx || !t || !out) return ARKS_E_INVALID_ARG;
  *out = nullptr;
  if (const char* why = tables_shape_error(t)) return fail(ctx, ARKS_E_BAD_TABLE, "arks_tables: %s", why);
  CK(cudaSetDevice(ctx->device));
  auto S = [&](uint32_t id) {
    return std::string((const char*)t->str_bytes + t->str_off[id], t->str_off[id + 1] - t->str_off[id]);
  };
  for (uint32_t i = 0; i < t->n_rl; i++)
    if (t->rl_rule[i] >= ARKS_N_RULES) return fail(ctx, ARKS_E_BAD_TABLE, "unknown rate-limit rule %u", t->rl_rule[i]);
  for (uint32_t i = 0; i < t->n_qitems; i++)
    if (t->qitem_type[i] >= ARKS_N_QT) return fail(ctx, ARKS_E_BAD_TABLE, "unknown quota type %u", t->qitem_type[i]);
  for (uint32_t q = 0; q < t->n_qos; q++) {
    if (t->qos_rl_off[q + 1] - t->qos_rl_off[q] > 255) return fail(ctx, ARKS_E_BAD_TABLE, "more than 255 rate limits");
    if (t->qos_quota[q] >= (int32_t)t->n_quotas || t->qos_quota[q] < ARKS_QUOTA_MISSING)
      return fail(ctx, ARKS_E_BAD_TABLE, "qos %u: bad quota index", q);
  }
  for (uint32_t q = 0; q < t->n_quotas; q++)
    if (t->quota_item_off[q + 1] - t->quota_item_off[q] > 255) return fail(ctx, ARKS_E_BAD_TABLE, "more than 255 quota items");

  // string pool on the device: token strings and model names, deduplicated by content
  std::vector<uint8_t> pool;
  std::unordered_map<std::string, uint32_t> pool_at;
  auto intern = [&](const std::string& s) {
    auto it = pool_at.find(s);
    if (it != pool_at.end()) return it->second;
    uint32_t off = (uint32_t)pool.size();
    pool.insert(pool.end(), s.begin(), s.end());
    pool_at.emplace(s, off);
    return off;
  };
  // endpoints by (namespace, name); first object wins on duplicates
  std::unordered_map<std::string, int32_t> ep_by_key;
  for (uint32_t e = 0; e < t->n_endpoints; e++) ep_by_key.emplace(S(t->ep_ns_str[e]) + '\0' + S(t->ep_name_str[e]), (int32_t)e);

  HostTables ht;
  ht.n_tokens = t->n_tokens; ht.n_qos = t->n_qos; ht.n_quotas = t->n_quotas; ht.n_endpoints = t->n_endpoints;
  ht.n_backends = t->n_backends;
  ht.ep_backend_off.assign(t->ep_backend_off, t->ep_backend_off + t->n_endpoints + 1);
  std::vector<uint32_t> tok_off(t->n_tokens), tok_len(t->n_tokens), qmodel_off(t->n_qos), qmodel_len(t->n_qos);
  std::vector<int32_t> qos_ep(t->n_qos);
  uint32_t cap = 16;
  while (cap < 2 * t->n_tokens + 2) cap <<= 1;
  std::vector<TokSlot> slots(cap, TokSlot{0, -1, 0});
  ht.qos_key.resize(t->n_qos);
  for (uint32_t k = 0; k < t->n_tokens; k++) {
    std::string tk = S(t->tok_token_str[k]), ns = S(t->tok_ns_str[k]), nm = S(t->tok_name_str[k]);
    tok_off[k] = intern(tk);
    tok_len[k] = (uint32_t)tk.size();
    unsigned long long h = 0xcbf29ce484222325ull;
    for (unsigned char c : tk) h = (h ^ c) * 0x100000001b3ull;
    uint32_t s = (uint32_t)h & (cap - 1);
    bool dup = false;
    while (slots[s].tok >= 0) {
      if (slots[s].hash == h && S(t->tok_token_str[slots[s].tok]) == tk) { dup = true; break; }  // first object wins
      s = (s + 1) & (cap - 1);
    }
    if (!dup) slots[s] = TokSlot{h, (int)k, 0};
    for (uint32_t q = t->tok_qos_off[k]; q < t->tok_qos_off[k + 1]; q++) {
      std::string model = S(t->qos_model_str[q]);
      qmodel_off[q] = intern(model);
      qmodel_len[q] = (uint32_t)model.size();
      auto it = ep_by_key.find(ns + '\0' + model);
      qos_ep[q] = it == ep_by_key.end() ? -1 : it->second;
      ht.qos_key[q] = ns + '\0' + nm + '\0' + model;
      int32_t qt = t->qos_quota[q];
      if (qt >= 0 && S(t->quota_ns_str[qt]) != ns)
        return fail(ctx, ARKS_E_BAD_TABLE, "qos %u references a quota of another namespace", q);
    }
  }
  ht.quota_key.resize(t->n_quotas);
  for (uint32_t q = 0; q < t->n_quotas; q++) ht.quota_key[q] = S(t->quota_ns_str[q]) + '\0' + S(t->quota_name_str[q]);

  // counters are carried over by key (Redis keys survive a CRD edit): which old row feeds every new row
  std::vector<int32_t> qos_from(t->n_qos + 1, -1), quota_from(t->n_quotas + 1, -1);
  std::vector<int32_t> old_to_new;  // qos index of the outgoing generation -> this one
  uint32_t base_generation;
  std::unordered_map<std::string, uint32_t> vocab_bind;  // model name -> BPE vocabulary slot, as bound now
  {
    // the only part that looks at the current generation: short, so that a commit on the batch thread never waits for
    // the tens of milliseconds a prepare on the config thread takes
    std::lock_guard<std::mutex> cfg_guard(ctx->cfg_mu);
    base_generation = ctx->generation;
    vocab_bind = ctx->vocab_bind;
    old_to_new.assign(ctx->loaded ? ctx->ht.n_qos : 0, -1);
  if (ctx->loaded) {
    std::unordered_map<std::string, uint32_t> oq, ou;
    for (uint32_t q = 0; q < ctx->ht.n_qos; q++) oq.emplace(ctx->ht.qos_key[q], q);
    for (uint32_t q = 0; q < ctx->ht.n_quotas; q++) ou.emplace(ctx->ht.quota_key[q], q);
    for (uint32_t q = 0; q < t->n_qos; q++) {
      auto it = oq.find(ht.qos_key[q]);
      if (it != oq.end()) {
        qos_from[q] = (int32_t)it->second;
        if (old_to_new[it->second] < 0) old_to_new[it->second] = (int32_t)q;  // first entry with the key, as in the lookup
      }
    }
    for (uint32_t q = 0; q < t->n_quotas; q++) {
      auto it = ou.find(ht.quota_key[q]);
      if (it != ou.end()) quota_from[q] = (int32_t)it->second;
    }
  }
  }

  // the BPE vocabulary of every qos entry, by its model name (the ArksEndpoint name)
  std::vector<uint8_t> qos_vocab(t->n_qos, 0);
  uint32_t vocab_used = 0;
  if (!vocab_bind.empty())
    for (uint32_t q = 0; q < t->n_qos; q++) {
      auto it = vocab_bind.find(S(t->qos_model_str[q]));
      if (it == vocab_bind.end()) continue;
      qos_vocab[q] = (uint8_t)it->second;
      vocab_used |= 1u << it->second;
    }
  vocab_used &= ~1u;

  // Build the new generation completely before touching the old one, on the config stream: a failed allocation or upload
  // leaves the context serving the previous tables and counters, and the data path never waits for any of this.
  // ONE allocation, ONE upload and ONE memset per generation (a config thread that makes dozens of driver calls competes
  // with the batch thread for the context lock): arrays are first only laid out, 256-byte aligned, uploads in front and the
  // zero-initialised counters behind them.
  struct Piece { const void* src; size_t bytes, span; void** out; size_t off; };
  std::vector<Piece> pieces;
  std::vector<void*> fresh;
  auto drop_fresh = [&]() {
    cudaStreamSynchronize(ctx->cfg_stream);
    for (void* p : fresh) cudaFree(p);
  };
  auto put = [&](const void* src, size_t bytes, void** out, size_t alloc_bytes = 0) -> int {
    const size_t span = ((alloc_bytes > bytes ? alloc_bytes : bytes) + 64 + 255) & ~(size_t)255;
    pieces.push_back(Piece{src, src ? bytes : 0, span, out, 0});
    return 0;
  };
#define PUT(vec, field) put((vec).data(), (vec).size() * sizeof((vec)[0]), (void**)&d.field)
  DevTables d{};
  std::vector<uint32_t> v_tok_qos_off(t->tok_qos_off, t->tok_qos_off + t->n_tokens + 1);
  std::vector<int32_t> v_qos_quota(t->qos_quota, t->qos_quota + t->n_qos);
  std::vector<uint32_t> v_qos_rl_off(t->qos_rl_off, t->qos_rl_off + t->n_qos + 1);
  std::vector<uint8_t> v_rl_rule(t->rl_rule, t->rl_rule + t->n_rl);
  std::vector<int64_t> v_rl_value(t->rl_value, t->rl_value + t->n_rl);
  std::vector<uint32_t> v_qi_off(t->quota_item_off, t->quota_item_off + t->n_quotas + 1);
  std::vector<uint8_t> v_qi_type(t->qitem_type, t->qitem_type + t->n_qitems);
  std::vector<int64_t> v_qi_val(t->qitem_value, t->qitem_value + t->n_qitems);
  std::vector<uint32_t> v_ep_off(t->ep_backend_off, t->ep_backend_off + t->n_endpoints + 1);
  std::vector<int32_t> v_bw(t->backend_weight, t->backend_weight + t->n_backends);
  PUT(pool, pool);
  PUT(slots, tok_slots);
  d.tok_mask = cap - 1;
  PUT(tok_off, tok_str_off);
  PUT(tok_len, tok_str_len);
  PUT(v_tok_qos_off, tok_qos_off);
  PUT(qmodel_off, qos_model_off);
  PUT(qmodel_len, qos_model_len);
  PUT(v_qos_quota, qos_quota);
  PUT(qos_ep, qos_ep);
  PUT(qos_vocab, qos_vocab);
  PUT(v_qos_rl_off, qos_rl_off);
  PUT(v_rl_rule, rl_rule);
  PUT(v_rl_value, rl_value);
  PUT(v_qi_off, quota_item_off);
  PUT(v_qi_type, qitem_type);
  PUT(v_qi_val, qitem_value);
  PUT(v_ep_off, ep_backend_off);
  PUT(v_bw, backend_weight);
  long long *n_rate = nullptr, *n_quota = nullptr, *n_metrics = nullptr, *n_qdelta = nullptr, *n_qtmp = nullptr, *n_qexp = nullptr;
  int32_t *n_qos_from = nullptr, *n_quota_from = nullptr;
  {
    int rc;
    if ((rc = put(nullptr, 0, (void**)&n_rate, (size_t)32 * t->n_qos))) return rc;
    if ((rc = put(nullptr, 0, (void**)&n_quota, (size_t)24 * t->n_quotas))) return rc;
    if ((rc = put(nullptr, 0, (void**)&n_metrics, (size_t)8 * ARKS_METRIC_COLS * t->n_qos))) return rc;
    if ((rc = put(qos_from.data(), (size_t)4 * (t->n_qos + 1), (void**)&n_qos_from))) return rc;
    if ((rc = put(quota_from.data(), (size_t)4 * (t->n_quotas + 1), (void**)&n_quota_from))) return rc;
    if (ctx->share_quota) {
      if ((rc = put(nullptr, 0, (void**)&n_qdelta, (size_t)24 * t->n_quotas))) return rc;
      // two scratch vectors as long as the delta (host-form apply, export snapshot)
      if ((rc = put(nullptr, 0, (void**)&n_qtmp, (size_t)24 * t->n_quotas))) return rc;
      if ((rc = put(nullptr, 0, (void**)&n_qexp, (size_t)24 * t->n_quotas))) return rc;
    }
  }
#undef PUT
  {
    size_t up = 0, total = 0;
    for (Piece& pc : pieces)
      if (pc.src) { pc.off = up; up += pc.span; }
    total = up;
    for (Piece& pc : pieces)
      if (!pc.src) { pc.off = total; total += pc.span; }
    uint8_t* arena = nullptr;
    cudaError_t e = cudaMalloc(&arena, total + 256);
    if (e == cudaSuccess) {
      fresh.push_back(arena);
      std::vector<uint8_t> stage(up + 1, 0);
      for (const Piece& pc : pieces)
        if (pc.src && pc.bytes) memcpy(stage.data() + pc.off, pc.src, pc.bytes);
      e = cudaMemcpyAsync(arena, stage.data(), up, cudaMemcpyHostToDevice, ctx->cfg_stream);
      if (e == cudaSuccess && total > up) e = cudaMemsetAsync(arena + up, 0, total - up, ctx->cfg_stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->cfg_stream);  // the CONFIG stream: the data path is not involved
    }
    if (e != cudaSuccess) {
      drop_fresh();
      return fail(ctx, ARKS_E_CUDA, "arks_prepare_tables: %s (tables unchanged)", cudaGetErrorString(e));
    }
    for (const Piece& pc : pieces) *pc.out = arena + pc.off;
  }
  arks_prepared* p = new arks_prepared();
  p->allocs = fresh;
  p->rate = n_rate; p->quota = n_quota; p->metrics = n_metrics; p->qdelta = n_qdelta; p->qtmp = n_qtmp; p->qexp = n_qexp;
  p->d_qos_from = n_qos_from; p->d_quota_from = n_quota_from;
  d.n_qos = t->n_qos;
  p->d = d;
  p->ht = std::move(ht);
  p->old_to_new = std::move(old_to_new);
  p->base_generation = base_generation;
  p->n_qos = t->n_qos;
  p->n_quotas = t->n_quotas;
  p->vocab_used = vocab_used;
  *out = p;
  return 0;
}

// The swap: stream-ordered between the batch queued before this call and the one queued after it. Counters are carried
// into the new arrays by a few small kernels on the compute stream; the old generation is released once they have run.
// Call from the thread that submits batches. No host-side wait.
int arks_commit_tables(arks_ctx* ctx, arks_prepared* p) {
  if (!ctx || !p) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  std::lock_guard<std::mutex> cfg_guard(ctx->cfg_mu);
  if (p->base_generation != ctx->generation)
    return fail(ctx, ARKS_E_INVALID_ARG, "prepared against generation %u, the context is at %u: prepare again", p->base_generation, ctx->generation);
  if (p->vocab_used & ~ctx->vocab_loaded)
    return fail(ctx, ARKS_E_INVALID_ARG, "prepared with a BPE vocabulary slot that has been emptied since: prepare again");
  if (ctx->loaded) {
    auto carry = [&](long long* dst, const long long* src, const int32_t* map, uint32_t n_new, uint32_t cols, uint32_t ds, uint32_t ss, int cm) {
      if (!dst || !src || !n_new) return;
      const uint32_t total = n_new * cols;
      carry_rows_kernel<<<(total + 255) / 256, 256, 0, ctx->stream>>>(dst, src, map, n_new, cols, ds, ss, cm);
      ctx->launches += 1;
    };
    carry(p->rate, ctx->d_rate, p->d_qos_from, p->n_qos, 4, p->n_qos, ctx->ht.n_qos, 1);
    carry(p->metrics, ctx->d_metrics, p->d_qos_from, p->n_qos, ARKS_METRIC_COLS, 0, 0, 0);
    carry(p->quota, ctx->d_quota, p->d_quota_from, p->n_quotas, 3, 0, 0, 0);
    carry(p->qdelta, ctx->d_qdelta, p->d_quota_from, p->n_quotas, 3, 0, 0, 0);
    CK(cudaGetLastError());
  }
  // retire the outgoing generation: freed stream-ordered, after the carry kernels and everything queued before them
  for (void* q : ctx->table_allocs) cudaFreeAsync(q, ctx->stream);  // the one arena of the outgoing generation
  ctx->table_allocs = std::move(p->allocs);
  ctx->d_rate = p->rate; ctx->d_quota = p->quota; ctx->d_metrics = p->metrics;
  ctx->d_qdelta = p->qdelta; ctx->d_qtmp = p->qtmp; ctx->d_qexp = p->qexp;
  ctx->d_qos_from = p->d_qos_from; ctx->d_quota_from = p->d_quota_from;
  ctx->qexp_valid = false;
  ctx->d_backend_weight = const_cast<int32_t*>(p->d.backend_weight);
  DevTables d = p->d;
  d.rate = ctx->d_rate;
  d.metrics = ctx->metrics_on ? ctx->d_metrics : nullptr;
  d.quota = ctx->d_quota;
  d.qdelta = ctx->d_qdelta;
  ctx->dt = d;
  if (ctx->loaded) {
    ctx->remap.push_back(std::move(p->old_to_new));
    if (ctx->remap.size() > ARKS_GEN_HISTORY) ctx->remap.pop_front();
  }
  ctx->ht = std::move(p->ht);
  ctx->vocab_used = p->vocab_used;
  ctx->vocab_multi = p->vocab_used != 0;
  ctx->generation++;
  ctx->loaded = true;
  delete p;
  return 0;
}

// cold start / blocking form: prepare + commit on the calling thread
int arks_load_tables(arks_ctx* ctx, const arks_tables* t) {
  arks_prepared* p = nullptr;
  int rc = arks_prepare_tables(ctx, t, &p);
  if (rc) return rc;
  rc = arks_commit_tables(ctx, p);
  if (rc) { free_prepared(ctx, p); return rc; }
  CK(cudaStreamSynchronize(ctx->stream));
  return 0;
}


// ---- object-level config plane: config_store.h keeps the objects, these are the C entry points ----
static void free_store(ConfigStore* s) { delete s; }
static ConfigStore& store_of(arks_ctx* ctx) {
  if (!ctx->store) ctx->store = new ConfigStore();
  return *ctx->store;
}
static bool str_ok(const char* p, uint32_t n) { return p || !n; }

int arks_upsert_token(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const char* token,
                      uint32_t token_len, const arks_qos_spec* qos, uint32_t n_qos) {
  if (!ctx || !str_ok(ns, ns_len) || !str_ok(name, name_len) || !str_ok(token, token_len) || (n_qos && !qos)) return ARKS_E_INVALID_ARG;
  for (uint32_t i = 0; i < n_qos; i++)
    if (!str_ok(qos[i].model, qos[i].model_len) || !str_ok(qos[i].quota, qos[i].quota_len) || (qos[i].n_rl && (!qos[i].rl_rule || !qos[i].rl_value)))
      return fail(ctx, ARKS_E_INVALID_ARG, "arks_upsert_token: qos %u has a NULL field", i);
  std::lock_guard<std::mutex> g(ctx->cfg_mu);
  store_of(ctx).upsert_token(ns, ns_len, name, name_len, token, token_len, qos, n_qos);
  return 0;
}
int arks_upsert_quota(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const uint8_t* item_type,
                      const int64_t* item_value, uint32_t n_items) {
  if (!ctx || !str_ok(ns, ns_len) || !str_ok(name, name_len) || (n_items && (!item_type || !item_value))) return ARKS_E_INVALID_ARG;
  std::lock_guard<std::mutex> g(ctx->cfg_mu);
  store_of(ctx).upsert_quota(ns, ns_len, name, name_len, item_type, item_value, n_items);
  return 0;
}
int arks_upsert_endpoint(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len,
                         const int32_t* backend_weight, uint32_t n_backends) {
  if (!ctx || !str_ok(ns, ns_len) || !str_ok(name, name_len) || (n_backends && !backend_weight)) return ARKS_E_INVALID_ARG;
  std::lock_guard<std::mutex> g(ctx->cfg_mu);
  store_of(ctx).upsert_endpoint(ns, ns_len, name, name_len, backend_weight, n_backends);
  return 0;
}
static int store_erase(arks_ctx* ctx, int which, const char* what, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len) {
  if (!ctx || !str_ok(ns, ns_len) || !str_ok(name, name_len)) return ARKS_E_INVALID_ARG;
  std::lock_guard<std::mutex> g(ctx->cfg_mu);
  if (!store_of(ctx).erase(which, ns, ns_len, name, name_len))
    return fail(ctx, ARKS_E_INVALID_ARG, "%s %.*s/%.*s is not in the store", what, (int)ns_len, ns ? ns : "", (int)name_len, name ? name : "");
  return 0;
}
int arks_delete_token(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len) {
  return store_erase(ctx, 0, "ArksToken", ns, ns_len, name, name_len);
}
int arks_delete_quota(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len) {
  return store_erase(ctx, 1, "ArksQuota", ns, ns_len, name, name_len);
}
int arks_delete_endpoint(arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len) {
  return store_erase(ctx, 2, "ArksEndpoint", ns, ns_len, name, name_len);
}
// store -> arks_tables (the flat form arks_prepare_tables validates and uploads), objects in (namespace, name) order
int arks_config_prepare(arks_ctx* ctx, arks_prepared** out) {
  if (!ctx || !out) return ARKS_E_INVALID_ARG;
  FlatTables flat;
  {
    std::lock_guard<std::mutex> g(ctx->cfg_mu);
    store_of(ctx).flatten(&flat);
  }
  const arks_tables t = flat.view();
  return arks_prepare_tables(ctx, &t, out);
}

// the host tables of the current generation are replaced by arks_commit_tables (batch thread) under cfg_mu: readers on the
// config thread take it too
int32_t arks_find_quota(const arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len) {
  if (!ctx) return -1;
  std::lock_guard<std::mutex> g(const_cast<arks_ctx*>(ctx)->cfg_mu);
  if (!ctx->loaded) return -1;
  const std::string k = std::string(ns ? ns : "", ns_len) + '\0' + std::string(name ? name : "", name_len);
  for (uint32_t q = 0; q < ctx->ht.n_quotas; q++)
    if (ctx->ht.quota_key[q] == k) return (int32_t)q;
  return -1;
}
int32_t arks_find_qos(const arks_ctx* ctx, const char* ns, uint32_t ns_len, const char* user, uint32_t user_len, const char* model,
                      uint32_t model_len) {
  if (!ctx) return -1;
  std::lock_guard<std::mutex> g(const_cast<arks_ctx*>(ctx)->cfg_mu);
  if (!ctx->loaded) return -1;
  const std::string k = std::string(ns ? ns : "", ns_len) + '\0' + std::string(user ? user : "", user_len) + '\0' + std::string(model ? model : "", model_len);
  for (uint32_t q = 0; q < ctx->ht.n_qos; q++)
    if (ctx->ht.qos_key[q] == k) return (int32_t)q;
  return -1;
}

uint32_t arks_table_generation(const arks_ctx* ctx) { return ctx ? ctx->generation : 0; }
int arks_set_precharge(arks_ctx* ctx, int on) {
  if (!ctx) return ARKS_E_INVALID_ARG;
  ctx->precharge = on != 0;
  return 0;
}
int arks_set_stream_metering(arks_ctx* ctx, int on) {
  if (!ctx) return ARKS_E_INVALID_ARG;
  if (on && !ctx->bpe_on) return fail(ctx, ARKS_E_NOT_LOADED, "stream metering needs a vocabulary (arks_load_bpe)");
  ctx->meter = on != 0;
  return 0;
}

int arks_update_endpoint_weights(arks_ctx* ctx, uint32_t ep, uint32_t n, const int32_t* w) {
  if (!ctx || !ctx->loaded) return ARKS_E_NOT_LOADED;
  if (ep >= ctx->ht.n_endpoints || ctx->ht.ep_backend_off[ep + 1] - ctx->ht.ep_backend_off[ep] != n)
    return fail(ctx, ARKS_E_INVALID_ARG, "endpoint %u has a different backend count", ep);
  if (n == 0) return 0;
  if (!w) return ARKS_E_INVALID_ARG;
  for (uint32_t i = 0; i < n; i++)
    if (w[i] < 0) return fail(ctx, ARKS_E_INVALID_ARG, "endpoint %u: negative backend weight", ep);
  CK(cudaSetDevice(ctx->device));
  // stream-ordered: lands between the previous and the next batch
  CK(cudaMemcpyAsync(ctx->d_backend_weight + ctx->ht.ep_backend_off[ep], w, n * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// fixed-window roll-over: a new window is a new Redis key, i.e. every counter of that rule reads 0
static int roll_windows(arks_ctx* ctx, int64_t now) {
  for (int r = 0; r < 4; r++)
    if (window_start(now, r) < ctx->last_win[r])
      return fail(ctx, ARKS_E_TIME_WENT_BACK, "now_unix %lld is before the current %s window", (long long)now,
                  r == 0 ? "rpm" : r == 1 ? "rpd" : r == 2 ? "tpm" : "tpd");
  for (int r = 0; r < 4; r++) {
    int64_t ws = window_start(now, r);
    if (ws != ctx->last_win[r]) {
      if (ctx->last_win[r] != INT64_MIN && ctx->ht.n_qos)
        CK(cudaMemsetAsync(ctx->d_rate + (size_t)r * ctx->ht.n_qos, 0, (size_t)8 * ctx->ht.n_qos, ctx->stream));
      ctx->last_win[r] = ws;
    }
  }
  return 0;
}

// ---- staging slots --------------------------------------------------------------------------------
static int ensure_slot(arks_ctx* ctx, int k, bool want_req, bool want_resp) {
  arks_ctx::Slot& sl = ctx->slots[k];
  if (want_req && !sl.d_req_bodies) {
    CK(cudaMalloc(&sl.d_req_bodies, ctx->max_bytes + 64));  // + slack: the fast path reads whole 32-byte chunks
    CK(cudaMalloc(&sl.d_req_meta, ctx->meta_cap));
    CK(cudaMallocHost(&sl.h_req_meta, ctx->meta_cap));
    CK(cudaEventCreateWithFlags(&sl.req_copied, cudaEventDisableTiming));
    CK(cudaMallocHost(&sl.h_req_result, ctx->result_cap));
    CK(cudaEventCreateWithFlags(&sl.req_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&sl.req_ran, cudaEventDisableTiming));
  }
  if (want_resp && !sl.d_resp_bodies) {
    CK(cudaMalloc(&sl.d_resp_bodies, ctx->max_bytes + 64));
    CK(cudaMalloc(&sl.d_resp_meta, ctx->meta_cap));
    CK(cudaMallocHost(&sl.h_resp_meta, ctx->meta_cap));
    CK(cudaEventCreateWithFlags(&sl.resp_copied, cudaEventDisableTiming));
    CK(cudaMallocHost(&sl.h_resp_result, ctx->result_cap));
    CK(cudaEventCreateWithFlags(&sl.resp_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&sl.resp_ran, cudaEventDisableTiming));
  }
  return 0;
}

int arks_select_slot(arks_ctx* ctx, int slot) {
  if (!ctx || slot < 0 || slot >= arks_ctx::kSlots) return ARKS_E_INVALID_ARG;
  ctx->cur = slot;
  return 0;
}

int arks_set_profiling(arks_ctx* ctx, int on) {
  if (!ctx) return ARKS_E_INVALID_ARG;
  ctx->prof = on != 0;
  return 0;
}

int arks_last_kernel_ms(arks_ctx* ctx, float* ms, int cap) {
  if (!ctx || !ms) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (ctx->ev_n == 0) return 0;
  // request: scan stage, rank_hot + limit_admit, fast-path kernel alone (0 if not used), BPE kernels (0 if off)
  // response: scan stage, fast-path kernel alone, BPE kernels
  // both: + the meter kernel when it ran (N5)
  float v[5] = {0, 0, 0, 0, 0};
  int n = 0;
  CK(cudaEventElapsedTime(&v[n++], ctx->ev[0], ctx->ev[1]));
  if (ctx->is_req_timing) CK(cudaEventElapsedTime(&v[n++], ctx->ev_admit0, ctx->ev[2]));
  if (ctx->ev_fast_set) CK(cudaEventElapsedTime(&v[n], ctx->ev_fast[0], ctx->ev_fast[1]));
  n++;
  if (ctx->ev_bpe_set) CK(cudaEventElapsedTime(&v[n], ctx->ev_bpe[0], ctx->ev_bpe[1]));
  n++;
  if (ctx->ev_meter_set) CK(cudaEventElapsedTime(&v[n++], ctx->ev_meter[0], ctx->ev_meter[1]));
  for (int k = 0; k < n && k < cap; k++) ms[k] = v[k];
  return n < cap ? n : cap;
}

// ---- request phase ------------------------------------------------------------------------------
int arks_stage_request_batch(arks_ctx* ctx, const arks_request_batch* b) {
  if (!ctx || !b) return ARKS_E_INVALID_ARG;
  // a batch that is refused below, for any reason, leaves nothing to run in this slot (not even its previous tenant)
  ctx->slots[ctx->cur].req_staged = false;
  ctx->last_route = -1;  // until the bodies are on their way
  if (!ctx->loaded) return fail(ctx, ARKS_E_NOT_LOADED, "arks_load_tables has not been called");
  const uint32_t n = b->n;
  if (n > ctx->max_batch) return fail(ctx, ARKS_E_CAPACITY, "batch of %u exceeds max_batch %u", n, ctx->max_batch);
  if (b->bodies_bytes > ctx->max_bytes) return fail(ctx, ARKS_E_CAPACITY, "batch bytes exceed max_batch_bytes");
  CK(cudaSetDevice(ctx->device));
  int rc = ensure_slot(ctx, ctx->cur, true, false);
  if (rc) return rc;
  arks_ctx::Slot& sl = ctx->slots[ctx->cur];
  sl.req_n = n;
  if (n == 0) { sl.req_staged = true; return 0; }
  if (!b->body_off || !b->body_len || !b->token_off || (b->bodies_bytes && !b->bodies) || (b->token_off[n] && !b->tokens))
    return fail(ctx, ARKS_E_INVALID_ARG, "request batch: null array");
  for (uint32_t i = 0; i < n; i++) {
    if ((b->body_off[i] & 15u) || (uint64_t)b->body_off[i] + b->body_len[i] > b->bodies_bytes)
      return fail(ctx, ARKS_E_INVALID_ARG, "body %u: offset not 16-byte aligned or out of range", i);
    if (b->token_off[i] > b->token_off[i + 1]) return fail(ctx, ARKS_E_INVALID_ARG, "token %u: offsets decrease", i);
  }
  const size_t tok_bytes = b->token_off[n];
  size_t o_off = 0, o_len = o_off + align_up((size_t)n * 4, 256), o_toff = o_len + align_up((size_t)n * 4, 256),
         o_rand = o_toff + align_up((size_t)(n + 1) * 4, 256), o_tok = o_rand + align_up((size_t)n * 8, 256),
         total = o_tok + align_up(tok_bytes + 1, 256);
  if (total > ctx->meta_cap) return fail(ctx, ARKS_E_CAPACITY, "token bytes exceed capacity");
  CK(cudaEventSynchronize(sl.req_copied));  // the pinned block may still feed the previous copy of this slot
  uint8_t* h = sl.h_req_meta;
  memcpy(h + o_off, b->body_off, (size_t)n * 4);
  memcpy(h + o_len, b->body_len, (size_t)n * 4);
  memcpy(h + o_toff, b->token_off, (size_t)(n + 1) * 4);
  if (b->pick_rand) memcpy(h + o_rand, b->pick_rand, (size_t)n * 8);
  if (tok_bytes) memcpy(h + o_tok, b->tokens, tok_bytes);
  // (a micro-batch whose tokens leave no room for its bodies behind the metadata takes the large path: separate buffer)
  const bool small = b->bodies_bytes <= kSmallBatchBytes && total + b->bodies_bytes <= ctx->meta_cap;
  if (small) {
    // one upload for a handful of bodies (the extra memcpy is cheaper than a second copy call); above that the bodies go
    // up from the caller's buffer, as in the large path, but still on the compute stream (no cross-stream event)
    if (b->bodies_bytes <= kTinyBatchBytes) {
      memcpy(h + total, b->bodies, b->bodies_bytes);
      CK(cudaMemcpyAsync(sl.d_req_meta, h, total + b->bodies_bytes, cudaMemcpyHostToDevice, ctx->stream));
    } else {
      CK(cudaMemcpyAsync(sl.d_req_meta, h, total, cudaMemcpyHostToDevice, ctx->stream));
      CK(cudaMemcpyAsync(sl.d_req_meta + total, b->bodies, b->bodies_bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    CK(cudaEventRecord(sl.req_copied, ctx->stream));
  } else {
    // uploads run on their own stream so that they overlap the kernels of the batches queued before this one
    CK(cudaStreamWaitEvent(ctx->h2d, sl.req_ran, 0));  // the previous tenant of this slot's device buffers is done
    CK(cudaMemcpyAsync(sl.d_req_bodies, b->bodies, b->bodies_bytes, cudaMemcpyHostToDevice, ctx->h2d));
    CK(cudaMemcpyAsync(sl.d_req_meta, h, total, cudaMemcpyHostToDevice, ctx->h2d));
    CK(cudaEventRecord(sl.req_copied, ctx->h2d));
  }
  ReqDev& r = sl.rq;
  r.bodies = small ? sl.d_req_meta + total : sl.d_req_bodies;
  r.body_off = (const uint32_t*)(sl.d_req_meta + o_off);
  r.body_len = (const uint32_t*)(sl.d_req_meta + o_len);
  r.token_off = (const uint32_t*)(sl.d_req_meta + o_toff);
  r.pick_rand = b->pick_rand ? (const unsigned long long*)(sl.d_req_meta + o_rand) : nullptr;
  r.tokens = sl.d_req_meta + o_tok;
  r.n = n;
  sl.req_staged = true;
  ctx->last_route = small ? (b->bodies_bytes <= kTinyBatchBytes ? 0 : 1) : 2;
  return 0;
}

// offsets of the 11 result arrays inside the packed result block of a batch of n (dense: one D2H for any n)
constexpr int kReqResultArrays = 11;
static void result_offsets(size_t n, size_t offs[kReqResultArrays + 1]) {
  const size_t a1 = align_up(n, 16), a4 = align_up(n * 4, 16), a8 = align_up(n * 8, 16);
  offs[0] = 0; offs[1] = a1; offs[2] = 2 * a1; offs[3] = 3 * a1; offs[4] = offs[3] + a4; offs[5] = offs[4] + a4;
  offs[6] = offs[5] + a4; offs[7] = offs[6] + a8; offs[8] = offs[7] + a8;
  offs[9] = offs[8] + a4; offs[10] = offs[9] + a4; offs[11] = offs[10] + a4;
}
// Micro-batches write their result rows straight into the slot's pinned host block (zero copy over PCIe: the block is
// device-addressable under unified addressing): no D2H copy node between the last kernel and the host's wake-up.
constexpr uint32_t kZeroCopyRows = 2048;
static void carve_request(arks_ctx* ctx, ReqDev& r, size_t batch_n, uint8_t* result_base) {
  const size_t n = ctx->max_batch;
  uint8_t* p = ctx->d_inter;
  r.st_reason = p; p += align_up(n, 256);
  r.st_flags = p; p += align_up(n, 256);
  r.st_qos = (int32_t*)p; p += align_up(n * 4, 256);
  r.st_tok = (int32_t*)p; p += align_up(n * 4, 256);
  r.gslot = (int32_t*)p; p += align_up(n * 4, 256);
  r.gnext = (int32_t*)p; p += align_up(n * 4, 256);
  r.gkey = (int32_t*)p; p += align_up((size_t)ctx->gsize * 4, 256);   // gkey and ghead are contiguous: one memset(-1)
  r.ghead = (int32_t*)p; p += align_up((size_t)ctx->gsize * 4, 256);
  r.gcnt = (int32_t*)p; p += align_up((size_t)ctx->gsize * 4, 256) + 256;  // + the hot-group counter word
  r.gsnap = (long long*)p; p += align_up((size_t)ctx->gsize * 32, 256);
  r.hot_n = (int32_t*)p; p += 256;
  r.hot_list = (int32_t*)p; p += align_up((n / kHotGroup + 2) * 4, 256);
  r.hotrank = (int32_t*)p;
  size_t offs[kReqResultArrays + 1];
  result_offsets(batch_n, offs);
  uint8_t* q = result_base;
  r.reason = q + offs[0];
  r.detail = q + offs[1];
  r.flags = q + offs[2];
  r.qos = (int32_t*)(q + offs[3]);
  r.token = (int32_t*)(q + offs[4]);
  r.pick = (int32_t*)(q + offs[5]);
  r.cur_usage = (long long*)(q + offs[6]);
  r.limit_max = (long long*)(q + offs[7]);
  r.model_off = (uint32_t*)(q + offs[8]);
  r.model_len = (uint32_t*)(q + offs[9]);
  r.bpe = (uint32_t*)(q + offs[10]);
}

// A warp is as slow as its slowest body and pays for every code path any of its lanes takes, so a small batch is spread
// over more warps with fewer bodies each (the SMs are idle anyway): about 2048 warps, the number one full wave keeps
// resident, is the target. 64 requests -> 64 warps of one body; 65 536 -> 2048 warps of 32.
static uint32_t bodies_per_warp(uint32_t n) {
  const uint32_t b = (n + 2047) / 2048;
  return b < 1 ? 1 : b > 32 ? 32 : b;
}
static uint32_t scan_grid(uint32_t n, uint32_t bpw) { return ((n + bpw - 1) / bpw + kWarpsPerBlock - 1) / kWarpsPerBlock; }

// batches below this size are a handful of warps: the three small launches would cost more than they save
constexpr uint32_t kSortMinBatch = 4096;
// from this size on requests / complete response bodies go through the two-stage scan (mask_scan.cuh first); below it
// the exact kernel alone is one launch and spreads the few bodies over more warps (bodies_per_warp)


// queue the counting sort by body length; returns the permutation (device pointer) or null when the batch is scanned as is
static const uint32_t* queue_length_order(arks_ctx* ctx, const uint32_t* d_body_len, uint32_t n) {
  if (!ctx->sort_lanes || n < kSortMinBatch) return nullptr;
  cudaMemsetAsync(ctx->d_lenhist, 0, (size_t)4 * kLenBuckets, ctx->stream);
  len_hist_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_body_len, n, ctx->d_lenhist);
  len_scan_kernel<<<1, 1024, 0, ctx->stream>>>(ctx->d_lenhist);
  len_scatter_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(d_body_len, n, ctx->d_lenhist, ctx->d_perm);
  ctx->launches += 3;
  return ctx->d_perm;
}

int arks_run_request_batch(arks_ctx* ctx, int64_t now_unix) {
  if (!ctx || !ctx->loaded) return ARKS_E_INVALID_ARG;
  arks_ctx::Slot& sl = ctx->slots[ctx->cur];
  if (!sl.req_staged) return fail(ctx, ARKS_E_INVALID_ARG, "no request batch staged in slot %d", ctx->cur);
  CK(cudaSetDevice(ctx->device));
  int rc = roll_windows(ctx, now_unix);
  if (rc) return rc;
  const uint32_t n = sl.req_n;
  ctx->fetch_n = n;
  ctx->ev_n = 0;
  ctx->ev_fast_set = false;
  ctx->ev_bpe_set = false;
  ctx->ev_meter_set = false;
  ctx->last_two_stage = false;
  if (n == 0) return 0;
  CK(cudaStreamWaitEvent(ctx->stream, sl.req_copied, 0));
  ReqDev& r = sl.rq;
  sl.req_zc = n <= kZeroCopyRows && sl.h_req_result;
  carve_request(ctx, r, n, sl.req_zc ? sl.h_req_result : ctx->d_result);
  r.meter = ctx->meter ? 1 : 0;
  // batch-local group table sized to the batch (2x, power of two); the three arrays are contiguous
  uint32_t g = 64;
  while (g < 2 * n) g <<= 1;
  r.gmask = g - 1;
  // gkey | ghead | gcnt are laid out back to back for THIS batch's table size: one memset(0xff) clears all three
  r.ghead = r.gkey + g;
  r.gcnt = r.gkey + 2 * (size_t)g;
  r.hot_n = r.gkey + 3 * (size_t)g;  // one more word: the hot-group counter, also starting at -1
  CK(cudaMemsetAsync(r.gkey, 0xff, (size_t)g * 12 + 8, ctx->stream));  // + the hot-group and declined-rows counters
  const uint32_t tpb = kWarpsPerBlock * 32;
  r.slow_n = reinterpret_cast<uint32_t*>(r.hot_n + 1);  // cleared to -1 by the group table's memset
  r.slow_list = ctx->d_slow + 64;
  ctx->last_slow_n = r.slow_n;
  if (ctx->prof) CK(cudaEventRecord(ctx->ev[0], ctx->stream));
  if (ctx->fast_scan && n <= ctx->warp_max) {
    // latency path: a warp per body (warp_scan.cuh), the exact engine for what it declines
    r.perm = nullptr;
    warp_request_kernel<<<(n + kWdWarps - 1) / kWdWarps, kWdWarps * 32, kWdSmemPerBlock, ctx->stream>>>(ctx->dt, r);
    r.bpw = 1;
    switch (ctx->sched[0]) {
#define ARKS_LAUNCH(S) case S: scan_request_kernel<S, true><<<scan_grid(n, r.bpw), tpb, kSmemPerBlock, ctx->stream>>>(ctx->dt, r); break;
      ARKS_FOR_SCHED(ARKS_LAUNCH)
#undef ARKS_LAUNCH
    }
    ctx->launches += 1;
    ctx->last_two_stage = true;
  } else if (ctx->fast_scan && n >= ctx->fast_min) {
    // two-stage scan: the fast path (mask_scan.cuh) decides everything plain, the exact engine what it declines. The batch
    // stays in arrival order (every block orders its own 128 documents: fast_block_order) unless ARKS_SORT=2 asks for the
    // global length order the exact engine uses
    r.perm = ctx->sort_fast ? queue_length_order(ctx, r.body_len, n) : nullptr;
    if (ctx->prof) CK(cudaEventRecord(ctx->ev_fast[0], ctx->stream));
    if (ctx->split)
      fast_request_kernel2<8><<<(n + kSplitDocs - 1) / kSplitDocs, kFastThreads, sizeof(FastSplitSmem), ctx->stream>>>(ctx->dt, r, ctx->regroup);
    else if (ctx->walk8)
      fast_request_kernel<8><<<(n + kFastThreads - 1) / kFastThreads, kFastThreads, sizeof(FastBlockSmem), ctx->stream>>>(ctx->dt, r, ctx->regroup);
    else
      fast_request_kernel<0><<<(n + kFastThreads - 1) / kFastThreads, kFastThreads, sizeof(FastBlockSmem), ctx->stream>>>(ctx->dt, r, ctx->regroup);
    if (ctx->prof) { CK(cudaEventRecord(ctx->ev_fast[1], ctx->stream)); ctx->ev_fast_set = true; }
    r.perm = nullptr;
    r.bpw = 32;
    switch (ctx->sched[0]) {
#define ARKS_LAUNCH(S) case S: scan_request_kernel<S, true><<<scan_grid(n, r.bpw), tpb, kSmemPerBlock, ctx->stream>>>(ctx->dt, r); break;
      ARKS_FOR_SCHED(ARKS_LAUNCH)
#undef ARKS_LAUNCH
    }
    ctx->launches += 1;
    ctx->last_two_stage = true;
  } else {
    r.perm = queue_length_order(ctx, r.body_len, n);
    r.bpw = bodies_per_warp(n);
    switch (ctx->sched[0]) {
#define ARKS_LAUNCH(S) case S: scan_request_kernel<S, false><<<scan_grid(n, r.bpw), tpb, kSmemPerBlock, ctx->stream>>>(ctx->dt, r); break;
      ARKS_FOR_SCHED(ARKS_LAUNCH)
#undef ARKS_LAUNCH
    }
  }
  if (ctx->prof) CK(cudaEventRecord(ctx->ev[1], ctx->stream));
  if (ctx->bpe_on) {
    if (ctx->prof) CK(cudaEventRecord(ctx->ev_bpe[0], ctx->stream));
    rc = queue_bpe(ctx, r.bodies, r.body_off, r.body_len, n, r.bpe, ctx->meter ? r.st_flags : nullptr, ARKS_FLAG_METERED, r.st_qos);
    if (rc) return rc;
    if (ctx->prof) { CK(cudaEventRecord(ctx->ev_bpe[1], ctx->stream)); ctx->ev_bpe_set = true; }
  }
  if (ctx->prof) CK(cudaEventRecord(ctx->ev_admit0, ctx->stream));
  if (n > (uint32_t)kHotGroup) {  // a group can only be hot if the batch is larger than the threshold
    rank_hot_groups_kernel<<<296, 256, 0, ctx->stream>>>(r);  // exits at once when scan_request listed no hot group
    ctx->launches += 1;
  }
  r.precharge = ctx->precharge && ctx->bpe_on ? 1 : 0;
  limit_admit_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(ctx->dt, r);
  if (ctx->prof) { CK(cudaEventRecord(ctx->ev[2], ctx->stream)); ctx->ev_n = 3; ctx->is_req_timing = true; }
  if (ctx->meter) {  // N5: the prompts of the admitted metered rows are charged when the micro-batch commits
    rc = queue_meter(ctx, n, r.reason, r.flags, ARKS_FLAG_METERED, r.qos, ctx->bpe_on ? r.bpe : nullptr, r.body_len, 0);
    if (rc) return rc;
  }
  CK(cudaEventRecord(sl.req_ran, ctx->stream));
  ctx->launches += 2;
  CK(cudaGetLastError());
  return 0;
}

// enqueue the D2H of the packed result block of the batch just run in the current slot (no host wait)
static int enqueue_request_fetch(arks_ctx* ctx) {
  arks_ctx::Slot& sl = ctx->slots[ctx->cur];
  const size_t n = ctx->fetch_n;
  sl.req_fetch_n = (uint32_t)n;
  if (n == 0) return 0;
  size_t offs[kReqResultArrays + 1];
  result_offsets(n, offs);
  if (!sl.req_zc) CK(cudaMemcpyAsync(sl.h_req_result, ctx->d_result, offs[kReqResultArrays], cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(sl.req_done, ctx->stream));
  return 0;
}
// Wait for an event by polling it: cudaEventSynchronize from the completion thread would sit inside the driver while the
// dispatcher thread is trying to queue the next batch (measured: two batches in flight were slower than one).
static cudaError_t wait_event_polling(cudaEvent_t ev) {
  for (uint32_t spins = 0;; spins++) {
    const cudaError_t e = cudaEventQuery(ev);
    if (e != cudaErrorNotReady) return e;
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
    if (spins > 200000) return cudaEventSynchronize(ev);  // something is slow (a large batch): stop burning the core
  }
}
static int finish_request_fetch(arks_ctx* ctx, int slot, arks_request_result* out) {
  arks_ctx::Slot& sl = ctx->slots[slot];
  const size_t n = sl.req_fetch_n;
  if (n == 0) return 0;
  CK(wait_event_polling(sl.req_done));
  const uint8_t* h = sl.h_req_result;
  size_t offs[kReqResultArrays + 1];
  result_offsets(n, offs);
  memcpy(out->reason, h + offs[0], n);
  memcpy(out->detail, h + offs[1], n);
  memcpy(out->flags, h + offs[2], n);
  memcpy(out->qos, h + offs[3], n * 4);
  memcpy(out->token, h + offs[4], n * 4);
  memcpy(out->pick, h + offs[5], n * 4);
  memcpy(out->cur_usage, h + offs[6], n * 8);
  memcpy(out->limit_max, h + offs[7], n * 8);
  if (out->model_off) memcpy(out->model_off, h + offs[8], n * 4);
  if (out->model_len) memcpy(out->model_len, h + offs[9], n * 4);
  if (out->bpe_count) memcpy(out->bpe_count, h + offs[10], n * 4);
  return 0;
}
int arks_fetch_request_result(arks_ctx* ctx, arks_request_result* out) {
  if (!ctx || !out) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  int rc = ensure_slot(ctx, ctx->cur, true, false);
  if (rc) return rc;
  rc = enqueue_request_fetch(ctx);
  if (rc) return rc;
  return finish_request_fetch(ctx, ctx->cur, out);
}
// asynchronous form: H2D + kernels + D2H are queued on the stream and the call returns; arks_wait_request blocks
// until that slot's results are in `out`. Up to kSlots batches can be in flight (one per slot).
int arks_submit_request_async(arks_ctx* ctx, const arks_request_batch* b) {
  int rc = arks_stage_request_batch(ctx, b);
  if (rc) return rc;
  rc = arks_run_request_batch(ctx, b->now_unix);
  if (rc) return rc;
  return enqueue_request_fetch(ctx);
}
int arks_wait_request(arks_ctx* ctx, int slot, arks_request_result* out) {
  if (!ctx || !out || slot < 0 || slot >= arks_ctx::kSlots) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  return finish_request_fetch(ctx, slot, out);
}

int arks_submit_request_batch(arks_ctx* ctx, const arks_request_batch* b, arks_request_result* r) {
  int rc = arks_stage_request_batch(ctx, b);
  if (rc) return rc;
  rc = arks_run_request_batch(ctx, b->now_unix);
  if (rc) return rc;
  return arks_fetch_request_result(ctx, r);
}

// ---- response phase -----------------------------------------------------------------------------
// qos index `q` issued under table generation `g` -> index in the current tables, or -1
static int32_t resolve_qos(const arks_ctx* ctx, int32_t q, uint32_t g) {
  if (q < 0 || g > ctx->generation) return -1;
  const uint32_t steps = ctx->generation - g;
  if (steps > ctx->remap.size()) return -1;
  for (size_t k = ctx->remap.size() - steps; k < ctx->remap.size(); k++) {
    if ((size_t)q >= ctx->remap[k].size()) return -1;
    q = ctx->remap[k][(size_t)q];
    if (q < 0) return -1;
  }
  return (uint32_t)q < ctx->ht.n_qos ? q : -1;
}
int arks_stage_response_batch(arks_ctx* ctx, const arks_response_batch* b) {
  if (!ctx || !b) return ARKS_E_INVALID_ARG;
  // a batch that is refused below, for any reason, leaves nothing to run in this slot (not even its previous tenant)
  ctx->slots[ctx->cur].resp_staged = false;
  ctx->last_route = -1;  // until the bodies are on their way
  if (!ctx->loaded) return fail(ctx, ARKS_E_NOT_LOADED, "arks_load_tables has not been called");
  const uint32_t n = b->n;
  if (n > ctx->max_batch) return fail(ctx, ARKS_E_CAPACITY, "batch of %u exceeds max_batch %u", n, ctx->max_batch);
  if (b->bodies_bytes > ctx->max_bytes) return fail(ctx, ARKS_E_CAPACITY, "batch bytes exceed max_batch_bytes");
  CK(cudaSetDevice(ctx->device));
  int rc = ensure_slot(ctx, ctx->cur, false, true);
  if (rc) return rc;
  arks_ctx::Slot& sl = ctx->slots[ctx->cur];
  sl.resp_n = n;
  if (n == 0) { sl.resp_staged = true; return 0; }
  if (!b->body_off || !b->body_len || !b->qos || !b->flags || (b->bodies_bytes && !b->bodies)) return fail(ctx, ARKS_E_INVALID_ARG, "response batch: null array");
  uint32_t n_sse = 0, n_metered = 0;
  for (uint32_t i = 0; i < n; i++) {
    n_sse += (b->flags[i] & ARKS_RESP_STREAM) != 0;
    n_metered += (b->flags[i] & (ARKS_RESP_STREAM | ARKS_RESP_METERED)) == (ARKS_RESP_STREAM | ARKS_RESP_METERED);
    if ((b->body_off[i] & 15u) || (uint64_t)b->body_off[i] + b->body_len[i] > b->bodies_bytes)
      return fail(ctx, ARKS_E_INVALID_ARG, "body %u: offset not 16-byte aligned or out of range", i);
  }
  sl.resp_mode = n_sse == 0 ? 1 : n_sse == n ? 2 : 0;
  sl.resp_n_sse = n_sse;
  sl.resp_metered = n_metered != 0;
  size_t o_off = 0, o_len = align_up((size_t)n * 4, 256), o_qos = o_len * 2, o_fl = o_len * 3, o_kind = o_fl + align_up(n, 256),
         o_pre = o_kind + (sl.resp_mode == 0 ? o_len : 0), total = o_pre + (b->precharged ? o_len : 0);
  if (total + (b->bodies_bytes <= kTinyBatchBytes ? b->bodies_bytes : 0) > ctx->meta_cap) return fail(ctx, ARKS_E_CAPACITY, "response metadata exceeds capacity");
  CK(cudaEventSynchronize(sl.resp_copied));
  uint8_t* h = sl.h_resp_meta;
  if (sl.resp_mode == 0) {  // mixed batch: complete bodies first, SSE chunks after; each kind goes to its own kernel
    uint32_t* kind = reinterpret_cast<uint32_t*>(h + o_kind);
    uint32_t a = 0, c = n - n_sse;
    for (uint32_t i = 0; i < n; i++) kind[(b->flags[i] & ARKS_RESP_STREAM) ? c++ : a++] = i;
  }
  memcpy(h + o_off, b->body_off, (size_t)n * 4);
  memcpy(h + o_len, b->body_len, (size_t)n * 4);
  {
    // A row's qos index is positional in the tables of the generation that decided its request. Rows of an older
    // generation are carried to the current one by key; a row that cannot be resolved (never had a qos entry, index out
    // of range, key removed, generation older than the history) is marked -1 and answered ARKS_R_QOS_GONE by the kernel:
    // one stale stream never fails the micro-batch it shares with other tenants.
    int32_t* hq = reinterpret_cast<int32_t*>(h + o_qos);
    for (uint32_t i = 0; i < n; i++) hq[i] = resolve_qos(ctx, b->qos[i], b->gen ? b->gen[i] : ctx->generation);
  }
  memcpy(h + o_fl, b->flags, n);
  if (b->precharged) memcpy(h + o_pre, b->precharged, (size_t)n * 4);
  const bool small = b->bodies_bytes <= kSmallBatchBytes;
  if (small) {  // uploads on the compute stream (see kSmallBatchBytes / kTinyBatchBytes)
    if (b->bodies_bytes <= kTinyBatchBytes) {
      memcpy(h + total, b->bodies, b->bodies_bytes);
      CK(cudaMemcpyAsync(sl.d_resp_meta, h, total + b->bodies_bytes, cudaMemcpyHostToDevice, ctx->stream));
    } else {
      CK(cudaMemcpyAsync(sl.d_resp_meta, h, total, cudaMemcpyHostToDevice, ctx->stream));
      CK(cudaMemcpyAsync(sl.d_resp_meta + total, b->bodies, b->bodies_bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    CK(cudaEventRecord(sl.resp_copied, ctx->stream));
  } else {
    CK(cudaStreamWaitEvent(ctx->h2d, sl.resp_ran, 0));
    CK(cudaMemcpyAsync(sl.d_resp_bodies, b->bodies, b->bodies_bytes, cudaMemcpyHostToDevice, ctx->h2d));
    CK(cudaMemcpyAsync(sl.d_resp_meta, h, total, cudaMemcpyHostToDevice, ctx->h2d));
    CK(cudaEventRecord(sl.resp_copied, ctx->h2d));
  }
  RespDev& r = sl.rp;
  r.bodies = small ? sl.d_resp_meta + total : sl.d_resp_bodies;
  r.body_off = (const uint32_t*)(sl.d_resp_meta + o_off);
  r.body_len = (const uint32_t*)(sl.d_resp_meta + o_len);
  r.qos = (const int32_t*)(sl.d_resp_meta + o_qos);
  r.flags = sl.d_resp_meta + o_fl;
  r.precharged = b->precharged ? (const uint32_t*)(sl.d_resp_meta + o_pre) : nullptr;
  r.n = n;
  sl.d_resp_kind = reinterpret_cast<const uint32_t*>(sl.d_resp_meta + o_kind);
  sl.resp_zc = n <= kZeroCopyRows && sl.h_resp_result;
  uint8_t* rb = sl.resp_zc ? sl.h_resp_result : ctx->d_result;
  r.reason = rb;
  r.counted = rb + align_up(n, 16);
  r.usage = (long long*)(rb + 2 * align_up(n, 16));
  r.bpe = (uint32_t*)(rb + 2 * align_up(n, 16) + (size_t)n * 24);
  sl.resp_staged = true;
  ctx->last_route = small ? (b->bodies_bytes <= kTinyBatchBytes ? 0 : 1) : 2;
  return 0;
}

int arks_run_response_batch(arks_ctx* ctx, int64_t now_unix) {
  if (!ctx || !ctx->loaded) return ARKS_E_INVALID_ARG;
  arks_ctx::Slot& sl = ctx->slots[ctx->cur];
  if (!sl.resp_staged) return fail(ctx, ARKS_E_INVALID_ARG, "no response batch staged in slot %d", ctx->cur);
  CK(cudaSetDevice(ctx->device));
  int rc = roll_windows(ctx, now_unix);
  if (rc) return rc;
  const uint32_t n = sl.resp_n;
  ctx->fetch_n = n;
  ctx->ev_n = 0;
  ctx->ev_fast_set = false;
  ctx->ev_bpe_set = false;
  ctx->ev_meter_set = false;
  ctx->last_two_stage = false;
  if (n == 0) return 0;
  const uint32_t tpb = kWarpsPerBlock * 32;
  CK(cudaStreamWaitEvent(ctx->stream, sl.resp_copied, 0));
  if (ctx->prof) CK(cudaEventRecord(ctx->ev[0], ctx->stream));
  // complete bodies and SSE chunks have their own kernels; a mixed batch is two launches over the two halves of its
  // kind index (arrival order inside a kind), a homogeneous one a single launch in length order
  auto launch_json = [&](RespDev rp) {
    rp.bpw = bodies_per_warp(rp.n);
    const dim3 grid(scan_grid(rp.n, rp.bpw));
    switch (ctx->sched[1]) {
#define ARKS_LAUNCH(S) case S: scan_response_kernel<S, false><<<grid, tpb, kSmemPerBlock, ctx->stream>>>(ctx->dt, rp); break;
      ARKS_FOR_SCHED(ARKS_LAUNCH)
#undef ARKS_LAUNCH
    }
  };
  auto launch_json_two_stage = [&](RespDev rp) -> int {
    rp.slow_n = ctx->d_slow;
    rp.slow_list = ctx->d_slow + 64;
    ctx->last_slow_n = rp.slow_n;
    CK(cudaMemsetAsync(ctx->d_slow, 0xff, 4, ctx->stream));
    rp.perm = ctx->sort_fast ? queue_length_order(ctx, rp.body_len, rp.n) : nullptr;
    if (ctx->prof) CK(cudaEventRecord(ctx->ev_fast[0], ctx->stream));
    if (ctx->split)
      fast_response_kernel2<8><<<(rp.n + kSplitDocs - 1) / kSplitDocs, kFastThreads, sizeof(FastSplitSmem), ctx->stream>>>(ctx->dt, rp, ctx->regroup);
    else if (ctx->walk8)
      fast_response_kernel<8><<<(rp.n + kFastThreads - 1) / kFastThreads, kFastThreads, sizeof(FastBlockSmem), ctx->stream>>>(ctx->dt, rp, ctx->regroup);
    else
      fast_response_kernel<0><<<(rp.n + kFastThreads - 1) / kFastThreads, kFastThreads, sizeof(FastBlockSmem), ctx->stream>>>(ctx->dt, rp, ctx->regroup);
    if (ctx->prof) { CK(cudaEventRecord(ctx->ev_fast[1], ctx->stream)); ctx->ev_fast_set = true; }
    rp.perm = nullptr;
    rp.bpw = 32;
    const dim3 grid(scan_grid(rp.n, rp.bpw));
    switch (ctx->sched[1]) {
#define ARKS_LAUNCH(S) case S: scan_response_kernel<S, true><<<grid, tpb, kSmemPerBlock, ctx->stream>>>(ctx->dt, rp); break;
      ARKS_FOR_SCHED(ARKS_LAUNCH)
#undef ARKS_LAUNCH
    }
    ctx->launches += 1;
    ctx->last_two_stage = true;
    return 0;
  };
  auto launch_sse = [&](RespDev rp) {
    rp.bpw = bodies_per_warp(rp.n);
    const dim3 grid(scan_grid(rp.n, rp.bpw));
    switch (ctx->sched[2]) {
#define ARKS_LAUNCH(S) case S: scan_sse_kernel<S><<<grid, tpb, kSseSmemPerBlock, ctx->stream>>>(ctx->dt, rp); break;
      ARKS_FOR_SCHED(ARKS_LAUNCH)
#undef ARKS_LAUNCH
    }
  };
  if (sl.resp_mode == 0) {
    RespDev rj = sl.rp, rs = sl.rp;
    rj.n = n - sl.resp_n_sse; rj.perm = sl.d_resp_kind;
    rs.n = sl.resp_n_sse;     rs.perm = sl.d_resp_kind + rj.n;
    launch_json(rj);
    launch_sse(rs);
    ctx->launches += 1;
  } else {
    if (sl.resp_mode == 1 && ctx->fast_scan && n <= ctx->warp_max) {
      RespDev rp = sl.rp;
      rp.slow_n = ctx->d_slow;
      rp.slow_list = ctx->d_slow + 64;
      rp.perm = nullptr;
      ctx->last_slow_n = rp.slow_n;
      CK(cudaMemsetAsync(ctx->d_slow, 0xff, 4, ctx->stream));
      warp_response_kernel<<<(n + kWdWarps - 1) / kWdWarps, kWdWarps * 32, kWdSmemPerBlock, ctx->stream>>>(ctx->dt, rp);
      rp.bpw = 1;
      const dim3 grid(scan_grid(n, rp.bpw));
      switch (ctx->sched[1]) {
#define ARKS_LAUNCH(S) case S: scan_response_kernel<S, true><<<grid, tpb, kSmemPerBlock, ctx->stream>>>(ctx->dt, rp); break;
        ARKS_FOR_SCHED(ARKS_LAUNCH)
#undef ARKS_LAUNCH
      }
      ctx->launches += 1;
      ctx->last_two_stage = true;
    } else if (sl.resp_mode == 1 && ctx->fast_scan && n >= ctx->fast_min) {
      rc = launch_json_two_stage(sl.rp);
      if (rc) return rc;
    } else {
      sl.rp.perm = queue_length_order(ctx, sl.rp.body_len, n);
      if (sl.resp_mode == 1) launch_json(sl.rp); else launch_sse(sl.rp);
    }
  }
  if (ctx->prof) { CK(cudaEventRecord(ctx->ev[1], ctx->stream)); ctx->ev_n = 2; ctx->is_req_timing = false; }
  if (ctx->bpe_on) {
    if (ctx->prof) CK(cudaEventRecord(ctx->ev_bpe[0], ctx->stream));
    rc = queue_bpe(ctx, sl.rp.bodies, sl.rp.body_off, sl.rp.body_len, n, sl.rp.bpe, sl.resp_metered ? sl.rp.flags : nullptr,
                   ARKS_RESP_STREAM | ARKS_RESP_METERED, sl.rp.qos);
    if (rc) return rc;
    if (ctx->prof) { CK(cudaEventRecord(ctx->ev_bpe[1], ctx->stream)); ctx->ev_bpe_set = true; }
  } else {
    CK(cudaMemsetAsync(sl.rp.bpe, 0, (size_t)n * 4, ctx->stream));
  }
  if (sl.resp_metered) {  // N5: metered chunks answered ARKS_R_OK are billed their completion count
    rc = queue_meter(ctx, n, sl.rp.reason, sl.rp.flags, ARKS_RESP_STREAM | ARKS_RESP_METERED, sl.rp.qos, ctx->bpe_on ? sl.rp.bpe : nullptr,
                     sl.rp.body_len, 1);
    if (rc) return rc;
  }
  CK(cudaEventRecord(sl.resp_ran, ctx->stream));
  ctx->launches += 1;
  CK(cudaGetLastError());
  return 0;
}

static int enqueue_response_fetch(arks_ctx* ctx) {
  arks_ctx::Slot& sl = ctx->slots[ctx->cur];
  const size_t n = ctx->fetch_n;
  sl.resp_fetch_n = (uint32_t)n;
  if (n == 0) return 0;
  const size_t o1 = align_up(n, 16);
  if (!sl.resp_zc) CK(cudaMemcpyAsync(sl.h_resp_result, ctx->d_result, 2 * o1 + n * 28, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(sl.resp_done, ctx->stream));
  return 0;
}
static int finish_response_fetch(arks_ctx* ctx, int slot, arks_response_result* out) {
  arks_ctx::Slot& sl = ctx->slots[slot];
  const size_t n = sl.resp_fetch_n;
  if (n == 0) return 0;
  CK(wait_event_polling(sl.resp_done));
  const size_t o1 = align_up(n, 16);
  const uint8_t* h = sl.h_resp_result;
  memcpy(out->reason, h, n);
  memcpy(out->counted, h + o1, n);
  memcpy(out->usage, h + 2 * o1, n * 24);
  if (out->bpe_count) memcpy(out->bpe_count, h + 2 * o1 + n * 24, n * 4);
  return 0;
}
int arks_fetch_response_result(arks_ctx* ctx, arks_response_result* out) {
  if (!ctx || !out) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  int rc = ensure_slot(ctx, ctx->cur, false, true);
  if (rc) return rc;
  rc = enqueue_response_fetch(ctx);
  if (rc) return rc;
  return finish_response_fetch(ctx, ctx->cur, out);
}
int arks_submit_response_async(arks_ctx* ctx, const arks_response_batch* b) {
  int rc = arks_stage_response_batch(ctx, b);
  if (rc) return rc;
  rc = arks_run_response_batch(ctx, b->now_unix);
  if (rc) return rc;
  return enqueue_response_fetch(ctx);
}
int arks_wait_response(arks_ctx* ctx, int slot, arks_response_result* out) {
  if (!ctx || !out || slot < 0 || slot >= arks_ctx::kSlots) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  return finish_response_fetch(ctx, slot, out);
}

int arks_submit_response_batch(arks_ctx* ctx, const arks_response_batch* b, arks_response_result* r) {
  int rc = arks_stage_response_batch(ctx, b);
  if (rc) return rc;
  rc = arks_run_response_batch(ctx, b->now_unix);
  if (rc) return rc;
  return arks_fetch_response_result(ctx, r);
}

// ---- quota.QuotaService surface / snapshots -------------------------------------------------------
int arks_snapshot_quota(arks_ctx* ctx, int64_t* usage) {
  if (!ctx || !ctx->loaded) return ARKS_E_NOT_LOADED;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  if (ctx->ht.n_quotas) CK(cudaMemcpy(usage, ctx->d_quota, (size_t)24 * ctx->ht.n_quotas, cudaMemcpyDeviceToHost));
  return 0;
}
int arks_set_quota_usage(arks_ctx* ctx, uint32_t quota, const int64_t usage[3]) {
  if (!ctx || !ctx->loaded) return ARKS_E_NOT_LOADED;
  if (quota >= ctx->ht.n_quotas) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  CK(cudaMemcpy(ctx->d_quota + (size_t)3 * quota, usage, 24, cudaMemcpyHostToDevice));
  return 0;
}
int arks_incr_quota_usage(arks_ctx* ctx, uint32_t quota, const int64_t delta[3]) {
  if (!ctx || !ctx->loaded) return ARKS_E_NOT_LOADED;
  if (quota >= ctx->ht.n_quotas) return ARKS_E_INVALID_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  long long cur[3];
  CK(cudaMemcpy(cur, ctx->d_quota + (size_t)3 * quota, 24, cudaMemcpyDeviceToHost));
  for (int k = 0; k < 3; k++) cur[k] = (long long)((unsigned long long)cur[k] + (unsigned long long)delta[k]);
  CK(cudaMemcpy(ctx->d_quota + (size_t)3 * quota, cur, 24, cudaMemcpyHostToDevice));
  return 0;
}
int arks_snapshot_rate(arks_ctx* ctx, int64_t now_unix, int64_t* counters) {
  if (!ctx || !ctx->loaded) return ARKS_E_NOT_LOADED;
  CK(cudaSetDevice(ctx->device));
  CK(cudaStreamSynchronize(ctx->stream));
  const size_t nq = ctx->ht.n_qos;
  std::vector<long long> tmp(4 * nq + 1);
  if (nq) CK(cudaMemcpy(tmp.data(), ctx->d_rate, 32 * nq, cudaMemcpyDeviceToHost));
  for (size_t q = 0; q < nq; q++)
    for (int r = 0; r < 4; r++)
      counters[q * 4 + r] = window_start(now_unix, r) == ctx->last_win[r] ? tmp[(size_t)r * nq + q] : 0;
  return 0;
}

// ---- multi-GPU: quotas shared across GPUs (SURVEY.md §8e) -------------------------------------------
// Every GPU applies its own increments to its replica immediately and also accumulates them in a delta vector.
// A fold epoch = sum the delta vectors over all GPUs (caller: ncclAllReduce / torch.distributed), then on every GPU
// quota += reduced - own_delta, own_delta = 0. Between epochs a replica lags the others' increments (bounded
// staleness, the same class of over-admission the reference's non-atomic Redis path has).
int arks_enable_quota_sharing(arks_ctx* ctx, int on) {
  if (!ctx) return ARKS_E_INVALID_ARG;
  if (ctx->loaded) return fail(ctx, ARKS_E_INVALID_ARG, "enable quota sharing before arks_load_tables");
  ctx->share_quota = on != 0;
  return 0;
}
int arks_take_quota_delta(arks_ctx* ctx, int64_t* delta_out) {
  if (!ctx || !ctx->loaded || !ctx->d_qdelta) return fail(ctx, ARKS_E_INVALID_ARG, "quota sharing is not enabled");
  CK(cudaSetDevice(ctx->device));
  const size_t n = (size_t)3 * ctx->ht.n_quotas;
  CK(cudaMemcpyAsync(delta_out, ctx->d_qdelta, n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_qdelta, 0, n * 8, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return 0;
}
int arks_apply_quota_delta(arks_ctx* ctx, const int64_t* remote_delta) {
  if (!ctx || !ctx->loaded || !ctx->d_qdelta) return fail(ctx, ARKS_E_INVALID_ARG, "quota sharing is not enabled");
  CK(cudaSetDevice(ctx->device));
  const size_t n = (size_t)3 * ctx->ht.n_quotas;
  if (!n) return 0;
  CK(cudaMemcpyAsync(ctx->d_qtmp, remote_delta, n * 8, cudaMemcpyHostToDevice, ctx->stream));
  add_quota_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(ctx->d_quota, ctx->d_qtmp, n);
  ctx->launches += 1;
  CK(cudaStreamSynchronize(ctx->stream));
  return 0;
}
void* arks_quota_delta_dev(arks_ctx* ctx) { return ctx ? (void*)ctx->d_qdelta : nullptr; }
int arks_export_quota_delta_dev(arks_ctx* ctx, void* dst_dev) {
  if (!ctx || !ctx->loaded || !ctx->d_qdelta) return fail(ctx, ARKS_E_INVALID_ARG, "quota sharing is not enabled");
  CK(cudaSetDevice(ctx->device));
  // the library keeps its own copy of what it handed out: the fold subtracts exactly this snapshot
  CK(cudaMemcpyAsync(ctx->d_qexp, ctx->d_qdelta, (size_t)24 * ctx->ht.n_quotas, cudaMemcpyDeviceToDevice, ctx->stream));
  if (dst_dev) CK(cudaMemcpyAsync(dst_dev, ctx->d_qexp, (size_t)24 * ctx->ht.n_quotas, cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->qexp_valid = true;
  return 0;
}
int arks_fold_quota_delta_dev(arks_ctx* ctx, const void* reduced_dev, const void* own_dev) {
  if (!ctx || !ctx->loaded || !ctx->d_qdelta) return fail(ctx, ARKS_E_INVALID_ARG, "quota sharing is not enabled");
  if (!reduced_dev) return fail(ctx, ARKS_E_INVALID_ARG, "reduced_dev is null");
  if (!own_dev && !ctx->qexp_valid) return fail(ctx, ARKS_E_INVALID_ARG, "fold without a preceding arks_export_quota_delta_dev");
  CK(cudaSetDevice(ctx->device));
  const size_t n = (size_t)3 * ctx->ht.n_quotas;
  if (!n) return 0;
  fold_quota_delta_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(
      ctx->d_quota, ctx->d_qdelta, (const long long*)reduced_dev, own_dev ? (const long long*)own_dev : ctx->d_qexp, n);
  ctx->qexp_valid = false;
  ctx->launches += 1;
  CK(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// ---- the fold over NCCL, inside the library ----
struct NcclApi {
  void* dl = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclComm_t comm = nullptr;
  int rank = 0, world = 0;
  uint32_t* d_idx = nullptr;   // local indices of the shared quotas
  long long* d_msg = nullptr;  // what crosses the fabric: n_shared x 3 int64
  uint32_t n_shared = 0;
  bool all_rows = true;
  uint32_t generation = 0;     // the table generation the indices in d_idx belong to
};
static int nccl_load(arks_ctx* ctx) {
  if (ctx->nccl) return 0;
  const char* name = getenv("ARKS_NCCL_LIB");
  void* dl = dlopen(name && *name ? name : "libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
  if (!dl) return fail(ctx, ARKS_E_INVALID_ARG, "dlopen(%s): %s", name && *name ? name : "libnccl.so.2", dlerror());
  NcclApi* a = new NcclApi();
  a->dl = dl;
  a->GetUniqueId = (decltype(a->GetUniqueId))dlsym(dl, "ncclGetUniqueId");
  a->CommInitRank = (decltype(a->CommInitRank))dlsym(dl, "ncclCommInitRank");
  a->AllReduce = (decltype(a->AllReduce))dlsym(dl, "ncclAllReduce");
  a->CommDestroy = (decltype(a->CommDestroy))dlsym(dl, "ncclCommDestroy");
  a->GetErrorString = (decltype(a->GetErrorString))dlsym(dl, "ncclGetErrorString");
  if (!a->GetUniqueId || !a->CommInitRank || !a->AllReduce || !a->CommDestroy || !a->GetErrorString) {
    delete a;
    return fail(ctx, ARKS_E_INVALID_ARG, "libnccl lacks an entry point this library needs");
  }
  ctx->nccl = a;
  return 0;
}
#define NCK(call)                                                                                                \
  do {                                                                                                           \
    ncclResult_t r_ = (call);                                                                                    \
    if (r_ != ncclSuccess) return fail(ctx, ARKS_E_CUDA, "%s: %s", #call, ctx->nccl->GetErrorString(r_));        \
  } while (0)
int arks_comm_unique_id(arks_ctx* ctx, void* out) {
  if (!ctx || !out) return ARKS_E_INVALID_ARG;
  static_assert(sizeof(ncclUniqueId) == ARKS_UNIQUE_ID_BYTES, "ncclUniqueId is 128 bytes");
  int rc = nccl_load(ctx);
  if (rc) return rc;
  ncclUniqueId id;
  NCK(ctx->nccl->GetUniqueId(&id));
  memcpy(out, &id, sizeof id);
  return 0;
}
int arks_comm_set_shared(arks_ctx* ctx, const uint32_t* shared, uint32_t n_shared) {
  if (!ctx || !ctx->nccl) return fail(ctx, ARKS_E_INVALID_ARG, "arks_comm_init first");
  if (!ctx->loaded || !ctx->d_qdelta) return fail(ctx, ARKS_E_INVALID_ARG, "quota sharing is not enabled (or no tables yet)");
  CK(cudaSetDevice(ctx->device));
  NcclApi& a = *ctx->nccl;
  std::vector<uint32_t> idx;
  a.all_rows = !shared;
  if (shared) idx.assign(shared, shared + n_shared);
  else {
    idx.resize(ctx->ht.n_quotas);
    for (uint32_t q = 0; q < ctx->ht.n_quotas; q++) idx[q] = q;
  }
  for (uint32_t q : idx)
    if (q >= ctx->ht.n_quotas) return fail(ctx, ARKS_E_INVALID_ARG, "shared quota index %u out of range", q);
  CK(cudaStreamSynchronize(ctx->stream));
  cudaFree(a.d_idx);
  cudaFree(a.d_msg);
  a.d_idx = nullptr; a.d_msg = nullptr;
  a.n_shared = (uint32_t)idx.size();
  a.generation = ctx->generation;
  CK(cudaMalloc(&a.d_idx, idx.size() * 4 + 64));
  CK(cudaMalloc(&a.d_msg, idx.size() * 24 + 64));
  CK(cudaMemcpy(a.d_idx, idx.data(), idx.size() * 4, cudaMemcpyHostToDevice));
  return 0;
}
int arks_comm_init(arks_ctx* ctx, int rank, int world, const void* unique_id, const uint32_t* shared, uint32_t n_shared) {
  if (!ctx || !unique_id || world < 1 || rank < 0 || rank >= world) return ARKS_E_INVALID_ARG;
  int rc = nccl_load(ctx);
  if (rc) return rc;
  CK(cudaSetDevice(ctx->device));
  NcclApi& a = *ctx->nccl;
  if (a.comm) { a.CommDestroy(a.comm); a.comm = nullptr; }
  ncclUniqueId id;
  memcpy(&id, unique_id, sizeof id);
  NCK(a.CommInitRank(&a.comm, world, id, rank));
  a.rank = rank; a.world = world;
  return arks_comm_set_shared(ctx, shared, n_shared);
}
int arks_fold_quota_allreduce(arks_ctx* ctx, int wait) {
  if (!ctx || !ctx->nccl || !ctx->nccl->comm) return fail(ctx, ARKS_E_INVALID_ARG, "arks_comm_init first");
  if (!ctx->loaded || !ctx->d_qdelta) return fail(ctx, ARKS_E_INVALID_ARG, "quota sharing is not enabled");
  NcclApi& a = *ctx->nccl;
  // local quota indices are positional in the generation they were given for: a swap since then may have moved or removed them
  if (a.generation != ctx->generation || (a.all_rows && a.n_shared != ctx->ht.n_quotas))
    return fail(ctx, ARKS_E_INVALID_ARG, "the tables changed since arks_comm_set_shared (generation %u, now %u): call it again", a.generation,
                ctx->generation);
  CK(cudaSetDevice(ctx->device));
  const size_t n_all = (size_t)3 * ctx->ht.n_quotas;
  if (!n_all) return 0;
  // everything below is ordered on the compute stream, between two batches
  CK(cudaMemcpyAsync(ctx->d_qexp, ctx->d_qdelta, n_all * 8, cudaMemcpyDeviceToDevice, ctx->stream));
  if (a.n_shared) {
    gather_shared_kernel<<<(a.n_shared * 3 + 255) / 256, 256, 0, ctx->stream>>>(a.d_msg, ctx->d_qexp, a.d_idx, a.n_shared);
    NCK(a.AllReduce(a.d_msg, a.d_msg, (size_t)a.n_shared * 3, ncclInt64, ncclSum, a.comm, ctx->stream));
  }
  const size_t span = n_all > (size_t)a.n_shared * 3 ? n_all : (size_t)a.n_shared * 3;
  fold_shared_kernel<<<(unsigned)((span + 255) / 256), 256, 0, ctx->stream>>>(ctx->d_quota, ctx->d_qdelta, a.d_msg, ctx->d_qexp, a.d_idx,
                                                                              a.n_shared, n_all);
  ctx->launches += a.n_shared ? 2 : 1;
  ctx->qexp_valid = false;
  CK(cudaGetLastError());
  if (wait) CK(cudaStreamSynchronize(ctx->stream));
  return 0;
}
void arks_comm_destroy(arks_ctx* ctx) {
  if (!ctx || !ctx->nccl) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  NcclApi* a = ctx->nccl;
  if (a->comm) a->CommDestroy(a->comm);
  cudaFree(a->d_idx);
  cudaFree(a->d_msg);
  // the shared object stays loaded: other contexts (and torch) may be using it
  delete a;
  ctx->nccl = nullptr;
}

}  // extern "C"
