// arks_host.cc — see arks_host.h. Build: g++ -O2 -std=c++20 -shared -fPIC -pthread, linked against libarksgw.so
// (no CUDA headers or runtime needed here: the C ABI is the only thing this file knows about the device).
#include "arks_host.h"

// weak: the host links against any provider of the C ABI, and one without the report (a CPU stand-in) leaves it null
extern "C" int arks_set_ratelimit_report(arks_ctx* ctx, int on) __attribute__((weak));
extern "C" int arks_set_sliding_window(arks_ctx* ctx, int on) __attribute__((weak));

#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <thread>

namespace arks_host {

namespace {

constexpr uint8_t kReasonHostError = 255;
constexpr int kSlots = 4;           // staging slots of the library: batches in flight on the device
constexpr int kBlocks = kSlots + 3; // host staging blocks per kind: in flight + open (two for responses) + one being handed back

// rows start on 32-byte boundaries: the ABI asks for 16, the library reads 32-aligned bodies a whole 32-byte sector at a time
inline size_t align16(size_t x) { return (x + 31) & ~size_t(31); }

template <class T>
T* pinned(size_t n) {  // page-locked so the library's cudaMemcpyAsync is a real DMA; falls back to pageable memory
  void* p = arks_alloc_pinned(n * sizeof(T) + 64);
  if (!p) p = aligned_alloc(64, (n * sizeof(T) + 127) & ~size_t(63));
  return static_cast<T*>(p);
}

// One staging block. Rows are reserved WITHOUT the batcher mutex: the open block's fill level lives in one 64-bit word
//   [63] closed | [62:41] token bytes | [40:14] body bytes / 16 | [13:0] rows
// that every arriving row advances with a compare-and-swap; the dispatcher ends the block by setting the closed bit (the
// value it gets back is the final fill level). A block that is not the open one always has the bit set, so a stale
// pointer can never reserve into a block that is queued on the device or back in the pool. Owners then copy their bytes
// in and bump `filled`. (A mutex here serialises the producers on lock hand-overs.)
constexpr uint64_t kClosed = 1ull << 63;
constexpr uint32_t kMaxRows = (1u << 14) - 1;
inline uint32_t st_rows(uint64_t s) { return (uint32_t)(s & 0x3fff); }
inline size_t st_bytes(uint64_t s) { return (size_t)((s >> 14) & 0x7ffffff) << 4; }
inline size_t st_tok(uint64_t s) { return (size_t)((s >> 41) & 0x3fffff); }
inline uint64_t st_add(size_t body16, size_t tok) { return 1ull + ((uint64_t)(body16 >> 4) << 14) + ((uint64_t)tok << 41); }
struct Block {
  std::atomic<uint64_t> state{kClosed};
  uint8_t* bodies = nullptr;
  uint32_t *body_off = nullptr, *body_len = nullptr;
  uint8_t* tokens = nullptr;      // requests
  uint32_t* token_off = nullptr;  // n + 1: entry r is written by the OWNER of row r (entry n by the dispatcher)
  uint8_t* tok_len = nullptr;     // n: length of row r's token (<= 255), written by its owner
  uint64_t* rnd = nullptr;
  int32_t* qos = nullptr;         // responses
  uint32_t* gen = nullptr;
  uint32_t* pre = nullptr;        // N4: the request phase's estimate of each row's stream
  uint8_t* flags = nullptr;
  // per-row completion
  RequestCallback* rcb = nullptr;
  ResponseCallback* pcb = nullptr;
  void** user = nullptr;
  // results
  uint8_t *reason = nullptr, *detail = nullptr, *rflags = nullptr, *counted = nullptr;
  int32_t *rqos = nullptr, *rtoken = nullptr, *rpick = nullptr;
  int64_t *cur_usage = nullptr, *limit_max = nullptr, *usage = nullptr;
  uint32_t *model_off = nullptr, *model_len = nullptr, *bpe = nullptr;
  uint8_t* rl_entry = nullptr;  // 2 per row: the rate-limit report (arks_set_ratelimit_report)
  int64_t *rl_limit = nullptr, *rl_remaining = nullptr;
  uint32_t *rl_reset = nullptr, *rl_retry = nullptr;  // 2 and 1 per row: the sliding window's times (arks_set_sliding_window)
  // bookkeeping
  uint32_t n = 0;
  size_t bytes = 0, tok_bytes = 0;
  std::atomic<uint32_t> filled{0};  // rows whose owner finished copying
  std::atomic<uint8_t>* ready = nullptr;  // per row: its owner finished copying (what a cut looks at when `filled` lags)
  uint32_t cut = 0;        // rows below this index have been put into segments (dispatcher only)
  uint32_t delivered = 0;  // rows whose decision was handed over; the block goes back to the pool at n
};
// rows [lo, hi) of a closed block: what one submission carries. A block is normally one segment; when an owner is late with
// its copy (the OS took its core away between reserving the row and filling it) the rows around it go ahead without it.
struct Seg {
  Block* b = nullptr;
  uint32_t lo = 0, hi = 0;
};

struct InFlight {
  Seg req;  // either may be empty (b == nullptr)
  Seg resp;
  int slot;
  int rc_req, rc_resp;
  uint64_t cycle;
  int64_t now;
  uint32_t gen;
};

// what a blocking call parks on
struct Parked {
  std::atomic<uint32_t> ready{0};
  RequestDecision rd{};
  ResponseDecision pd{};
};
void wake_request(void* user, const RequestDecision& d) {
  Parked* p = static_cast<Parked*>(user);
  p->rd = d;
  p->ready.store(1, std::memory_order_release);
  p->ready.notify_one();
}
void wake_response(void* user, const ResponseDecision& d) {
  Parked* p = static_cast<Parked*>(user);
  p->pd = d;
  p->ready.store(1, std::memory_order_release);
  p->ready.notify_one();
}

}  // namespace

// TEST HOOK (ARKS_HOST_TEST_STALL="<row>:<microseconds>:<every>"): the owner of that row of every <every>-th request block
// sleeps between reserving the row and filling it — what an owner that lost its core looks like to the dispatcher
static const char* g_test_stall_env = getenv("ARKS_HOST_TEST_STALL");
static void test_stall(const char* e, uint32_t row) {
  static std::atomic<uint32_t> seen{0};
  const uint32_t r = (uint32_t)strtoul(e, nullptr, 10);
  const char* c = strchr(e, ':');
  if (row != r || !c) return;
  const unsigned long us = strtoul(c + 1, nullptr, 10);
  const char* c2 = strchr(c + 1, ':');
  const uint32_t every = c2 ? (uint32_t)strtoul(c2 + 1, nullptr, 10) : 1;
  if (seen.fetch_add(1) % (every ? every : 1) == 0) std::this_thread::sleep_for(std::chrono::microseconds(us));
}

struct Batcher::Impl {
  arks_ctx* ctx;
  BatcherOptions opt;
  size_t tok_cap;
  Block req_blk[kBlocks], resp_blk[kBlocks];
  std::vector<Block*> free_req, free_resp;  // blocks nobody uses
  std::atomic<Block*> open_req{nullptr};
  std::atomic<Block*> open_resp[2] = {nullptr, nullptr};  // complete bodies / SSE chunks: kept apart so that every batch is homogeneous
                                             // (the library has faster kernels for all-JSON and all-SSE batches)
  int resp_turn = 0;
  // closed blocks that are not fully submitted yet: segments ready to go and rows whose owner is late, per kind
  // (0 requests, 1 complete response bodies, 2 SSE chunks)
  std::deque<Seg> pending[3];
  std::vector<Seg> late[3];  // one-row segments waiting for their owner
  std::deque<InFlight> inflight;            // submitted, not completed (FIFO == device order)
  bool slot_busy[kSlots] = {false, false, false, false};
  mutable std::mutex mu;
  std::mutex cfg_mu;  // config calls among themselves
  NameBook names;     // generation -> names (published under cfg_mu, read by any stream thread)
  std::atomic<bool> precharge{false};  // N4: response batches carry the streams' estimates
  std::atomic<bool> rl_report{false};  // request decisions carry the rate-limit report
  std::atomic<bool> sliding{false};    // the limiter runs the sliding window
  int swap_in(arks_prepared* p);
  int publish(arks_prepared* p, const NameTables* nm);
  std::condition_variable cv_work, cv_space, cv_done;
  bool stop = false;
  bool cycling = false;  // a cycle is being run (by the dispatcher thread or by a leading caller): one submitter at a time
  uint64_t cycle = 0;
  int64_t (*clock)(void*) = nullptr;
  void* clock_arg = nullptr;
  BatcherStats st{};
  std::thread dispatcher, completer;

  bool submit_request(std::string_view token, std::string_view body, uint64_t pick_rand, RequestCallback cb, void* user, bool can_lead);
  bool submit_response(int32_t qos, uint32_t gen, std::string_view body, uint8_t flags, ResponseCallback cb, void* user, bool can_lead,
                       uint32_t precharged);
  int64_t last_now = INT64_MIN;  // batches never carry an earlier clock reading than their predecessor
  std::vector<uint32_t> seg_token_off;  // dispatcher only: the token CSR of a segment (see the request submit)

  void alloc(Block& b, bool is_req) {
    const uint32_t m = opt.max_batch;
    b.bodies = pinned<uint8_t>(opt.max_bytes + 16);
    b.body_off = pinned<uint32_t>(m);
    b.body_len = pinned<uint32_t>(m);
    b.user = new void*[m];
    b.ready = new std::atomic<uint8_t>[m];
    for (uint32_t i = 0; i < m; i++) b.ready[i].store(0, std::memory_order_relaxed);
    if (is_req) {
      b.tokens = pinned<uint8_t>(tok_cap);
      b.token_off = pinned<uint32_t>(m + 1);
      b.tok_len = new uint8_t[m];
      b.rnd = pinned<uint64_t>(m);
      b.rcb = new RequestCallback[m];
      b.reason = new uint8_t[m]; b.detail = new uint8_t[m]; b.rflags = new uint8_t[m];
      b.rqos = new int32_t[m]; b.rtoken = new int32_t[m]; b.rpick = new int32_t[m];
      b.cur_usage = new int64_t[m]; b.limit_max = new int64_t[m];
      b.model_off = new uint32_t[m]; b.model_len = new uint32_t[m]; b.bpe = new uint32_t[m];
      b.rl_entry = new uint8_t[2 * (size_t)m]; b.rl_limit = new int64_t[2 * (size_t)m]; b.rl_remaining = new int64_t[2 * (size_t)m];
      b.rl_reset = new uint32_t[2 * (size_t)m]; b.rl_retry = new uint32_t[m];
    } else {
      b.qos = pinned<int32_t>(m);
      b.gen = pinned<uint32_t>(m);
      b.pre = pinned<uint32_t>(m);
      b.flags = pinned<uint8_t>(m);
      b.pcb = new ResponseCallback[m];
      b.reason = new uint8_t[m]; b.counted = new uint8_t[m]; b.usage = new int64_t[3 * (size_t)m];
    }
  }

  // Reserve one row in the open block of `open` (see Block). Returns false only when the batcher is shutting down.
  bool reserve(std::atomic<Block*>& open, size_t need, size_t tok, Block** out, uint32_t* row, size_t* off, size_t* toff) {
    for (unsigned spins = 0;; spins++) {
      Block* b = open.load(std::memory_order_acquire);
      uint64_t s = b->state.load(std::memory_order_relaxed);
      bool full = false;
      while (!(s & kClosed)) {
        if (st_rows(s) >= opt.max_batch || st_bytes(s) + need > opt.max_bytes || st_tok(s) + tok > tok_cap) { full = true; break; }
        if (b->state.compare_exchange_weak(s, s + st_add(need, tok), std::memory_order_acq_rel, std::memory_order_relaxed)) {
          *out = b; *row = st_rows(s); *off = st_bytes(s); *toff = st_tok(s);
          return true;
        }
      }
      if (full) {  // wait for the dispatcher to swap the block
        std::unique_lock<std::mutex> lk(mu);
        if (stop) return false;
        cv_work.notify_one();
        cv_space.wait_for(lk, std::chrono::microseconds(50));
      } else if (spins > 64) {
        std::this_thread::yield();  // closed: the new open block is published before the bit is set, one reload finds it
      }
    }
  }
  // What the first row of a block owes the batcher: wake the dispatcher — or, for a blocking caller that finds the batcher
  // idle, become the cycle's leader. Taking the mutex also orders this arrival against a dispatcher that is just about
  // to sleep on cv_work (it evaluates has_work() under the same mutex).
  bool first_row(bool can_lead) {
    bool lead;
    {
      std::lock_guard<std::mutex> g(mu);
      lead = can_lead && may_lead();
      if (lead) cycling = true;
    }
    if (!lead) cv_work.notify_one();
    return lead;
  }

  // How long a closed block waits for its row owners before the rows that ARE filled go ahead without the late ones. A
  // copy takes well under a microsecond; an owner that is later than this lost its core (preempted, or the whole group
  // throttled by a CPU quota) and may be gone for milliseconds.
  static constexpr int64_t kFillGraceNs = 15000;
  // give the owners of a freshly closed block their grace (no lock held: they never take it)
  void wait_grace(Block* b) {
    if (b->filled.load(std::memory_order_acquire) == b->n) return;
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
      if (b->filled.load(std::memory_order_acquire) == b->n) break;
      const int64_t waited = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
      if (waited > kFillGraceNs) break;
      std::this_thread::yield();
    }
    note(t_fill, 4, (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count());
  }
  // Cut a closed block into segments of filled rows (pending[k]) and late rows (late[k]). Lock held.
  void cut_block(Block* b, int k) {
    if (b->filled.load(std::memory_order_acquire) == b->n) {
      pending[k].push_back(Seg{b, 0, b->n});
      b->cut = b->n;
      return;
    }
    uint32_t lo = 0;
    for (uint32_t i = 0; i <= b->n; i++) {
      const bool ok = i < b->n && b->ready[i].load(std::memory_order_acquire);
      if (!ok) {
        if (i > lo) pending[k].push_back(Seg{b, lo, i});
        if (i < b->n) { late[k].push_back(Seg{b, i, i + 1}); st_late_rows.fetch_add(1, std::memory_order_relaxed); }
        lo = i + 1;
      }
    }
    b->cut = b->n;
  }
  // late rows whose owner has arrived become one-row segments
  void collect_late(int k) {
    for (size_t j = 0; j < late[k].size();) {
      if (late[k][j].b->ready[late[k][j].lo].load(std::memory_order_acquire)) {
        pending[k].push_back(late[k][j]);
        late[k][j] = late[k].back();
        late[k].pop_back();
      } else {
        j++;
      }
    }
  }
  std::atomic<uint64_t> st_late_rows{0};
  int free_slot() const {  // -1 while max_inflight batches are already queued on the device
    int busy = 0, first = -1;
    for (int k = 0; k < kSlots; k++) {
      if (slot_busy[k]) busy++;
      else if (first < 0) first = k;
    }
    return busy < (int)opt.max_inflight ? first : -1;
  }

  static uint32_t rows_of(const std::atomic<Block*>& b) { return st_rows(b.load(std::memory_order_acquire)->state.load(std::memory_order_acquire)); }
  bool waiting(int k) const { return !pending[k].empty() || !late[k].empty(); }
  bool has_work() const {
    return rows_of(open_req) || rows_of(open_resp[0]) || rows_of(open_resp[1]) || waiting(0) || waiting(1) || waiting(2);
  }
  // end the open block: a fresh one is published first (arrivals that lose the race go there), then the closed bit freezes
  // the fill level of the old one. Lock held.
  Block* close_open(std::atomic<Block*>& open, std::vector<Block*>& pool) {
    Block* b = open.load(std::memory_order_relaxed);
    Block* nb = pool.back();
    pool.pop_back();
    nb->state.store(0, std::memory_order_release);
    open.store(nb, std::memory_order_release);
    const uint64_t s = b->state.fetch_or(kClosed, std::memory_order_acq_rel);
    b->n = st_rows(s);
    b->bytes = st_bytes(s);
    b->tok_bytes = st_tok(s);
    return b;
  }
  // Closing an open block needs a fresh one from the pool; segments and late rows of blocks that are already closed do not —
  // and they must keep moving when the pool is empty, or the blocks they belong to would never come back to it.
  bool can_cycle() const {
    if (cycling || free_slot() < 0) return false;
    if (waiting(0) || waiting(1) || waiting(2)) return true;
    return (rows_of(open_req) || rows_of(open_resp[0]) || rows_of(open_resp[1])) && !free_req.empty() && !free_resp.empty();
  }

  // One cycle: close the open blocks and queue them on the device (asynchronous submits, one staging slot). Entered
  // and left with `lk` held and `cycling` set by the caller; the lock is dropped while the device is being talked to.
  // With one batch in flight the cycle also waits for the batch and hands every row its decision.
  void run_cycle(std::unique_lock<std::mutex>& lk) {
    InFlight f{Seg{}, Seg{}, free_slot(), 0, 0, 0, 0, 0};
    slot_busy[f.slot] = true;
    // what is already cut goes first (order of arrival); otherwise the open block is closed now
    // (late rows do not hold the open block back: only segments that are ready to go are ahead of it)
    Block* fresh_req = pending[0].empty() && rows_of(open_req) && !free_req.empty() ? close_open(open_req, free_req) : nullptr;
    // one response batch per cycle (a staging slot holds one): alternate when both kinds are waiting
    const bool has0 = waiting(1) || rows_of(open_resp[0]), has1 = waiting(2) || rows_of(open_resp[1]);
    const int kind = has0 && has1 ? (resp_turn ^= 1) : (has1 ? 1 : 0);
    Block* fresh_resp = pending[1 + kind].empty() && rows_of(open_resp[kind]) && !free_resp.empty() ? close_open(open_resp[kind], free_resp) : nullptr;
    f.cycle = cycle++;
    const auto prev_end = last_cycle_end;  // (statistics; read under the lock: the completion thread writes them)
    const bool prev_work = last_had_work;
    int64_t now = clock ? clock(clock_arg) : (int64_t)time(nullptr);
    // a wall clock that steps back (NTP) must not fail the batch (ARKS_E_TIME_WENT_BACK fails every row of it): the
    // limiter's windows only move forward, like Redis keys that already exist
    if (now < last_now) now = last_now;
    last_now = now;
    f.now = now;
    lk.unlock();
    cv_space.notify_all();
    const auto t_a = std::chrono::steady_clock::now();
    if (fresh_req) wait_grace(fresh_req);
    if (fresh_resp) wait_grace(fresh_resp);
    lk.lock();  // the segment lists are read by has_work() under the lock
    if (fresh_req) { fresh_req->token_off[fresh_req->n] = (uint32_t)fresh_req->tok_bytes; cut_block(fresh_req, 0); }
    if (fresh_resp) cut_block(fresh_resp, 1 + kind);
    collect_late(0);
    collect_late(1 + kind);
    if (!pending[0].empty()) { f.req = pending[0].front(); pending[0].pop_front(); }
    if (!pending[1 + kind].empty()) { f.resp = pending[1 + kind].front(); pending[1 + kind].pop_front(); }
    if (!f.req.b && !f.resp.b) {  // only late rows are left and their owners are still away
      slot_busy[f.slot] = false;
      lk.unlock();
      std::this_thread::sleep_for(std::chrono::microseconds(5));
      lk.lock();
      return;
    }
    lk.unlock();
    arks_select_slot(ctx, f.slot);
    f.gen = arks_table_generation(ctx);  // LoadTables only runs between cycles: this is the batch's generation
    auto span_end = [](const Block& b, uint32_t hi) { return (size_t)b.body_off[hi - 1] + align16(b.body_len[hi - 1]); };
    if (f.req.b) {
      Block& b = *f.req.b;
      const uint32_t lo = f.req.lo, n = f.req.hi - lo;
      arks_request_batch rb{};
      rb.n = n; rb.bodies = b.bodies; rb.body_off = b.body_off + lo; rb.body_len = b.body_len + lo;
      rb.bodies_bytes = span_end(b, f.req.hi);  // offsets stay relative to the block: rows in front of a segment ride along
      rb.tokens = b.tokens; rb.pick_rand = b.rnd + lo; rb.now_unix = now;
      if (lo == 0 && f.req.hi == b.n) {
        rb.token_off = b.token_off;  // the whole block: every entry is written (the last one by the dispatcher when it closed it)
      } else {
        // A segment: entry `hi` of the block's CSR belongs to the row BEHIND the segment, whose owner may have reserved it and
        // not written a byte yet (that is why the block was cut). The end of the segment's last token is its own start + length.
        seg_token_off.resize((size_t)n + 1);
        memcpy(seg_token_off.data(), b.token_off + lo, (size_t)n * 4);
        seg_token_off[n] = b.token_off[f.req.hi - 1] + b.tok_len[f.req.hi - 1];
        rb.token_off = seg_token_off.data();  // copied by the library before arks_submit_request_async returns
      }
      f.rc_req = arks_submit_request_async(ctx, &rb);
    }
    if (f.resp.b) {
      Block& b = *f.resp.b;
      const uint32_t lo = f.resp.lo, n = f.resp.hi - lo;
      arks_response_batch rb{};
      rb.n = n; rb.bodies = b.bodies; rb.body_off = b.body_off + lo; rb.body_len = b.body_len + lo;
      rb.bodies_bytes = span_end(b, f.resp.hi);
      rb.qos = b.qos + lo; rb.flags = b.flags + lo; rb.now_unix = now; rb.gen = b.gen + lo;
      rb.precharged = precharge.load(std::memory_order_relaxed) ? b.pre + lo : nullptr;
      f.rc_resp = arks_submit_response_async(ctx, &rb);
    }
    const auto t_b = std::chrono::steady_clock::now();
    note(t_submit, 0, (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t_b - t_a).count());
    if (prev_end.time_since_epoch().count() && prev_work && t_a > prev_end)
      note(t_gap, 3, (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t_a - prev_end).count());
    if (opt.max_inflight == 1) {  // nothing else can be queued meanwhile: finish the batch here, one thread hand-off less
      deliver(f);
      lk.lock();
      recycle(f);
      return;
    }
    lk.lock();
    inflight.push_back(f);
    cv_done.notify_one();
  }

  // Thread 1: runs the cycles nobody else runs (see lead_cycle).
  void dispatch_loop() {
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
      cv_work.wait(lk, [&] { return (stop && !cycling) || can_cycle(); });
      if (!can_cycle()) {
        if (stop && !has_work()) return;
        continue;
      }
      cycling = true;
      if (opt.linger_us) {  // give concurrent streams a moment to join the cycle
        lk.unlock();
        std::this_thread::sleep_for(std::chrono::microseconds(opt.linger_us));
        lk.lock();
      }
      run_cycle(lk);
      cycling = false;
    }
  }
  // A blocked caller that finds the batcher idle runs the cycle for its own row itself: on a quiet system a request
  // then costs no thread hand-off at all (caller -> dispatcher -> caller otherwise). Lock held on entry and exit.
  bool may_lead() const { return opt.max_inflight == 1 && opt.linger_us == 0 && !cycling && free_slot() >= 0 && !free_req.empty() && !free_resp.empty(); }
  void lead_cycle(std::unique_lock<std::mutex>& lk) {
    run_cycle(lk);
    cycling = false;
    if (has_work()) cv_work.notify_one();
  }

  // Thread 2: waits for the oldest batch, hands every row its decision, recycles block and slot.
  void complete_loop() {
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
      cv_done.wait(lk, [&] { return !inflight.empty() || (stop && !has_work()); });
      if (inflight.empty()) {
        bool busy = false;
        for (int k = 0; k < kSlots; k++) busy |= slot_busy[k];
        if (!busy) return;  // stop requested, nothing queued, nothing being submitted
        cv_done.wait_for(lk, std::chrono::milliseconds(1));
        continue;
      }
      InFlight f = inflight.front();
      inflight.pop_front();
      lk.unlock();
      deliver(f);
      lk.lock();
      recycle(f);
    }
  }

  std::atomic<uint64_t> t_submit{0}, t_device{0}, t_deliver{0}, t_gap{0};
  std::atomic<uint64_t> t_max[5] = {}, t_slow[5] = {};  // submit, device, deliver, gap, fill
  std::atomic<uint64_t> t_fill{0};
  std::chrono::steady_clock::time_point last_cycle_end{};
  bool last_had_work = false;
  void note(std::atomic<uint64_t>& acc, int k, uint64_t ns) {
    acc.fetch_add(ns, std::memory_order_relaxed);
    if (ns > t_max[k].load(std::memory_order_relaxed)) t_max[k].store(ns, std::memory_order_relaxed);
    if (ns > 100000) t_slow[k].fetch_add(1, std::memory_order_relaxed);
  }
  // wait for a submitted batch and hand every row its decision (no lock held)
  void deliver(InFlight& f) {
    auto t0 = std::chrono::steady_clock::now();
    auto lap = [&](std::atomic<uint64_t>& acc) {
      const auto t1 = std::chrono::steady_clock::now();
      note(acc, &acc == &t_device ? 1 : 2, (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(t1 - t0).count());
      t0 = t1;
    };
    if (f.req.b) {
      Block& b = *f.req.b;
      const uint32_t lo = f.req.lo, hi = f.req.hi;
      int rc = f.rc_req;
      if (rc == 0) {
        // a batch run without the rate-limit report leaves these arrays as they are: no figures
        memset(b.rl_entry + 2 * (size_t)lo, ARKS_RL_NONE, 2 * (size_t)(hi - lo));
        memset(b.rl_retry + lo, 0xFF, 4 * (size_t)(hi - lo));  // ... and these without the sliding window (no time is 2^32 - 1 s)
        arks_request_result rr{b.reason + lo, b.detail + lo, b.rflags + lo, b.rqos + lo, b.rtoken + lo, b.rpick + lo, b.cur_usage + lo,
                               b.limit_max + lo, b.model_off + lo, b.model_len + lo, b.bpe + lo, b.rl_entry + 2 * (size_t)lo,
                               b.rl_limit + 2 * (size_t)lo, b.rl_remaining + 2 * (size_t)lo, b.rl_reset + 2 * (size_t)lo,
                               b.rl_retry + lo};
        rc = arks_wait_request(ctx, f.slot, &rr);
      }
      lap(t_device);
      for (uint32_t i = lo; i < hi; i++) {
        RequestDecision d{};
        d.rl_entry[0] = d.rl_entry[1] = ARKS_RL_NONE;
        if (rc) d.reason = kReasonHostError;
        else {
          d.reason = b.reason[i]; d.detail = b.detail[i]; d.flags = b.rflags[i];
          d.qos = b.rqos[i]; d.token = b.rtoken[i]; d.pick = b.rpick[i];
          d.cur_usage = b.cur_usage[i]; d.limit_max = b.limit_max[i];
          d.model_off = b.model_off[i]; d.model_len = b.model_len[i]; d.bpe_count = b.bpe[i];
          for (int t = 0; t < 2; t++) {
            d.rl_entry[t] = b.rl_entry[2 * (size_t)i + t];
            d.rl_limit[t] = b.rl_limit[2 * (size_t)i + t];
            d.rl_remaining[t] = b.rl_remaining[2 * (size_t)i + t];
          }
          if (b.rl_retry[i] != 0xFFFFFFFFu) {
            d.rl_sliding = 1;
            d.rl_reset[0] = b.rl_reset[2 * (size_t)i];
            d.rl_reset[1] = b.rl_reset[2 * (size_t)i + 1];
            d.rl_retry = b.rl_retry[i];
          }
        }
        d.cycle = f.cycle; d.index = i - lo; d.now_unix = f.now; d.gen = f.gen;
        b.rcb[i](b.user[i], d);
      }
      lap(t_deliver);
    }
    if (f.resp.b) {
      Block& b = *f.resp.b;
      const uint32_t lo = f.resp.lo, hi = f.resp.hi;
      int rc = f.rc_resp;
      if (rc == 0) {
        arks_response_result rr{b.reason + lo, b.counted + lo, b.usage + 3 * (size_t)lo, nullptr};  // no completion BPE count wanted
        rc = arks_wait_response(ctx, f.slot, &rr);
      }
      lap(t_device);
      for (uint32_t i = lo; i < hi; i++) {
        ResponseDecision d{};
        if (rc) d.reason = kReasonHostError;
        else {
          d.reason = b.reason[i]; d.counted = b.counted[i];
          for (int k = 0; k < 3; k++) d.usage[k] = b.usage[3 * (size_t)i + k];
        }
        d.cycle = f.cycle; d.index = i - lo; d.now_unix = f.now;
        b.pcb[i](b.user[i], d);
      }
      lap(t_deliver);
    }
  }
  // stats, slot and — once every row of a block has its decision — the block back to the pools (lock held)
  void retire(Seg& g, std::vector<Block*>& pool) {
    Block* b = g.b;
    b->delivered += g.hi - g.lo;
    if (b->delivered != b->n || b->cut != b->n) return;  // other segments / late rows of the block are still on their way
    for (uint32_t i = 0; i < b->n; i++) b->ready[i].store(0, std::memory_order_relaxed);
    b->n = 0; b->bytes = 0; b->tok_bytes = 0; b->cut = 0; b->delivered = 0;
    b->filled.store(0, std::memory_order_relaxed);
    b->state.store(kClosed, std::memory_order_release);
    pool.push_back(b);
  }
  void recycle(InFlight& f) {
    st.cycles++;
    last_cycle_end = std::chrono::steady_clock::now();
    last_had_work = has_work();
    if (f.req.b) {
      const uint32_t n = f.req.hi - f.req.lo;
      st.request_batches++; st.requests += n;
      if (n > st.max_request_batch) st.max_request_batch = n;
      retire(f.req, free_req);
    }
    if (f.resp.b) {
      const uint32_t n = f.resp.hi - f.resp.lo;
      st.response_batches++; st.responses += n;
      if (n > st.max_response_batch) st.max_response_batch = n;
      retire(f.resp, free_resp);
    }
    slot_busy[f.slot] = false;
    cv_work.notify_one();
  }
};

Batcher::Batcher(arks_ctx* ctx, const BatcherOptions& opt) : p_(new Impl()) {
  p_->ctx = ctx;
  p_->opt = opt;
  if (p_->opt.max_batch > kMaxRows) p_->opt.max_batch = kMaxRows;  // the fill-level word has 14 bits of rows
  if (p_->opt.max_bytes > (size_t(1) << 30)) p_->opt.max_bytes = size_t(1) << 30;
  p_->tok_cap = (size_t)opt.max_batch * 256;
  for (int k = 0; k < kBlocks; k++) {
    p_->alloc(p_->req_blk[k], true);
    p_->alloc(p_->resp_blk[k], false);
    p_->free_req.push_back(&p_->req_blk[k]);
    p_->free_resp.push_back(&p_->resp_blk[k]);
  }
  p_->open_req = p_->free_req.back(); p_->free_req.pop_back();
  p_->open_req.load()->state.store(0);
  for (int k = 0; k < 2; k++) { p_->open_resp[k] = p_->free_resp.back(); p_->free_resp.pop_back(); p_->open_resp[k].load()->state.store(0); }
  p_->dispatcher = std::thread([this] { p_->dispatch_loop(); });
  if (opt.max_inflight > 1) p_->completer = std::thread([this] { p_->complete_loop(); });
}
Batcher::~Batcher() {
  {
    std::lock_guard<std::mutex> g(p_->mu);
    p_->stop = true;
  }
  p_->cv_work.notify_all();
  p_->dispatcher.join();
  p_->cv_done.notify_all();
  if (p_->completer.joinable()) p_->completer.join();
  delete p_;  // staging blocks are left to the process (pinned host memory of a long-lived server object)
}
void Batcher::SetClock(int64_t (*clock)(void*), void* arg) {
  std::lock_guard<std::mutex> g(p_->mu);
  p_->clock = clock;
  p_->clock_arg = arg;
}
void Batcher::ResetTailStats() {
  for (int k = 0; k < 5; k++) { p_->t_max[k].store(0); p_->t_slow[k].store(0); }
}
BatcherStats Batcher::Stats() const {
  std::lock_guard<std::mutex> g(p_->mu);
  BatcherStats s = p_->st;
  s.ns_submit = p_->t_submit.load();
  s.ns_device = p_->t_device.load();
  s.ns_deliver = p_->t_deliver.load();
  s.max_ns_submit = p_->t_max[0].load(); s.max_ns_device = p_->t_max[1].load(); s.max_ns_deliver = p_->t_max[2].load(); s.max_ns_gap = p_->t_max[3].load();
  s.slow_submit = p_->t_slow[0].load(); s.slow_device = p_->t_slow[1].load(); s.slow_deliver = p_->t_slow[2].load(); s.slow_gap = p_->t_slow[3].load();
  s.ns_fill = p_->t_fill.load(); s.max_ns_fill = p_->t_max[4].load(); s.slow_fill = p_->t_slow[4].load();
  s.late_rows = p_->st_late_rows.load();
  return s;
}

bool Batcher::Impl::submit_request(std::string_view token, std::string_view body, uint64_t pick_rand, RequestCallback cb, void* user,
                                   bool can_lead) {
  Impl& I = *this;
  const size_t need = align16(body.size());
  if (need > I.opt.max_bytes || token.size() > 255) return false;
  Block* b;
  uint32_t row;
  size_t off, toff;
  if (!I.reserve(I.open_req, need, token.size(), &b, &row, &off, &toff)) return false;
  if (const char* e = g_test_stall_env) test_stall(e, row);  // the worst moment to lose the core: the row is reserved, nothing of it is written
  b->body_off[row] = (uint32_t)off;
  b->body_len[row] = (uint32_t)body.size();
  b->token_off[row] = (uint32_t)toff;
  b->tok_len[row] = (uint8_t)token.size();
  b->rnd[row] = pick_rand;
  b->rcb[row] = cb;
  b->user[row] = user;
  const bool lead = row == 0 && I.first_row(can_lead);
  memcpy(b->bodies + off, body.data(), body.size());
  memset(b->bodies + off + body.size(), 0, need - body.size());
  memcpy(b->tokens + toff, token.data(), token.size());
  b->ready[row].store(1, std::memory_order_release);
  b->filled.fetch_add(1, std::memory_order_release);
  if (lead) {
    std::unique_lock<std::mutex> lk(I.mu);
    I.lead_cycle(lk);
  }
  return true;
}

bool Batcher::Impl::submit_response(int32_t qos, uint32_t gen, std::string_view body, uint8_t flags, ResponseCallback cb, void* user,
                                    bool can_lead, uint32_t precharged) {
  Impl& I = *this;
  const size_t need = align16(body.size());
  if (need > I.opt.max_bytes) return false;
  Block* b;
  uint32_t row;
  size_t off, toff;
  if (!I.reserve(I.open_resp[(flags & ARKS_RESP_STREAM) ? 1 : 0], need, 0, &b, &row, &off, &toff)) return false;
  b->body_off[row] = (uint32_t)off;
  b->body_len[row] = (uint32_t)body.size();
  b->qos[row] = qos;
  b->gen[row] = gen;
  b->pre[row] = precharged;
  b->flags[row] = flags;
  b->pcb[row] = cb;
  b->user[row] = user;
  const bool lead = row == 0 && I.first_row(can_lead);
  memcpy(b->bodies + off, body.data(), body.size());
  memset(b->bodies + off + body.size(), 0, need - body.size());
  b->ready[row].store(1, std::memory_order_release);
  b->filled.fetch_add(1, std::memory_order_release);
  if (lead) {
    std::unique_lock<std::mutex> lk(I.mu);
    I.lead_cycle(lk);
  }
  return true;
}

bool Batcher::SubmitRequest(std::string_view token, std::string_view body, uint64_t pick_rand, RequestCallback cb, void* user) {
  return p_->submit_request(token, body, pick_rand, cb, user, false);
}
bool Batcher::SubmitResponse(int32_t qos, uint32_t gen, std::string_view body, uint8_t flags, ResponseCallback cb, void* user, uint32_t precharged) {
  return p_->submit_response(qos, gen, body, flags, cb, user, false, precharged);
}
uint32_t Batcher::Generation() const { return arks_table_generation(p_->ctx); }
int Batcher::SetPrecharge(bool on) {
  const int rc = arks_set_precharge(p_->ctx, on ? 1 : 0);
  if (!rc) p_->precharge.store(on, std::memory_order_relaxed);
  return rc;
}
bool Batcher::Precharge() const { return p_->precharge.load(std::memory_order_relaxed); }
int Batcher::SetRatelimitReport(bool on) {
  if (!arks_set_ratelimit_report) return ARKS_E_NOT_LOADED;  // a provider of the C ABI without the report
  const int rc = arks_set_ratelimit_report(p_->ctx, on ? 1 : 0);
  if (!rc) p_->rl_report.store(on, std::memory_order_relaxed);
  return rc;
}
bool Batcher::RatelimitReport() const { return p_->rl_report.load(std::memory_order_relaxed); }
int Batcher::SetSlidingWindow(bool on) {
  if (!arks_set_sliding_window) return ARKS_E_NOT_LOADED;  // a provider of the C ABI without the sliding window
  const int rc = arks_set_sliding_window(p_->ctx, on ? 1 : 0);
  if (!rc) p_->sliding.store(on, std::memory_order_relaxed);
  return rc;
}
bool Batcher::SlidingWindow() const { return p_->sliding.load(std::memory_order_relaxed); }
// config calls are serialised among themselves; the swap itself happens between two cycles
int Batcher::LoadTables(const arks_tables* t, const NameTables* names) {
  Impl& I = *p_;
  std::lock_guard<std::mutex> one(I.cfg_mu);
  arks_prepared* p = nullptr;
  int rc = arks_prepare_tables(I.ctx, t, &p);  // batches keep cycling meanwhile
  return rc ? rc : I.publish(p, names);
}
int Batcher::ApplyConfig(const NameTables* names) {
  Impl& I = *p_;
  std::lock_guard<std::mutex> one(I.cfg_mu);
  arks_prepared* p = nullptr;
  int rc = arks_config_prepare(I.ctx, &p);
  return rc ? rc : I.publish(p, names);
}
NameBook& Batcher::Names() { return p_->names; }
// under cfg_mu: a commit raises the generation by one, and nobody else commits meanwhile, so the names can be in the book
// under their number before the first decision of that generation exists
int Batcher::Impl::publish(arks_prepared* p, const NameTables* nm) {
  const uint32_t next = arks_table_generation(ctx) + 1;
  if (nm) names.Publish(next, *nm);
  const int rc = swap_in(p);
  if (rc && nm) names.Drop(next);
  return rc;
}
arks_ctx* Batcher::Context() const { return p_->ctx; }
int Batcher::Impl::swap_in(arks_prepared* p) {
  Impl& I = *this;
  std::unique_lock<std::mutex> lk(I.mu);
  // become the one "cycle" in progress for the length of the commit: no submission interleaves with the pointer swap.
  // Batches already queued on the device are NOT waited for: the commit is ordered behind them on the stream.
  while (I.cycling) I.cv_space.wait_for(lk, std::chrono::microseconds(20));
  I.cycling = true;
  lk.unlock();
  const int rc = arks_commit_tables(I.ctx, p);
  if (rc) arks_discard_prepared(I.ctx, p);
  lk.lock();
  I.cycling = false;
  lk.unlock();
  I.cv_work.notify_all();
  I.cv_space.notify_all();
  return rc;
}

RequestDecision Batcher::HandleRequestBody(std::string_view token, std::string_view body, uint64_t pick_rand) {
  Parked p;
  if (!p_->submit_request(token, body, pick_rand, wake_request, &p, true)) {
    RequestDecision d{};
    d.reason = kReasonHostError;
    return d;
  }
  p.ready.wait(0, std::memory_order_acquire);  // futex sleep until the completion thread hands the decision over
  return p.rd;
}
ResponseDecision Batcher::HandleResponseBody(int32_t qos, uint32_t gen, std::string_view body, uint8_t flags, uint32_t precharged) {
  Parked p;
  if (!p_->submit_response(qos, gen, body, flags, wake_response, &p, true, precharged)) {
    ResponseDecision d{};
    d.reason = kReasonHostError;
    return d;
  }
  p.ready.wait(0, std::memory_order_acquire);
  return p.pd;
}

// ---- error shaping (A13) ---------------------------------------------------------------------------------------
int ReasonHttpStatus(uint8_t r) {
  switch (r) {
    case ARKS_R_OK: case ARKS_R_PENDING: case ARKS_R_QOS_GONE: return 200;
    case ARKS_R_NO_TOKEN: return 401;
    case ARKS_R_REQUEST_BODY: case ARKS_R_NO_MODEL: case ARKS_R_NO_MODEL_BACKENDS: case ARKS_R_STREAM_OPTIONS: return 400;
    case ARKS_R_RATE_LIMIT: case ARKS_R_QUOTA: return 429;
    default: return 500;
  }
}
const char* ReasonHeader(uint8_t r) {
  switch (r) {
    case ARKS_R_NO_TOKEN: case ARKS_R_TOKEN_NOT_FOUND: case ARKS_R_MODEL_NOT_IN_TOKEN: return "x-error-token";
    case ARKS_R_REQUEST_BODY: return "x-error-request-body-processing";
    case ARKS_R_NO_MODEL: return "x-error-no-model-in-request";
    case ARKS_R_NO_MODEL_BACKENDS: return "x-error-no-model-backends";
    case ARKS_R_STREAM_OPTIONS: return "x-error-no-stream-options-include-usage";
    case ARKS_R_RATE_LIMIT: return "x-error-rate-limit";
    case ARKS_R_QUOTA: case ARKS_R_QUOTA_CONFIG: case ARKS_R_QUOTA_CONFIG_RESP: return "x-error-quota";
    case ARKS_R_STREAMING: return "x-error-streaming";
    case ARKS_R_RESPONSE_UNMARSHAL: return "x-error-response-unmarshal";
    case ARKS_R_RESPONSE_UNKNOWN: return "x-error-response-unknown";
    default: return "x-error-response";
  }
}
// json-iterator ConfigFastest string encoding (EscapeHTML off): `"`, `\` and control bytes are escaped, the rest is raw
static std::string json_escape(std::string_view s) {
  std::string o;
  for (unsigned char c : s) {
    if (c == '"' || c == '\\') { o += '\\'; o += (char)c; }
    else if (c == '\n') o += "\\n";
    else if (c == '\r') o += "\\r";
    else if (c == '\t') o += "\\t";
    else if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; }
    else o += (char)c;
  }
  return o;
}
Action ErrorResponse(int status, std::vector<Header> headers, const std::string& message) {
  Action a;
  a.kind = Action::kImmediate;
  a.status = status;
  a.set_headers = std::move(headers);
  a.set_headers.push_back({"Content-Type", "application/json"});
  // generateErrorMessage marshals a map: Go does not fix the order of "message" and "code" (SURVEY.md §8a A13); this is
  // one of the two byte strings the reference produces
  a.body = "{\"error\":{\"message\":\"" + json_escape(message) + "\",\"code\":" + std::to_string(status) + "}}";
  return a;
}

// the string a raw JSON string span decodes to (jsoniter ReadString: surrogate pairs joined, lone surrogates -> U+FFFD)
std::string DecodeJsonString(std::string_view raw) {
  std::string o;
  auto put = [&](uint32_t r) {
    if (r > 0x10FFFF || (r >= 0xD800 && r <= 0xDFFF)) r = 0xFFFD;
    if (r <= 0x7F) o += (char)r;
    else if (r <= 0x7FF) { o += (char)(0xC0 | (r >> 6)); o += (char)(0x80 | (r & 0x3F)); }
    else if (r <= 0xFFFF) { o += (char)(0xE0 | (r >> 12)); o += (char)(0x80 | ((r >> 6) & 0x3F)); o += (char)(0x80 | (r & 0x3F)); }
    else { o += (char)(0xF0 | (r >> 18)); o += (char)(0x80 | ((r >> 12) & 0x3F)); o += (char)(0x80 | ((r >> 6) & 0x3F)); o += (char)(0x80 | (r & 0x3F)); }
  };
  auto hex4 = [&](size_t i) {
    uint32_t v = 0;
    for (size_t k = i; k < i + 4 && k < raw.size(); k++) {
      const unsigned char c = (unsigned char)raw[k];
      v = v * 16 + (c <= '9' ? c - '0' : (c | 0x20) - 'a' + 10);
    }
    return v;
  };
  size_t i = 0;
  while (i < raw.size()) {
    const char c = raw[i++];
    if (c != '\\' || i >= raw.size()) { o += c; continue; }
    char e = raw[i++];
    for (;;) {
      if (e != 'u') {
        o += e == 'b' ? '\b' : e == 'f' ? '\f' : e == 'n' ? '\n' : e == 'r' ? '\r' : e == 't' ? '\t' : e;
        break;
      }
      uint32_t r = hex4(i);
      i += 4;
      if (r < 0xD800 || r > 0xDFFF) { put(r); break; }
      if (i >= raw.size() || raw[i] != '\\') { put(r); break; }
      i++;
      e = i < raw.size() ? raw[i++] : '\\';
      if (e != 'u') { put(r); continue; }  // the next escape is decoded on its own
      const uint32_t r2 = hex4(i);
      i += 4;
      if (r < 0xDC00 && r2 >= 0xDC00 && r2 < 0xE000) put((((r - 0xD800) << 10) | (r2 - 0xDC00)) + 0x10000);
      else { put(r); put(r2); }
      break;
    }
  }
  return o;
}

static std::string model_of(const RequestDecision& d, std::string_view body) {
  const uint32_t len = d.model_len & 0x7fffffffu;
  if (len == 0 || (size_t)d.model_off + len > body.size()) return "";
  const std::string_view raw = body.substr(d.model_off, len);
  return (d.model_len & 0x80000000u) ? DecodeJsonString(raw) : std::string(raw);
}
// time.Time.MarshalJSON of a whole second in UTC (RFC 3339)
static std::string rfc3339(int64_t unix_s) {
  time_t t = (time_t)unix_s;
  struct tm g;
  gmtime_r(&t, &g);
  char b[40];
  strftime(b, sizeof b, "%Y-%m-%dT%H:%M:%SZ", &g);
  return b;
}
static int64_t window_len(const std::string& rule) { return rule == "rpm" || rule == "tpm" ? 60 : 86400; }  // rate_limiter.go:31-68
// Go truncates time relative to year 1 (62135596800 s before the epoch)
int64_t WindowEnd(int64_t now_unix, const std::string& rule) {
  const int64_t w = window_len(rule);
  int64_t r = (now_unix + 62135596800LL) % w;
  if (r < 0) r += w;
  return now_unix - r + w;
}
std::string GoDuration(int64_t seconds) {
  const int64_t h = seconds / 3600, m = seconds / 60 % 60, s = seconds % 60;
  if (h) return std::to_string(h) + "h" + std::to_string(m) + "m" + std::to_string(s) + "s";
  if (m) return std::to_string(m) + "m" + std::to_string(s) + "s";
  return std::to_string(s) + "s";
}
std::vector<Header> RatelimitHeaders(const RequestDecision& d, const NameTables& names) {
  std::vector<Header> out;
  if (d.reason != ARKS_R_OK && d.reason != ARKS_R_RATE_LIMIT && d.reason != ARKS_R_QUOTA) return out;
  if (d.qos < 0 || (size_t)d.qos >= names.qos_rule_names.size()) return out;
  const std::vector<std::string>& rules = names.qos_rule_names[(size_t)d.qos];
  if (d.rl_entry[0] == ARKS_RL_NONE && d.rl_entry[1] == ARKS_RL_NONE) return out;
  if (d.reason == ARKS_R_RATE_LIMIT && d.detail < rules.size())
    out.push_back({"retry-after", std::to_string(d.rl_sliding ? (int64_t)d.rl_retry : WindowEnd(d.now_unix, rules[d.detail]) - d.now_unix)});
  static const char* kind[2] = {"requests", "tokens"};
  for (int t = 0; t < 2; t++) {
    if (d.rl_entry[t] == ARKS_RL_NONE || d.rl_entry[t] >= rules.size()) continue;
    const std::string k = kind[t];
    out.push_back({"x-ratelimit-limit-" + k, std::to_string(d.rl_limit[t])});
    out.push_back({"x-ratelimit-remaining-" + k, std::to_string(d.rl_remaining[t])});
    out.push_back({"x-ratelimit-reset-" + k,
                   GoDuration(d.rl_sliding ? (int64_t)d.rl_reset[t] : WindowEnd(d.now_unix, rules[d.rl_entry[t]]) - d.now_unix)});
  }
  return out;
}

ErrorReply RequestErrorReply(const RequestDecision& d, const NameTables& names, std::string_view token, std::string_view body) {
  ErrorReply e{ReasonHttpStatus(d.reason), ReasonHeader(d.reason), "true", ""};
  const std::string model = model_of(d, body);
  switch (d.reason) {
    case ARKS_R_NO_TOKEN:  // handle_request.go:48-56
      e.message = "no token found in request headers";
      break;
    case ARKS_R_REQUEST_BODY:  // :97-104
      e.message = "error processing request body";
      break;
    case ARKS_R_NO_MODEL:  // :108-115: RawValue []byte(model) with model == ""
      e.header_value = "";
      e.message = "no model in request body";
      break;
    case ARKS_R_TOKEN_NOT_FOUND:  // :119-126, err from arks_impl.go:313-315
      e.header_value = "token not found: " + std::string(token);
      e.message = "error to get qos by token";
      break;
    case ARKS_R_MODEL_NOT_IN_TOKEN:  // arks_impl.go:337
      e.header_value = "model not found: " + model;
      e.message = "error to get qos by token";
      break;
    case ARKS_R_NO_MODEL_BACKENDS:  // :147-154
      e.header_value = model;
      e.message = "model " + model + " does not exist";
      break;
    case ARKS_R_STREAM_OPTIONS:  // :162-170
      e.header_value = "include_usage for stream_options not set";
      e.message = "no stream with usage option available";
      break;
    case ARKS_R_RATE_LIMIT: {  // check.go:140-152: RateLimitResponse.JSON(), ratelimiter/types.go:98-114
      std::string rule = "rpm";
      if (d.qos >= 0 && (size_t)d.qos < names.qos_rule_names.size() && d.detail < names.qos_rule_names[(size_t)d.qos].size())
        rule = names.qos_rule_names[(size_t)d.qos][d.detail];
      // expiresAt = now + TTL(key) in the reference (redis_impl.go:104-110; wall clock with nanoseconds, TTL with jitter):
      // the one field that is not a function of the request stream. Here: the end of the rule's fixed window.
      e.message = "{\"ruleName\":\"" + rule + "\",\"overLimit\":true,\"currentUsage\":" + std::to_string(d.cur_usage) +
                  ",\"limitMax\":" + std::to_string(d.limit_max) + ",\"expiresAt\":\"" +
                  rfc3339(d.rl_sliding ? d.now_unix + (int64_t)d.rl_retry : WindowEnd(d.now_unix, rule)) + "\"}";
      break;
    }
    case ARKS_R_QUOTA: {  // check.go:95-104: QuotaResult.JSON(), quota/types.go:41-55 (Identifier has no json tag)
      std::string ns, qname, type = "total";
      if (d.qos >= 0 && (size_t)d.qos < names.qos_quota_name.size()) {
        qname = names.qos_quota_name[(size_t)d.qos];
        const int32_t t = names.qos_token[(size_t)d.qos];
        if (t >= 0 && (size_t)t < names.token_namespace.size()) ns = names.token_namespace[(size_t)t];
        if (d.detail < names.qos_quota_item_types[(size_t)d.qos].size()) type = names.qos_quota_item_types[(size_t)d.qos][d.detail];
      }
      e.message = "{\"Identifier\":[{\"Key\":\"namespace\",\"Value\":\"" + json_escape(ns) + "\"},{\"Key\":\"quotaname\",\"Value\":\"" +
                  json_escape(qname) + "\"},{\"Key\":\"type\",\"Value\":\"" + type + "\"}],\"overLimit\":true,\"currentUsage\":" +
                  std::to_string(d.cur_usage) + ",\"limitMax\":" + std::to_string(d.limit_max) + "}";
      break;
    }
    case ARKS_R_QUOTA_CONFIG: {  // check.go:76-84: err.Error() of the client's Get (apimachinery NewNotFound)
      std::string qname;
      if (d.qos >= 0 && (size_t)d.qos < names.qos_quota_name.size()) qname = names.qos_quota_name[(size_t)d.qos];
      e.message = "ArksQuota.arks.ai \"" + qname + "\" not found";
      break;
    }
    default:  // reason 255: the row never reached the device (host error)
      e.status = 500;
      e.header = "x-error-rate-limit";
      e.header_value = "rate limit error";  // handle_request.go:199-205, the reference's only other 500 of this phase
      e.message = "rate limit error";
  }
  return e;
}

ErrorReply ResponseErrorReply(const ResponseDecision& d, const NameTables& names, int32_t qos, std::string_view last_chunk) {
  ErrorReply e{ReasonHttpStatus(d.reason), ReasonHeader(d.reason), "true", ""};
  switch (d.reason) {
    // the message of the next two is err.Error() of openai-go's stream / json-iterator: third-party wording that is not a
    // function the reference defines; a fixed text stands in for it
    case ARKS_R_STREAMING: e.message = "error to unmarshal response"; break;           // handle_response.go:125-133
    case ARKS_R_RESPONSE_UNMARSHAL: e.message = "error to unmarshal response"; break;  // :157-166
    case ARKS_R_RESPONSE_UNKNOWN:                                                      // :167-181
      e.message = last_chunk.empty() ? "unknown response" : std::string(last_chunk);
      break;
    case ARKS_R_QUOTA_CONFIG_RESP: {  // :215-223 via check.go:62-72
      std::string qname;
      if (qos >= 0 && (size_t)qos < names.qos_quota_name.size()) qname = names.qos_quota_name[(size_t)qos];
      e.message = "ArksQuota.arks.ai \"" + qname + "\" not found";
      break;
    }
    default: e.status = 500; e.header = "x-error-response-unknown"; e.message = "unknown response";
  }
  return e;
}

bool ParseNameTables(std::string_view text, NameTables* out) {
  NameTables n;
  auto split = [](std::string_view s, char sep) {
    std::vector<std::string> v;
    size_t p = 0;
    for (;;) {
      const size_t q = s.find(sep, p);
      v.emplace_back(s.substr(p, q == std::string_view::npos ? s.size() - p : q - p));
      if (q == std::string_view::npos) break;
      p = q + 1;
    }
    return v;
  };
  auto list = [&](const std::string& s) { return s.empty() ? std::vector<std::string>() : split(s, ','); };
  for (const std::string& line : split(text, '\n')) {
    if (line.empty()) continue;
    const std::vector<std::string> f = split(line, '\t');
    if (f[0] == "T" && f.size() == 3) {
      n.token_namespace.push_back(f[1]);
      n.token_user.push_back(f[2]);
    } else if (f[0] == "Q" && f.size() == 6) {
      n.qos_token.push_back(atoi(f[1].c_str()));
      n.qos_model.push_back(f[2]);
      n.qos_quota_name.push_back(f[3]);
      n.qos_rule_names.push_back(list(f[4]));
      n.qos_quota_item_types.push_back(list(f[5]));
    } else {
      return false;
    }
  }
  *out = std::move(n);
  return true;
}

// ---- NameBook ---------------------------------------------------------------------------------------------------
void NameBook::Publish(uint32_t gen, NameTables t) {
  auto sp = std::make_shared<const NameTables>(std::move(t));
  std::lock_guard<std::mutex> g(mu_);
  by_gen_[gen] = std::move(sp);
  while (by_gen_.size() > ARKS_GEN_HISTORY) by_gen_.erase(by_gen_.begin());
}
void NameBook::Drop(uint32_t gen) {
  std::lock_guard<std::mutex> g(mu_);
  by_gen_.erase(gen);
}
std::shared_ptr<const NameTables> NameBook::Latest() const {
  static const std::shared_ptr<const NameTables> empty = std::make_shared<const NameTables>();
  std::lock_guard<std::mutex> g(mu_);
  return by_gen_.empty() ? empty : by_gen_.rbegin()->second;
}
std::shared_ptr<const NameTables> NameBook::Of(uint32_t gen) const {
  {
    std::lock_guard<std::mutex> g(mu_);
    auto it = by_gen_.find(gen);
    if (it != by_gen_.end()) return it->second;
  }
  return Latest();
}

// ---- StreamProcessor --------------------------------------------------------------------------------------------
std::shared_ptr<const NameTables> StreamProcessor::NamesOf(uint32_t gen) const {
  if (book_) return book_->Of(gen);
  return std::shared_ptr<const NameTables>(std::shared_ptr<const NameTables>(), names_);  // not owned: the caller's table
}
static Action reply_action(const ErrorReply& e) { return ErrorResponse(e.status, {{e.header, e.header_value}}, e.message); }

Action StreamProcessor::OnRequestHeaders(const std::vector<Header>& headers) {
  std::vector<const uint8_t*> k(headers.size()), v(headers.size());
  std::vector<size_t> kl(headers.size()), vl(headers.size());
  for (size_t i = 0; i < headers.size(); i++) {
    k[i] = (const uint8_t*)headers[i].key.data(); kl[i] = headers[i].key.size();
    v[i] = (const uint8_t*)headers[i].value.data(); vl[i] = headers[i].value.size();
  }
  const uint8_t* tok = nullptr;
  const size_t n = arks_extract_bearer(k.data(), kl.data(), v.data(), vl.data(), headers.size(), &tok);
  if (n == 0) {
    RequestDecision d{};
    d.reason = ARKS_R_NO_TOKEN;
    return reply_action(RequestErrorReply(d, *NamesOf(0), "", ""));  // this reply names nothing
  }
  token_.assign((const char*)tok, n);
  Action a;
  a.kind = Action::kContinueRequestHeaders;
  a.set_headers.push_back({"x-went-into-req-headers", "true"});
  a.clear_route_cache = true;
  return a;
}
Action StreamProcessor::OnRequestBody(std::string_view body, uint64_t pick_rand) {
  req_ = b_->HandleRequestBody(token_, body, pick_rand);
  const std::shared_ptr<const NameTables> nm = NamesOf(req_.gen);  // the generation this decision's indices belong to
  rl_ = RatelimitHeaders(req_, *nm);
  if (req_.reason != ARKS_R_OK) {
    Action a = reply_action(RequestErrorReply(req_, *nm, token_, body));
    a.set_headers.insert(a.set_headers.end(), rl_.begin(), rl_.end());  // behind x-error-* and Content-Type
    rl_.clear();
    return a;
  }
  qos_ = req_.qos;
  gen_ = req_.gen;
  stream_ = req_.flags & 1;
  metered_ = (req_.flags & ARKS_FLAG_METERED) != 0;
  Action a;
  a.kind = Action::kContinueRequestBody;
  a.set_headers.push_back({"model", nm->qos_model[(size_t)req_.qos]});
  a.set_headers.push_back({"namespace", nm->token_namespace[(size_t)req_.token]});
  a.set_headers.push_back({"username", nm->token_user[(size_t)req_.token]});
  return a;
}
Action StreamProcessor::OnResponseHeaders(const std::vector<Header>& headers) {
  Action a;
  a.kind = Action::kContinueResponseHeaders;
  a.set_headers.push_back({"x-went-into-resp-headers", "true"});
  status_ = 0;
  for (const Header& h : headers) {
    if (h.key == ":status") {
      char* end = nullptr;
      const long s = strtol(h.value.c_str(), &end, 10);
      status_ = (end && *end == 0 && !h.value.empty()) ? (int)s : 0;
    }
    a.set_headers.push_back(h);
  }
  a.clear_route_cache = true;
  // gateway.go:115-121 -> responseErrorProcessing (:281-294): the headers of the reply built so far, an empty message
  if (status_ == 500) return ErrorResponse(500, a.set_headers, "");
  if (!rl_.empty()) {  // the gateway's rate-limit headers replace the upstream's of the same name
    auto ours = [&](const Header& h) {
      std::string k = h.key;
      for (char& c : k) c = (c >= 'A' && c <= 'Z') ? (char)(c + 32) : c;
      for (const Header& r : rl_)
        if (r.key == k) return true;
      return false;
    };
    std::vector<Header> keep;
    for (const Header& h : a.set_headers)
      if (!ours(h)) keep.push_back(h);
    keep.insert(keep.end(), rl_.begin(), rl_.end());
    a.set_headers = std::move(keep);
  }
  return a;
}
Action StreamProcessor::OnResponseBody(std::string_view body, bool end_of_stream) {
  // gateway.go:122-126: the upstream's error body is passed on; `resp` is still empty there, so no x-error-* header
  if (status_ != 200) return ErrorResponse(status_, {}, std::string(body));
  if (stream_) {
    resp_ = b_->HandleResponseBody(qos_, gen_, body, ARKS_RESP_STREAM | (metered_ ? ARKS_RESP_METERED : 0u), Estimate());
  } else {
    buffered_.append(body);  // requestBuffers, handle_response.go:134-155
    if (!end_of_stream) {
      Action a;
      a.kind = Action::kContinueResponseBody;
      return a;
    }
    resp_ = b_->HandleResponseBody(qos_, gen_, buffered_, ARKS_RESP_END_OF_STREAM, Estimate());
  }
  if (resp_.reason != ARKS_R_OK && resp_.reason != ARKS_R_PENDING && resp_.reason != ARKS_R_QOS_GONE)
    return reply_action(ResponseErrorReply(resp_, *NamesOf(gen_), qos_, body));
  Action a;
  a.kind = Action::kContinueResponseBody;
  return a;
}

}  // namespace arks_host

// ---- flat C surface ---------------------------------------------------------------------------------------------
using namespace arks_host;

struct arks_host_batcher {
  Batcher* b;
  std::atomic<int64_t> fixed_now{0};
};
static int put_reply(const ErrorReply& e, char* out, uint32_t out_cap) {
  const std::string o = std::to_string(e.status) + "\n" + e.header + "\n" + e.header_value + "\n" + e.message;
  if (o.size() + 1 > out_cap) return -1;
  memcpy(out, o.c_str(), o.size() + 1);
  return (int)o.size();
}
template <class F>
static int64_t run_threads(uint32_t n, uint32_t threads, int64_t* latency_ns, F&& one) {
  if (threads == 0) threads = 1;
  std::vector<std::thread> ts;
  std::atomic<uint32_t> ready{0};
  std::atomic<bool> go{false};
  const auto t0 = std::chrono::steady_clock::now();
  for (uint32_t t = 0; t < threads; t++)
    ts.emplace_back([&, t] {
      ready.fetch_add(1);
      while (!go.load(std::memory_order_acquire)) std::this_thread::yield();
      for (uint32_t i = t; i < n; i += threads) {
        const auto a = std::chrono::steady_clock::now();
        one(i);
        const auto b = std::chrono::steady_clock::now();
        if (latency_ns) latency_ns[i] = std::chrono::duration_cast<std::chrono::nanoseconds>(b - a).count();
      }
    });
  while (ready.load() != threads) std::this_thread::yield();
  const auto t1 = std::chrono::steady_clock::now();
  go.store(true, std::memory_order_release);
  for (auto& t : ts) t.join();
  (void)t0;
  return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t1).count();
}
static int64_t fixed_clock(void* arg) { return static_cast<arks_host_batcher*>(arg)->fixed_now.load(); }

extern "C" {
int arks_host_create(arks_ctx* ctx, uint32_t max_batch, uint64_t max_bytes, uint32_t linger_us, uint32_t max_inflight,
                     arks_host_batcher** out) {
  if (!ctx || !out) return ARKS_E_INVALID_ARG;
  BatcherOptions o;
  o.max_batch = max_batch; o.max_bytes = (size_t)max_bytes; o.linger_us = linger_us;
  if (max_inflight >= 1 && max_inflight <= 4) o.max_inflight = max_inflight;
  auto* h = new arks_host_batcher();
  h->b = new Batcher(ctx, o);
  *out = h;
  return 0;
}
void arks_host_destroy(arks_host_batcher* h) {
  if (!h) return;
  delete h->b;
  delete h;
}
void arks_host_set_fixed_clock(arks_host_batcher* h, int64_t now_unix) {
  h->fixed_now.store(now_unix);
  h->b->SetClock(fixed_clock, h);
}
int arks_host_request(arks_host_batcher* h, const uint8_t* token, uint32_t token_len, const uint8_t* body, uint32_t body_len,
                      uint64_t pick_rand, RequestDecision* out) {
  *out = h->b->HandleRequestBody(std::string_view((const char*)token, token_len), std::string_view((const char*)body, body_len), pick_rand);
  return out->reason == 255 ? ARKS_E_INVALID_ARG : 0;
}
int arks_host_response(arks_host_batcher* h, int32_t qos, uint32_t gen, const uint8_t* body, uint32_t body_len, uint8_t flags,
                       ResponseDecision* out) {
  if (gen == 0xffffffffu) gen = h->b->Generation();  // "the tables have not changed since the request"
  *out = h->b->HandleResponseBody(qos, gen, std::string_view((const char*)body, body_len), flags);
  return out->reason == 255 ? ARKS_E_INVALID_ARG : 0;
}
int arks_host_load_tables(arks_host_batcher* h, const arks_tables* t) { return h->b->LoadTables(t); }
int arks_host_apply_config(arks_host_batcher* h) { return h->b->ApplyConfig(); }
int arks_host_load_tables_named(arks_host_batcher* h, const arks_tables* t, const char* names, uint32_t names_len) {
  NameTables nm;
  if (!ParseNameTables(std::string_view(names, names_len), &nm)) return ARKS_E_INVALID_ARG;
  return h->b->LoadTables(t, &nm);
}
int arks_host_apply_config_named(arks_host_batcher* h, const char* names, uint32_t names_len) {
  NameTables nm;
  if (!ParseNameTables(std::string_view(names, names_len), &nm)) return ARKS_E_INVALID_ARG;
  return h->b->ApplyConfig(&nm);
}
int arks_host_set_precharge(arks_host_batcher* h, int on) { return h->b->SetPrecharge(on != 0); }
int arks_host_set_ratelimit_report(arks_host_batcher* h, int on) { return h->b->SetRatelimitReport(on != 0); }
int arks_host_set_sliding_window(arks_host_batcher* h, int on) { return h->b->SetSlidingWindow(on != 0); }
int arks_host_ratelimit_headers(arks_host_batcher* h, const RequestDecision* d, char* out, uint32_t out_cap) {
  std::string o;
  for (const Header& x : RatelimitHeaders(*d, *h->b->Names().Of(d->gen))) o += x.key + ": " + x.value + "\n";
  if (o.size() + 1 > out_cap) return -1;
  memcpy(out, o.c_str(), o.size() + 1);
  return (int)o.size();
}
int arks_host_response_pre(arks_host_batcher* h, int32_t qos, uint32_t gen, uint32_t precharged, const uint8_t* body, uint32_t body_len,
                           uint8_t flags, arks_host::ResponseDecision* out) {
  *out = h->b->HandleResponseBody(qos, gen == 0xffffffffu ? h->b->Generation() : gen, std::string_view((const char*)body, body_len), flags, precharged);
  return out->reason == 255 ? ARKS_E_INVALID_ARG : 0;
}
int arks_host_set_names(arks_host_batcher* h, const char* text, uint32_t len) {
  NameTables nm;  // the names of the generation that is current now
  if (!ParseNameTables(std::string_view(text, len), &nm)) return ARKS_E_INVALID_ARG;
  h->b->Names().Publish(h->b->Generation(), std::move(nm));
  return 0;
}
int arks_host_request_error_reply(arks_host_batcher* h, const RequestDecision* d, const uint8_t* token, uint32_t token_len,
                                  const uint8_t* body, uint32_t body_len, char* out, uint32_t out_cap) {
  return put_reply(RequestErrorReply(*d, *h->b->Names().Of(d->gen), std::string_view((const char*)token, token_len),
                                     std::string_view((const char*)body, body_len)), out, out_cap);
}
int arks_host_response_error_reply(arks_host_batcher* h, const ResponseDecision* d, int32_t qos, const uint8_t* chunk, uint32_t chunk_len,
                                   char* out, uint32_t out_cap) {
  return put_reply(ResponseErrorReply(*d, *h->b->Names().Latest(), qos, std::string_view((const char*)chunk, chunk_len)), out, out_cap);
}
int arks_host_response_error_reply_gen(arks_host_batcher* h, const ResponseDecision* d, int32_t qos, uint32_t gen, const uint8_t* chunk,
                                       uint32_t chunk_len, char* out, uint32_t out_cap) {
  return put_reply(ResponseErrorReply(*d, *h->b->Names().Of(gen), qos, std::string_view((const char*)chunk, chunk_len)), out, out_cap);
}
void arks_host_stats(arks_host_batcher* h, BatcherStats* out) { *out = h->b->Stats(); }

int64_t arks_host_run_requests(arks_host_batcher* h, uint32_t n, uint32_t threads, const uint8_t* bodies, const uint32_t* body_off,
                               const uint32_t* body_len, const uint8_t* tokens, const uint32_t* token_off, const uint64_t* pick_rand,
                               RequestDecision* out, int64_t* latency_ns) {
  return run_threads(n, threads, latency_ns, [&](uint32_t i) {
    out[i] = h->b->HandleRequestBody(std::string_view((const char*)tokens + token_off[i], token_off[i + 1] - token_off[i]),
                                     std::string_view((const char*)bodies + body_off[i], body_len[i]), pick_rand ? pick_rand[i] : 0);
  });
}
int64_t arks_host_run_responses(arks_host_batcher* h, uint32_t n, uint32_t threads, const uint8_t* bodies, const uint32_t* body_off,
                                const uint32_t* body_len, const int32_t* qos, const uint32_t* gen, const uint8_t* flags, ResponseDecision* out,
                                int64_t* latency_ns) {
  return run_threads(n, threads, latency_ns, [&](uint32_t i) {
    out[i] = h->b->HandleResponseBody(qos[i], gen ? gen[i] : h->b->Generation(),
                                      std::string_view((const char*)bodies + body_off[i], body_len[i]), flags[i]);
  });
}

// Open-loop load: requests ARRIVE at `rate_per_s` (exponential gaps, `producers` threads each owning every
// producers-th row) whether or not earlier ones have been answered; latency = decision handed over - scheduled arrival,
// so a stalled batcher shows up as latency instead of silently slowing the generator down.
struct OpenRow {
  int64_t sched_ns;
  int64_t call_ns;        // when the generator actually made the SubmitRequest call
  int64_t* latency_call;  // optional second clock: decision - call (what the batcher and the device added on their own)
  int64_t* latency;
  arks_host::RequestDecision* out;
  std::atomic<uint32_t>* left;
};
static inline int64_t mono_ns() {
  return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
static void open_row_done(void* user, const arks_host::RequestDecision& d) {
  OpenRow* r = static_cast<OpenRow*>(user);
  const int64_t t = mono_ns();
  *r->latency = t - r->sched_ns;
  if (r->latency_call) *r->latency_call = t - r->call_ns;
  *r->out = d;
  r->left->fetch_sub(1, std::memory_order_release);
}
// how late the load generator itself was (time of the SubmitRequest call minus the row's scheduled arrival), last run:
// {max ns, rows more than 100 us late, max ns one SubmitRequest call took}. A late producer shows up in the rows' latency
// (no coordinated omission) but is the harness's doing, not the batcher's.
static std::atomic<int64_t> g_late_max{0}, g_late_slow{0}, g_submit_max{0};
static int64_t* g_call_latency = nullptr;  // n entries for the next run, or null
void arks_host_open_loop_call_latency(int64_t* buf) { g_call_latency = buf; }
void arks_host_open_loop_lateness(int64_t out[3]) { out[0] = g_late_max.load(); out[1] = g_late_slow.load(); out[2] = g_submit_max.load(); }
void arks_host_reset_tail(arks_host_batcher* h) { h->b->ResetTailStats(); }
int64_t arks_host_open_loop_requests(arks_host_batcher* h, uint32_t n, double rate_per_s, uint32_t producers, const uint8_t* bodies,
                                     const uint32_t* body_off, const uint32_t* body_len, const uint8_t* tokens, const uint32_t* token_off,
                                     const uint64_t* pick_rand, arks_host::RequestDecision* out, int64_t* latency_ns) {
  if (producers == 0) producers = 1;
  std::vector<OpenRow> rows(n);
  std::atomic<uint32_t> left{n};
  std::vector<std::thread> ts;
  g_late_max = 0; g_late_slow = 0; g_submit_max = 0;
  const int64_t t0 = mono_ns() + 2'000'000;  // everybody starts 2 ms from now
  const double mean_gap_ns = 1e9 * producers / rate_per_s;
  for (uint32_t p = 0; p < producers; p++)
    ts.emplace_back([&, p] {
      uint64_t x = 0x9E3779B97F4A7C15ull * (p + 1);
      double t = (double)t0;
      for (uint32_t i = p; i < n; i += producers) {
        x ^= x << 13; x ^= x >> 7; x ^= x << 17;  // xorshift64
        const double u = ((x >> 11) + 1) * (1.0 / 9007199254740993.0);
        t += -mean_gap_ns * __builtin_log(u);
        const int64_t due = (int64_t)t;
        int64_t now;
        for (;;) {
          now = mono_ns();
          if (now >= due) break;
          if (due - now > 200'000) std::this_thread::sleep_for(std::chrono::microseconds(100));
        }
        if (now - due > g_late_max.load(std::memory_order_relaxed)) g_late_max.store(now - due, std::memory_order_relaxed);
        if (now - due > 100'000) g_late_slow.fetch_add(1, std::memory_order_relaxed);
        rows[i] = OpenRow{due, now, g_call_latency ? &g_call_latency[i] : nullptr, &latency_ns[i], &out[i], &left};
        const bool ok = h->b->SubmitRequest(std::string_view((const char*)tokens + token_off[i], token_off[i + 1] - token_off[i]),
                                            std::string_view((const char*)bodies + body_off[i], body_len[i]),
                                            pick_rand ? pick_rand[i] : 0, open_row_done, &rows[i]);
        if (!ok) { out[i] = arks_host::RequestDecision{}; out[i].reason = 255; latency_ns[i] = 0; left.fetch_sub(1); }
        const int64_t took = mono_ns() - now;
        if (took > g_submit_max.load(std::memory_order_relaxed)) g_submit_max.store(took, std::memory_order_relaxed);
      }
    });
  for (auto& t : ts) t.join();
  while (left.load(std::memory_order_acquire) != 0) std::this_thread::yield();
  return mono_ns() - t0;
}

static void dump(std::string& o, const Action& a) {
  o += std::to_string((int)a.kind) + " " + std::to_string(a.status) + " " + (a.clear_route_cache ? "1" : "0") + "\n";
  for (const Header& h : a.set_headers) o += h.key + ": " + h.value + "\n";
  o += "\n" + a.body + "\n--\n";
}
int arks_host_stream_transcript(arks_host_batcher* h, const char* const* req_hdr_keys,
                                const char* const* req_hdr_vals, uint32_t n_req_hdr, const uint8_t* req_body, uint32_t req_body_len,
                                const char* const* resp_hdr_keys, const char* const* resp_hdr_vals, uint32_t n_resp_hdr,
                                const uint8_t* const* resp_chunks, const uint32_t* resp_chunk_len, uint32_t n_resp_chunks,
                                uint64_t pick_rand, char* out, uint32_t out_cap) {
  StreamProcessor sp(h->b, &h->b->Names());
  std::string o;
  std::vector<Header> rh, ph;
  for (uint32_t i = 0; i < n_req_hdr; i++) rh.push_back({req_hdr_keys[i], req_hdr_vals[i]});
  for (uint32_t i = 0; i < n_resp_hdr; i++) ph.push_back({resp_hdr_keys[i], resp_hdr_vals[i]});
  // Server.Process: every message is answered; an ImmediateResponse ends the exchange on Envoy's side
  Action a = sp.OnRequestHeaders(rh);
  dump(o, a);
  if (a.kind != Action::kImmediate) {
    a = sp.OnRequestBody(std::string_view((const char*)req_body, req_body_len), pick_rand);
    dump(o, a);
  }
  if (a.kind != Action::kImmediate) {
    a = sp.OnResponseHeaders(ph);
    dump(o, a);
    for (uint32_t c = 0; c < n_resp_chunks && a.kind != Action::kImmediate; c++) {
      a = sp.OnResponseBody(std::string_view((const char*)resp_chunks[c], resp_chunk_len[c]), c + 1 == n_resp_chunks);
      dump(o, a);
    }
  }
  if (o.size() + 1 > out_cap) return -1;
  memcpy(out, o.c_str(), o.size() + 1);
  return (int)o.size();
}
}
