// host_machine.cpp — TEST-ONLY build of arks_b200/csrc/json_engine.cuh with g++ so the device state
// machines can be fuzzed against the oracle on CPU (tests/test_machine_vs_oracle.py). Not shipped.
#include <stddef.h>
#include <stdint.h>
#include <string.h>

// Bytes the caller's buffer holds behind the document (hm_set_past_end): the host drivers read them past the end instead
// of their fixed fills, as the device reads the padding, the next body or stale staging memory there.
static thread_local size_t g_past = 0;
#define ARKS_HOST_PAST_END(doc, len, p, dflt) ((size_t)(p) - (size_t)(len) < g_past ? (doc)[p] : (dflt))

#include "../arks_b200/csrc/json_engine.cuh"

#include <type_traits>

using namespace arks;

static int g_evsync = 0;  // schedule for JsonT documents: 0 consume_t, 1 consume_evsync, 4 / 8 consume_rounds<R>

// same bulk loop the kernels run, with units read straight from memory; past the end: the `avail` bytes the buffer holds
// from `body` on, then a fixed fill
template <class M>
static void feed(M& m, const uint8_t* body, size_t len, uint32_t begin = 0, size_t avail = (size_t)-1) {
  if (avail == (size_t)-1) avail = len + g_past;
  uint32_t pos = begin;
  // exercise window boundaries like the tiled kernels do: consume in 128-byte windows
  for (uint32_t wbeg = 0; wbeg < len; wbeg += 128) {
    uint32_t lim = (uint32_t)(len < wbeg + 128 ? len : wbeg + 128);
    auto load = [&](uint32_t u) {
      Unit16 q;
      uint8_t tmp[16];
      const size_t o = (size_t)u * 16;
      for (int k = 0; k < 16; k++) tmp[k] = o + k < avail ? body[o + k] : (uint8_t)(0xA5 ^ k);  // garbage past the end
      memcpy(q.w, tmp, 16);
      return q;
    };
    if constexpr (std::is_same<M, JsonT>::value) {
      if (g_evsync == 1) consume_evsync(m, pos, lim, load);
      else if (g_evsync == 4) consume_rounds<4>(m, pos, lim, load);
      else if (g_evsync == 8) consume_rounds<8>(m, pos, lim, load);
      else consume_t(m, pos, lim, load);
    } else {
      consume_t(m, pos, lim, load);
    }
    if (m.dead()) break;
  }
}

extern "C" {
void hm_set_evsync(int on) { g_evsync = on; }
void hm_set_past_end(size_t n) { g_past = n; }
int hm_parse_request(const uint8_t* body, size_t len, uint8_t* model_out, size_t cap, size_t* model_len, int* stream,
                     int* so_present, int* iu) {
  static thread_local JsonT m;
  static thread_local uint32_t stk[kStackWords];
  static thread_local JsonCold cold;
  m.init(K_REQ, body, stk, &cold, host_json_tables());
  feed(m, body, len);
  *stream = cold.stream3;
  *so_present = cold.so_present;
  *iu = cold.iu3;
  size_t k = 0;
  if (m.ok_at_end()) {
    if (cold.m_esc)
      decode_span(body + cold.m_start, cold.m_rawlen, [&](uint8_t b) {
        if (k < cap) model_out[k] = b;
        k++;
      });
    else {
      k = cold.m_rawlen;
      memcpy(model_out, body + cold.m_start, k < cap ? k : cap);
    }
  }
  *model_len = k;
  return m.ok_at_end() ? 0 : 1;
}
int hm_parse_response(const uint8_t* body, size_t len, size_t* model_nonempty, int64_t usage[3]) {
  static thread_local JsonT m;
  static thread_local uint32_t stk[kStackWords];
  static thread_local JsonCold cold;
  m.init(K_RESP, body, stk, &cold, host_json_tables());
  feed(m, body, len);
  *model_nonempty = cold.m_rawlen > 0;
  for (int k = 0; k < 3; k++) usage[k] = cold.usage[k];
  return m.ok_at_end() ? 0 : 1;
}
int hm_parse_sse(const uint8_t* body, size_t len, int64_t usage[3]) {
  static thread_local SseT m;
  static thread_local uint32_t stk[kStackWords];
  static thread_local JsonCold cold;
  m.init(body, stk, &cold, host_json_tables());
  feed(m, body, len);
  bool ok = m.finish((uint32_t)len);
  for (int k = 0; k < 3; k++) usage[k] = m.usage[k];
  return ok ? 0 : 1;
}
// The split path of the SSE kernel: SseSplit finds the events, every event is parsed on its own from a 16-byte
// aligned base (like a lane of the event phase), verdicts are combined in order. Returns 0/1 like hm_parse_sse, +2
// when the chunk was irregular and SseT ran instead.
int hm_parse_sse_split(const uint8_t* body, size_t len, int64_t usage[3]) {
  static thread_local uint32_t stk[kStackWords];
  static thread_local JsonCold cold;
  SseSplit sp;
  sp.init();
  uint32_t offs[4096], lens[4096], n_ev = 0;
  bool overflow = false;
  for (size_t ub = 0; ub < len; ub += 16) {
    uint8_t tmp[16];
    size_t n = len - ub < 16 ? len - ub : 16;
    for (int k = 0; k < 16; k++)  // past the end: the caller's bytes, then hostile padding: LF / CR
      tmp[k] = ub + k < len + g_past ? body[ub + k] : (uint8_t)(0x0a ^ (k & 1 ? 0x07 : 0));
    uint32_t q[4];
    memcpy(q, tmp, 16);
    sp.unit((uint32_t)ub, (uint32_t)n, q[0], q[1], q[2], q[3], [&](uint32_t off, uint32_t l) {
      if (n_ev < 4096) { offs[n_ev] = off; lens[n_ev] = l; n_ev++; } else overflow = true;
    });
  }
  sp.finish((uint32_t)len);
  if (sp.irregular() || overflow) return hm_parse_sse(body, len, usage) + 2;
  usage[0] = usage[1] = usage[2] = 0;
  bool fail = false;
  for (uint32_t e = 0; e < n_ev && !fail; e++) {
    const uint8_t* base = body + (offs[e] & ~15u);
    const uint32_t begin = offs[e] & 15u, end = begin + lens[e];
    JsonT m;
    m.init(K_EVT, base, stk, &cold, host_json_tables());
    feed(m, base, end, begin, len + g_past - (offs[e] & ~15u));
    SseEventVerdict v = sse_event_verdict(m, end);
    if (v.fail) fail = true;
    else if (v.no_choices) for (int k = 0; k < 3; k++) usage[k] = cold.usage[k];
  }
  if (fail) usage[0] = usage[1] = usage[2] = 0;
  return fail ? 1 : 0;
}
// Work profile of one document for the lock-step analysis (tools/lockstep_model.py): for every 128-byte window the number
// of advances the schedules need (one bulk skip and / or one table step each) and the number of events among them.
int hm_work_profile(int kind, const uint8_t* body, size_t len, uint32_t* advances, uint32_t* events, size_t max_windows) {
  static thread_local JsonT m;
  static thread_local uint32_t stk[kStackWords];
  static thread_local JsonCold cold;
  m.init(kind == 0 ? K_REQ : K_RESP, body, stk, &cold, host_json_tables());
  size_t n_win = (len + 127) / 128;
  if (n_win > max_windows) return -1;
  for (size_t w = 0; w < n_win; w++) advances[w] = events[w] = 0;
  uint32_t pos = 0;
  while (pos < len && !m.dead()) {
    const size_t w = pos >> 7;
    const uint32_t lim = (uint32_t)(len < (w + 1) * 128 ? len : (w + 1) * 128);
    const uint32_t ub = pos & ~15u;
    uint8_t tmp[16] = {0};
    memcpy(tmp, body + ub, len - ub < 16 ? len - ub : 16);
    uint32_t q[4];
    memcpy(q, tmp, 16);
    uint32_t o = pos & 15;
    advances[w]++;
    bool more = true;
    if (m.can_fast()) {
      const uint32_t rest = special_mask16(q[0], q[1], q[2], q[3]) >> o;
      uint32_t run = rest ? first_set(rest) : 16u - o;
      if (run > lim - pos) run = lim - pos;
      if (run) { m.skip(run, o, q[0], q[1], q[2], q[3]); pos += run; o += run; }
      more = o < 16 && pos < lim;
    }
    if (more) {
      const uint8_t c = body[pos];
      const uint32_t before = m.ss;
      const uint32_t t = m.tab[m.ss * kJsonClasses + m.cls[c]];
      if (t >= EV_BASE) events[w]++;
      (void)before;
      m.step(c, pos);
      pos++;
    }
  }
  return (int)n_win;
}
}

// ---- the fast path (arks_b200/csrc/mask_scan.cuh), host driver = exactly one lane's work: 1 = accepted (fields filled),
// 0 = the document is left to the exact engine ----
#include <cstdio>
#include <cstdlib>
#include "../arks_b200/csrc/mask_scan.cuh"
extern "C" {
// every call also runs the two-lane form of pass A (fast_scan_host_split): same verdict and same output, or the test dies.
// One stated exception (fast_esc_after): when the 32 bytes in front of the split point are all backslashes the second lane
// cannot know its escape carry, and the two-lane form declines a document the one-lane form may accept.
static void split_must_agree(bool ok, const FastOut& o, bool ok2, const FastOut& o2, const uint8_t* body, size_t len) {
  const uint32_t nch = (uint32_t)((len + 31) / 32), h = fast_split_point(nch);
  bool blind = ok && !ok2 && h && h < nch;
  for (uint32_t p = 32 * (h - 1); blind && p < 32 * h; p++) blind = body[p] == '\\';
  const bool same = blind || (ok == ok2 && (!ok || (o.m_start == o2.m_start && o.m_rawlen == o2.m_rawlen && o.m_esc == o2.m_esc && o.stream3 == o2.stream3 &&
                                                    o.so_present == o2.so_present && o.iu3 == o2.iu3 && o.usage[0] == o2.usage[0] &&
                                                    o.usage[1] == o2.usage[1] && o.usage[2] == o2.usage[2])));
  if (!same) {
    fprintf(stderr, "split pass A disagrees with the one-lane form (ok %d vs %d) on %zu bytes: %.*s\n", (int)ok, (int)ok2, len, (int)(len < 400 ? len : 400), body);
    abort();
  }
}
int hm_fast_request(const uint8_t* body, size_t len, uint32_t* span /* start, rawlen, esc */, int* stream, int* so_present, int* iu) {
  FastOut o{}, o2{};
  if (len > 0xffffffffu) return 0;
  const bool ok = fast_scan_host<K_REQ>(body, (uint32_t)len, o), ok2 = fast_scan_host_split<K_REQ>(body, (uint32_t)len, o2);
  split_must_agree(ok, o, ok2, o2, body, len);
  if (!ok) return 0;
  span[0] = o.m_start; span[1] = o.m_rawlen; span[2] = o.m_esc;
  *stream = (int)o.stream3; *so_present = (int)o.so_present; *iu = (int)o.iu3;
  return 1;
}
int hm_fast_response(const uint8_t* body, size_t len, uint32_t* span, int64_t* usage) {
  FastOut o{}, o2{};
  if (len > 0xffffffffu) return 0;
  const bool ok = fast_scan_host<K_RESP>(body, (uint32_t)len, o), ok2 = fast_scan_host_split<K_RESP>(body, (uint32_t)len, o2);
  split_must_agree(ok, o, ok2, o2, body, len);
  if (!ok) return 0;
  span[0] = o.m_start; span[1] = o.m_rawlen; span[2] = o.m_esc;
  usage[0] = o.usage[0]; usage[1] = o.usage[1]; usage[2] = o.usage[2];
  return 1;
}
// what the exact engine reports for the same document, in the same terms (raw model span instead of decoded bytes)
int hm_engine_request_span(const uint8_t* body, size_t len, uint32_t* span, int* stream, int* so_present, int* iu) {
  static thread_local JsonT m;
  static thread_local uint32_t stk[kStackWords];
  static thread_local JsonCold cold;
  m.init(K_REQ, body, stk, &cold, host_json_tables());
  feed(m, body, len);
  if (!m.ok_at_end()) return 0;
  span[0] = cold.m_rawlen ? cold.m_start : 0; span[1] = cold.m_rawlen; span[2] = cold.m_rawlen ? cold.m_esc : 0;
  *stream = (int)cold.stream3; *so_present = (int)cold.so_present; *iu = (int)cold.iu3;
  return 1;
}
int hm_engine_response_span(const uint8_t* body, size_t len, uint32_t* span, int64_t* usage) {
  static thread_local JsonT m;
  static thread_local uint32_t stk[kStackWords];
  static thread_local JsonCold cold;
  m.init(K_RESP, body, stk, &cold, host_json_tables());
  feed(m, body, len);
  if (!m.ok_at_end()) return 0;
  span[0] = cold.m_rawlen ? cold.m_start : 0; span[1] = cold.m_rawlen; span[2] = cold.m_rawlen ? cold.m_esc : 0;
  usage[0] = cold.usage[0]; usage[1] = cold.usage[1]; usage[2] = cold.usage[2];
  return 1;
}
}

// ---- the BPE token counter (arks_b200/csrc/bpe.cuh) on the host: the same scanner, pre-tokenizer and merge loop ----
static unsigned long long g_bpe_probes[2];  // slots read in the shared-memory table / in the full table
static unsigned long long g_bpe_pieces, g_bpe_text_bytes;
#define ARKS_BPE_PROBE(kind) (g_bpe_probes[kind]++)
#include "../arks_b200/csrc/bpe.cuh"
#include <vector>
static std::vector<BpeSlot> g_bpe_table, g_bpe_hot;
static std::vector<uint32_t> g_bpe_byte_id;
static std::vector<uint8_t> g_bpe_cls;
static BpeTablesDev g_bpe{};
extern "C" {
void hm_bpe_load(const uint32_t* byte_id, uint32_t n, const uint32_t* left, const uint32_t* right, const uint32_t* merged,
                 const uint8_t* cp_class, uint32_t flags) {
  g_bpe_byte_id.assign(byte_id, byte_id + 256);
  g_bpe_cls.assign(cp_class, cp_class + 0x110000 / 2);
  const uint32_t slots = bpe_table_slots(n);
  bpe_fill_table(g_bpe_table, slots, left, right, merged, n);
  bpe_fill_table(g_bpe_hot, kBpeHotSlots, left, right, merged, n < kBpeHotMerges ? n : kBpeHotMerges);
  g_bpe = BpeTablesDev{g_bpe_byte_id.data(), g_bpe_table.data(), slots - 1, g_bpe_hot.data(), g_bpe_cls.data(), flags};
}
// tokens of every `content` string of the body, or 0xFFFFFFFF (uncounted)
uint32_t hm_bpe_count(const uint8_t* body, size_t len) {
  std::vector<uint8_t> text(len + 8);
  uint32_t total = 0;
  const BpeScanOut o = bpe_scan_body(body, (uint32_t)len, text.data(), g_bpe, [&](uint32_t off, uint32_t n) {
    total += bpe_piece_tokens(text.data() + off, n, g_bpe.hot, g_bpe);
    g_bpe_pieces++;
    g_bpe_text_bytes += n;
  });
  return o.bad ? kBpeUncounted : total;
}
// table slots read since the last call: [0] hot (shared-memory) table, [1] full table; [2] pieces, [3] decoded text bytes
void hm_bpe_probes(unsigned long long* out) {
  out[0] = g_bpe_probes[0]; out[1] = g_bpe_probes[1]; out[2] = g_bpe_pieces; out[3] = g_bpe_text_bytes;
  g_bpe_probes[0] = g_bpe_probes[1] = g_bpe_pieces = g_bpe_text_bytes = 0;
}
// the pieces of one plain text (UTF-8), as end offsets (test of the pre-tokenizer alone)
int hm_bpe_pretokenize(const uint8_t* text, size_t len, uint32_t* ends, int cap) {
  int n = 0;
  bpe_pretokenize(text, 0, (uint32_t)len, g_bpe.cp_class, [&](uint32_t, uint32_t e) { if (n < cap) ends[n] = e; n++; });
  return n;
}
}

// ---- the warp-per-document latency path (arks_b200/csrc/warp_scan.cuh): its host driver runs the per-lane phases with the
// warp collectives written as loops ----
#include "../arks_b200/csrc/warp_scan.cuh"
extern "C" {
int hm_warp_request(const uint8_t* body, size_t len, uint32_t* span, int* stream, int* so_present, int* iu) {
  static thread_local uint32_t tok[wd::kFastMaxTok + 64];
  wd::FastOut o{};
  if (len > 0xffffffffu || !wd::fast_scan_host<K_REQ>(body, (uint32_t)len, o, tok)) return 0;
  span[0] = o.m_start; span[1] = o.m_rawlen; span[2] = o.m_esc;
  *stream = (int)o.stream3; *so_present = (int)o.so_present; *iu = (int)o.iu3;
  return 1;
}
int hm_warp_response(const uint8_t* body, size_t len, uint32_t* span, int64_t* usage) {
  static thread_local uint32_t tok[wd::kFastMaxTok + 64];
  wd::FastOut o{};
  if (len > 0xffffffffu || !wd::fast_scan_host<K_RESP>(body, (uint32_t)len, o, tok)) return 0;
  span[0] = o.m_start; span[1] = o.m_rawlen; span[2] = o.m_esc;
  usage[0] = o.usage[0]; usage[1] = o.usage[1]; usage[2] = o.usage[2];
  return 1;
}
}

// ---- the object store of the config plane (arks_b200/csrc/config_store.h is host-only C++): same calls as the ABI's
// arks_upsert_* / arks_delete_*, flatten() exposed as an arks_tables view for the oracle ----
#include "../arks_b200/csrc/config_store.h"
struct HmStore {
  arks::ConfigStore st;
  arks::FlatTables flat;
  arks_tables view;
};
extern "C" {
void* hm_store_new() { return new HmStore(); }
void hm_store_free(void* s) { delete static_cast<HmStore*>(s); }
void hm_store_upsert_token(void* s, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const char* token, uint32_t token_len,
                           const arks_qos_spec* qos, uint32_t n_qos) {
  static_cast<HmStore*>(s)->st.upsert_token(ns, ns_len, name, name_len, token, token_len, qos, n_qos);
}
void hm_store_upsert_quota(void* s, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const uint8_t* type,
                           const int64_t* value, uint32_t n) {
  static_cast<HmStore*>(s)->st.upsert_quota(ns, ns_len, name, name_len, type, value, n);
}
void hm_store_upsert_endpoint(void* s, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len, const int32_t* w, uint32_t n) {
  static_cast<HmStore*>(s)->st.upsert_endpoint(ns, ns_len, name, name_len, w, n);
}
int hm_store_erase(void* s, int which, const char* ns, uint32_t ns_len, const char* name, uint32_t name_len) {
  return static_cast<HmStore*>(s)->st.erase(which, ns, ns_len, name, name_len) ? 1 : 0;
}
// the snapshot shape check arks_prepare_tables applies (config_store.h): NULL = well formed
const char* hm_tables_shape_error(const arks_tables* t) { return arks::tables_shape_error(t); }
const arks_tables* hm_store_flatten(void* s) {
  HmStore* h = static_cast<HmStore*>(s);
  h->flat = arks::FlatTables();
  h->st.flatten(&h->flat);
  h->view = h->flat.view();
  return &h->view;
}
}
