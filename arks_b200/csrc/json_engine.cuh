// json_engine.cuh — the table-driven JSON / SSE engine of the scan kernels (device code, sm_90a; host build for tests).
//
// One lane == one document, 32 lanes in lock step. Every byte costs the same short instruction sequence on every lane:
//     class = CLS[byte];  t = TAB[state * 32 + class];  t < 240: next state, t >= 240: one of the EV_* events
// and only events (brackets, key boundaries, the end of a scalar) run handler code, so lanes that sit in different places
// of different documents stay converged. Two schedules drive it: consume_t (a byte or a bulk skip per lane per
// iteration) and consume_evsync (every lane runs up to its next event, then the warp handles the events together). The tables are generated (tools/gen_json_tables.py) from the
// grammar the oracle restates: flavor J = json-iterator ConfigFastest (request / response bodies), flavor E =
// encoding/json checkValid (SSE event data). What the gateway extracts is layered on top as hooks:
//   K_REQ   {model, stream, stream_options.include_usage}                   pkg/gateway/handle_request.go:87-104
//   K_RESP  {model, usage{prompt,completion,total}}                         pkg/gateway/handle_response.go:89-93,157
//   K_EVT   {error?, len(choices)==0, usage} of one SSE event's data        pkg/gateway/handle_response.go:113-124
#pragma once
#include "json_common.cuh"  // shared pieces: hashes, decode_span, out-of-line slow paths, SWAR byte masks
#include "json_tables.h"

namespace arks {

struct JsonTables {
  const uint8_t* cls;     // 256: byte -> class
  const uint8_t* tab_j;   // kJsonStatesJ x 32
  const uint8_t* tab_e;   // kJsonStatesE x 32
};
#if !defined(__CUDA_ARCH__)
static const uint8_t kJsonClsHost[256] = ARKS_JSON_CLASS_TABLE;
static const uint8_t kJsonTabJHost[kJsonStatesJ * kJsonClasses] = ARKS_JSON_TABLE_J;
static const uint8_t kJsonTabEHost[kJsonStatesE * kJsonClasses] = ARKS_JSON_TABLE_E;
inline JsonTables host_json_tables() { return JsonTables{kJsonClsHost, kJsonTabJHost, kJsonTabEHost}; }
#endif

enum : uint32_t { SKT_NONE = 0, SKT_MODEL = 1, SKT_UINT = 2 };  // value strings that are captured
enum : uint32_t { KK_NONE = 0, KK_STRUCT = 1, KK_EXACT = 2 };   // keys that are matched (jsoniter field hash / exact)

// State that is touched a handful of times per document lives in (local) memory, behind a pointer: only the dozen hot
// values stay in registers. With everything in registers ptxas spent more than half of the per-byte instructions on
// register-to-register copies at control-flow joins (one per field that any branch may have modified).
struct JsonCold {
  int64_t usage[3];  // prompt, completion, total
  int64_t cand[3];   // candidates of the usage object being read (committed when it closes)
  uint64_t nacc;     // number / string-number capture (gjson Result.Int); a number's start is in JsonT::sstart
  uint32_t nneg, nplain, sval_ok, sval_any;
  uint32_t cand_set, cand_nonnull;
  uint32_t m_start, m_rawlen, m_esc;  // raw span of the model string
  uint32_t stream3, so_present, iu3;  // tri-states: 0 nil, 1 false, 2 true
  uint32_t has_error_key, n_choices;
};

enum : uint32_t { CX_A = 0, CX_O = 1, CX_S = 2, CX_X = 3 };  // what kind of container a stack level is

struct JsonT {
  // ---- configuration (per lane constants)
  const uint8_t* base;  // document bytes (global memory): only slow paths and key verification read it
  const uint8_t* tab;   // kJsonStates x 32 bytes: next state, or an EV_* event (>= 240)
  const uint8_t* cls;   // byte -> class
  uint32_t* stk;        // container stack beyond the cached word (kStackWords words, caller owned)
  JsonCold* cold;
  // ---- hot state
  uint32_t ss, depth, cur_word, sstart;
  uint64_t khash;
  uint32_t hb;  // packed: kind | vm | l2 | ufield | skind | kkind | ncap (accessors below)

#define ARKS_BITS(name, sh, w)                                                              \
  ARKS_HD uint32_t name() const { return (hb >> sh) & ((1u << w) - 1u); }                     \
  ARKS_HD void set_##name(uint32_t v) { hb = (hb & ~(((1u << w) - 1u) << sh)) | (v << sh); }
  ARKS_BITS(kind, 0, 2)
  ARKS_BITS(vm, 2, 4)
  ARKS_BITS(l2, 6, 2)
  ARKS_BITS(ufield, 8, 2)
  ARKS_BITS(skind, 10, 2)
  ARKS_BITS(kkind, 12, 2)
  ARKS_BITS(ncap, 14, 2)
#undef ARKS_BITS
  static constexpr uint32_t kSideMask = 0xFC00u;  // skind | kkind | ncap: some byte-level capture is in progress

  ARKS_HD void init(uint32_t k, const uint8_t* b, uint32_t* stack_words, JsonCold* c, const JsonTables& t) {
    base = b; stk = stack_words; cold = c; cls = t.cls; tab = k == K_EVT ? t.tab_e : t.tab_j;
    ss = k == K_EVT ? TS_VAL_T : TS_TOP;  // jsoniter's struct decoder only accepts '{' or null at the top
    depth = 0; cur_word = 0; sstart = 0; khash = 0;
    hb = k;
    c->usage[0] = c->usage[1] = c->usage[2] = 0;
    c->cand[0] = c->cand[1] = c->cand[2] = 0;
    c->nacc = 0;
    c->nneg = 0; c->nplain = 1; c->sval_ok = 0; c->sval_any = 0;
    c->cand_set = 0; c->cand_nonnull = 0;
    c->m_start = 0; c->m_rawlen = 0; c->m_esc = 0; c->stream3 = 0; c->so_present = 0; c->iu3 = 0;
    c->has_error_key = 0; c->n_choices = 0;
  }
  // restart for the next SSE event (fresh ChatCompletionChunk per event)
  ARKS_HD void reset_event() {
    ss = TS_VAL_T; depth = 0; cur_word = 0; hb = K_EVT;
    JsonCold* c = cold;
    c->usage[0] = c->usage[1] = c->usage[2] = 0;
    c->cand_set = 0; c->cand_nonnull = 0;
    c->has_error_key = 0; c->n_choices = 0;
  }
  ARKS_HD bool failed() const { return ss == TS_ERRSTATE; }

  // ---- container stack: two bits per level (CX_*); the innermost 16 levels live in a register
  ARKS_HD uint32_t top_ctx() const { return (cur_word >> (2 * ((depth - 1) & 15))) & 3u; }
  ARKS_HD void push(uint32_t cx) {
    if (depth >= kMaxDepth) { ss = TS_ERRSTATE; return; }
    const uint32_t nd = depth + 1;
    if (depth > 0 && ((nd - 1) >> 4) != ((depth - 1) >> 4)) { stk[(depth - 1) >> 4] = cur_word; cur_word = 0; }
    const uint32_t sh = 2 * ((nd - 1) & 15);
    cur_word = (cur_word & ~(3u << sh)) | (cx << sh);
    depth = nd;
  }
  ARKS_HD void pop() {
    const uint32_t nd = depth - 1;
    if (nd > 0 && ((nd - 1) >> 4) != ((depth - 1) >> 4)) cur_word = stk[(nd - 1) >> 4];
    depth = nd;
  }

  // ---- events -----------------------------------------------------------------------------------
  // first non-blank byte of a value in an S / X / T context; true when the byte has been consumed here
  ARKS_HD bool special_value_begin(uint8_t c, uint32_t pos, uint32_t ps) {
    const uint32_t m = vm();
    JsonCold* q = cold;
    if (m == VM_SKIP) {
      if ((ps == TS_VAL_T) & (c == '{')) {  // top level of an SSE event: its keys are matched exactly
        push(CX_X);
        if (ss != TS_ERRSTATE) ss = TS_OBJX_FIRST;
        return true;
      }
      return false;
    }
    set_vm(VM_SKIP);
    if (m == VM_MODEL) {  // stringCodec -> ReadString: string or null
      if (c == '"') { set_skind(SKT_MODEL); sstart = pos + 1; }
      else if (c == 'n') { q->m_start = 0; q->m_rawlen = 0; q->m_esc = 0; }
      else { ss = TS_ERRSTATE; return true; }
      return false;
    }
    if (m == VM_BOOL_STREAM || m == VM_BOOL_IU) {  // OptionalDecoder{boolCodec}: ReadNil / ReadBool
      if (c != 'n' && c != 't' && c != 'f') { ss = TS_ERRSTATE; return true; }
      const uint32_t v = c == 'n' ? 0u : c == 'f' ? 1u : 2u;
      if (m == VM_BOOL_STREAM) q->stream3 = v; else q->iu3 = v;
      return false;
    }
    if (m == VM_SO) {  // OptionalDecoder{oneFieldStructDecoder}
      if (c == 'n') { q->so_present = 0; q->iu3 = 0; return false; }
      if (c != '{') { ss = TS_ERRSTATE; return true; }
      q->so_present = 1;  // an already allocated struct is reused: include_usage of an earlier occurrence persists
      push(CX_S);
      set_l2(L2_SO);
      if (ss != TS_ERRSTATE) ss = TS_STRUCT_FIRST;
      return true;
    }
    if (m == VM_UINT) {  // a usage counter: gjson Result.Int by JSON type
      const uint32_t f = ufield();
      q->cand_set |= 1u << f;
      q->cand_nonnull |= 1u << f;
      q->cand[f] = c == 't' ? 1 : 0;
      if (c == 'n') q->cand_nonnull &= ~(1u << f);
      if (c == '"') {
        set_skind(SKT_UINT);
        sstart = pos + 1;
        q->nacc = 0; q->nneg = 0; q->sval_ok = 1; q->sval_any = 0;
      } else if (c == '-' || is_digit(c)) {
        set_ncap(2);  // armed: this very byte is the number's first byte; it is captured when it is re-dispatched
        sstart = pos;  // no string is open while a number is captured
        q->nneg = 0; q->nacc = 0; q->nplain = 1;
      }
      return false;
    }
    if (m == VM_USAGE) {
      if (kind() == K_EVT) { q->usage[0] = q->usage[1] = q->usage[2] = 0; }  // Map(): the last "usage" member wins outright
      q->cand_set = 0; q->cand_nonnull = 0;
      if (c != '{') return false;
      push(CX_X);
      set_l2(L2_USAGE);
      if (ss != TS_ERRSTATE) ss = TS_OBJX_FIRST;
      return true;
    }
    // VM_ECHOICES
    q->n_choices = 0;
    if (c != '[') return false;
    push(CX_A);
    if (ss != TS_ERRSTATE) ss = TS_ARRC_FIRST;  // its first element raises EV_CHOICE_ELEM
    return true;
  }

  ARKS_HD void key_begin(uint32_t pos, uint32_t ps) {
    sstart = pos + 1;
    const bool strct = ps >= TS_STRUCT_FIRST;  // STRUCT_FIRST / STRUCT_KEY vs OBJX_FIRST / OBJX_KEY
    set_kkind(strct ? KK_STRUCT : KK_EXACT);
    khash = strct ? 0x811c9dc5ull : 0xcbf29ce484222325ull;
    ss = strct ? TS_STRS : TS_STRX;
  }
  ARKS_HD void key_end(uint32_t pos, uint32_t ps) {
    const uint32_t esc = ps & 1u;
    const bool strct = ps < TS_STRX;
    ss = strct ? TS_COLON_S : TS_COLON_X;
    set_kkind(KK_NONE);
    if (strct) {  // jsoniter readFieldHash + struct decoder dispatch
      uint64_t h = khash;
      if (esc) h = struct_key_hash_slow(base + sstart, pos - sstart);
      const uint32_t kd = kind();
      if (depth == 1) {
        if (h == H_MODEL) set_vm(VM_MODEL);
        else if (kd == K_REQ && h == H_STREAM) set_vm(VM_BOOL_STREAM);
        else if (kd == K_REQ && h == H_SO) set_vm(VM_SO);
        else if (kd == K_RESP && h == H_USAGE) set_vm(VM_USAGE);
      } else if (h == H_IU) {
        set_vm(VM_BOOL_IU);
      }
    } else {  // gjson Map(): case-sensitive, unescaped
      const int lo = depth == 2 ? 0 : 3;
      // cheap inline filter first: the out-of-line exact comparison (it re-reads the key bytes) only runs for keys whose
      // 64-bit hash already equals a candidate's, or that contain escapes
      const bool maybe = esc | (lo == 0 ? (khash == X_PROMPT) | (khash == X_COMPL) | (khash == X_TOTAL)
                                        : (khash == X_ERROR) | (khash == X_CHOICES) | (khash == X_USAGE));
      if (!maybe) return;
      const int hit = exact_key_match(base + sstart, pos - sstart, esc, khash, lo, lo + 3);
      if (hit < 0) return;
      if (hit < 3) { set_ufield((uint32_t)hit); set_vm(VM_UINT); }
      else if (hit == 3) cold->has_error_key = 1;
      else if (hit == 4) set_vm(VM_ECHOICES);
      else set_vm(VM_USAGE);
    }
  }
  // closing quote of a captured value string
  ARKS_HD void string_done(uint32_t pos, uint32_t esc) {
    JsonCold* q = cold;
    if (skind() == SKT_MODEL) {
      q->m_start = sstart; q->m_rawlen = pos - sstart; q->m_esc = esc;
    } else {  // SKT_UINT: gjson String -> parseInt(t.Str)
      int64_t v = 0;
      if (!esc && q->sval_ok && q->sval_any) v = q->nneg ? (int64_t)(0 - q->nacc) : (int64_t)q->nacc;
      q->cand[ufield()] = v;
    }
    set_skind(SKT_NONE);
  }
  ARKS_HD void close_container() {
    if (depth == 2) {
      if (l2() == L2_USAGE) {
        // apijson struct decoder over node.Map(): last duplicate wins; null leaves the field untouched
        JsonCold* q = cold;
        for (int f = 0; f < 3; f++)
          if ((q->cand_set >> f) & (q->cand_nonnull >> f) & 1) q->usage[f] = q->cand[f];
      }
      set_l2(L2_NONE);
    }
    pop();
    ss = depth == 0 ? TS_FINISH : TS_AFTER_A + top_ctx();
  }
  // a byte of a captured number: a plain integer is parsed on the fly (wrapping), anything else is re-read at its end
  ARKS_HD void capture_number_byte(uint8_t c) {
    JsonCold* q = cold;
    if (ncap() == 2) {  // the number's first byte
      set_ncap(1);
      if (c == '-') q->nneg = 1; else q->nacc = (uint64_t)(c - '0');
      return;
    }
    if (is_digit(c)) q->nacc = q->nacc * 10 + (uint64_t)(c - '0');
    else q->nplain = 0;
  }
  // `pos`: the byte after the number (a CR held back by the SSE line layer can make it one more)
  ARKS_HD void finish_number_capture(uint32_t pos) {
    JsonCold* q = cold;
    set_ncap(0);
    q->cand[ufield()] = captured_number_value(q->nacc, q->nneg, q->nplain, base + sstart, pos - sstart);
  }
  // side work of an ordinary (non-event) transition while something is being captured
  ARKS_HD void side_work(uint32_t ps, uint8_t c, uint32_t pos) {
    if (ncap()) capture_number_byte(c);
    else if (ps < TS_N_STRING_STATES) {  // an ordinary byte inside a string that was stepped (not bulk-skipped)
      const uint32_t kk = kkind();
      if (kk) khash = kk == KK_STRUCT ? fhash_step(khash, c) : xhash_step(khash, c);
      else if ((skind() == SKT_UINT) & !(ps & 1u)) {  // gjson parseInt over the raw string
        JsonCold* q = cold;
        if (c == '-' && !q->sval_any && !q->nneg && pos == sstart) q->nneg = 1;
        else if (is_digit(c)) { q->nacc = q->nacc * 10 + (uint64_t)(c - '0'); q->sval_any = 1; }
        else q->sval_ok = 0;
      }
    }
  }
  ARKS_HD void event(uint32_t t, uint32_t k, uint8_t c, uint32_t pos) {
    const uint32_t ps = ss;
    for (;;) {
      if (t == EV_ERR) { ss = TS_ERRSTATE; return; }
      if (t == EV_POP) { close_container(); return; }
      if (t == EV_PUSHO || t == EV_PUSHA || t == EV_TOP_OBJ) {
        push(t == EV_PUSHO ? CX_O : t == EV_PUSHA ? CX_A : CX_S);
        if (ss != TS_ERRSTATE) ss = t == EV_PUSHO ? TS_OBJ_FIRST : t == EV_PUSHA ? TS_ARR_FIRST : TS_STRUCT_FIRST;
        return;
      }
      if (t == EV_KEY_BEGIN) { key_begin(pos, ps); return; }
      if (t == EV_KEY_END) { key_end(pos, ps); return; }
      if (t == EV_STR_DONE) {
        if (skind() != SKT_NONE) string_done(pos, ps & 1u);
        ss = ps < TS_STRV_X ? TS_AFTER_S : TS_AFTER_X;
        return;
      }
      // the remaining events handle something and then dispatch the same byte again from another state
      if (t == EV_VALUE_BEGIN) {
        // most members of S / X objects are not read by the gateway: skip the handler for them
        if (((vm() != VM_SKIP) | (ps == TS_VAL_T)) && special_value_begin(c, pos, ps)) return;
        ss = ps == TS_VAL_S ? TS_VALG_S : ps == TS_VAL_X ? TS_VALG_X : TS_VALG_T;
      } else if (t == EV_NUM_DONE) {
        if (ncap()) finish_number_capture(pos);
        ss = TS_AFTER_X;
      } else {  // EV_CHOICE_ELEM
        cold->n_choices = 1;
        ss = TS_VAL_A;
      }
      t = tab[ss * kJsonClasses + k];
      if (t < EV_BASE) {
        const uint32_t from = ss;
        ss = t;
        if (hb & kSideMask) side_work(from, c, pos);
        return;
      }
    }
  }

  // ---- one byte: two table lookups; everything else is rare -----------------------------------------
  ARKS_HD void step(uint8_t c, uint32_t pos) {
    const uint32_t k = cls[c];
    const uint32_t t = tab[ss * kJsonClasses + k];
    if (t < EV_BASE) {
      const uint32_t ps = ss;
      ss = t;
      if (hb & kSideMask) side_work(ps, c, pos);
    } else {
      event(t, k, c, pos);
    }
  }

  ARKS_HD bool ok_at_end() const { return ss == TS_FINISH || ss == TS_STOP; }

  // ---- bulk interface: inside a string whose ordinary bytes need no per-byte work the caller skips straight to the next
  // '"', '\\' or byte < 0x20; matched keys still get their skipped bytes hashed.
  ARKS_HD bool can_fast() const { return (ss < TS_N_STRING_STATES) & (skind() != SKT_UINT); }
  ARKS_HD void skip(uint32_t n, uint32_t o, uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3) {
    const uint32_t kk = kkind();
    if (kk) {
      uint64_t h = khash;
      const bool fold = kk == KK_STRUCT;
      for (uint32_t k = o; k < o + n; k++) {
        const uint32_t lo = (k & 8) ? q2 : q0, hi = (k & 8) ? q3 : q1;
        const uint8_t b = (uint8_t)(((k & 4) ? hi : lo) >> (8 * (k & 3)));
        h = fold ? fhash_step(h, b) : xhash_step(h, b);
      }
      khash = h;
    }
  }
  ARKS_HD bool dead() const { return (ss - TS_STOP) < 2u; }  // TS_STOP or TS_ERRSTATE
};

// ---------------------------------------------------------------------------------------------
// SSE chunk machine: bufio.Scanner(ScanLines) + eventStreamDecoder.Next + Stream.Next
// (openai-go packages/ssestream, restated in oracle/ork_json.c: ork_sse_chunk / sse_event)
// ---------------------------------------------------------------------------------------------
struct SseT {
  JsonT ev;
  int64_t usage[3];
  uint32_t line_len;   // raw bytes of the current line (CR included)
  uint32_t name_len;   // bytes of the field name seen so far
  uint64_t name_acc;   // first 8 name bytes, little endian
  uint32_t data_pos;   // bytes of event data fed so far
  uint64_t data_head;  // first 8 bytes of the event data (the [DONE] probe)
  uint32_t ev_match;   // progress of matching the event type against "thread."
  uint32_t phase;      // 0 name, 1 just after ':', 2 value
  uint32_t field;      // 0 other, 1 data, 2 event
  uint32_t pending_cr, done, fail, thread_evt;

  ARKS_HD void init(const uint8_t* base, uint32_t* stack_words, JsonCold* cold, const JsonTables& tabs) {
    ev.init(K_EVT, base, stack_words, cold, tabs);
    usage[0] = usage[1] = usage[2] = 0;
    line_len = 0; name_len = 0; name_acc = 0; data_pos = 0; data_head = 0; ev_match = 0;
    phase = 0; field = 0; pending_cr = 0; done = 0; fail = 0; thread_evt = 0;
  }
  ARKS_HD void feed_data(uint8_t c, uint32_t pos) {
    if (data_pos < 8) data_head |= (uint64_t)c << (8 * data_pos);
    data_pos++;
    if (!done) ev.step(c, pos);
  }
  ARKS_HD void classify_name() {
    if (name_len == 4 && (uint32_t)name_acc == 0x61746164u /*data*/) field = 1;
    else if (name_len == 5 && (name_acc & 0xFFFFFFFFFFull) == 0x746e657665ull /*event*/) field = 2;
    else field = 0;
    if (field == 2) { ev_match = 0; thread_evt = 0; }  // `event = string(value)`: the last event line wins
  }
  ARKS_HD void line_byte(uint8_t c, uint32_t pos) {
    if (phase == 1) {  // first byte after the colon: one optional space is dropped
      phase = 2;
      if (c == ' ') return;
    }
    if (phase == 2) {
      if (field == 1) feed_data(c, pos);
      else if (field == 2 && ev_match < 7) {
        const uint64_t T = 0x2e646165726874ull;  // "thread." little endian
        if ((uint8_t)(T >> (8 * ev_match)) == c) { if (++ev_match == 7) thread_evt = 1; }
        else ev_match = 0xFF;
      }
      return;
    }
    if (c == ':') { classify_name(); phase = 1; return; }
    if (name_len < 8) name_acc |= (uint64_t)c << (8 * name_len);
    name_len++;
  }
  ARKS_HD void dispatch() {  // Stream.Next for one event
    if (!done) {
      const bool is_done = data_pos >= 6 && (data_head & 0xFFFFFFFFFFFFull) == 0x5d454e4f445bull;  // "[DONE]"
      if (is_done) done = 1;
      else if (!ev.ok_at_end() || ev.cold->has_error_key) fail = 1;
      else {
        const bool wrapped = thread_evt;
        const uint32_t nc = wrapped ? 0 : ev.cold->n_choices;
        if (nc == 0) {  // handle_response.go:119-123
          usage[0] = wrapped ? 0 : ev.cold->usage[0];
          usage[1] = wrapped ? 0 : ev.cold->usage[1];
          usage[2] = wrapped ? 0 : ev.cold->usage[2];
        }
      }
    }
    ev.reset_event();
    data_pos = 0; data_head = 0; thread_evt = 0; ev_match = 0;
  }
  ARKS_HD void end_line(uint32_t pos) {
    const uint32_t content = line_len - (pending_cr ? 1 : 0);  // dropCR
    if (content == 0) {
      dispatch();
    } else {
      if (phase == 0) classify_name();  // no colon: the whole line is the field name
      if (field == 1) feed_data('\n', pos);
    }
    line_len = 0; name_len = 0; name_acc = 0; phase = 0; field = 0; pending_cr = 0;
  }
  ARKS_HD void step(uint8_t c, uint32_t pos) {
    if (fail) return;
    if (c == '\n') { end_line(pos); return; }
    line_len++;
    if (line_len >= 65536) { fail = 1; return; }  // bufio.Scanner: token too long
    if (pending_cr) {  // the held CR was not the last byte of its line
      pending_cr = 0;
      line_byte('\r', pos);
    }
    if (c == '\r') { pending_cr = 1; return; }
    line_byte(c, pos);
  }
  ARKS_HD bool can_fast() const {
    return (phase == 2) & (field == 1) & !done & !fail & !pending_cr & (data_pos >= 8) & (line_len < 65000) & ev.can_fast();
  }
  ARKS_HD void skip(uint32_t k, uint32_t o, uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3) {
    line_len += k;
    data_pos += k;
    ev.skip(k, o, q0, q1, q2, q3);
  }
  ARKS_HD bool dead() const { return fail; }
  // end of chunk: an unterminated last line is still a token; a pending event is dropped
  ARKS_HD bool finish(uint32_t pos) {
    if (!fail && line_len > 0) end_line(pos);
    return !fail;
  }
};

// ---------------------------------------------------------------------------------------------
// SseSplit — the line layer of SseT alone, 16 bytes at a time, for chunks that look the way every OpenAI-compatible
// server writes them: only `data:` lines, comment lines and blank lines, no CR, exactly one data line per event and
// no line of 64 KiB. For such a chunk it reports the payload span of every event the decoder would dispatch, in
// order, stopping at the first `[DONE]`; the events can then be parsed independently of each other (one lane each,
// all lanes starting at the first byte of a JSON document, which is what keeps a warp converged). Anything else
// (`event:` lines, CR LF, multi-line data, empty events, over-long lines ...) sets `irregular` and the caller runs
// SseT over the whole chunk instead, so the verdict never depends on which of the two paths ran.
// ---------------------------------------------------------------------------------------------
ARKS_HD uint32_t eq_mask16(uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3, uint32_t c4) {
  uint32_t f[4] = {q0 ^ c4, q1 ^ c4, q2 ^ c4, q3 ^ c4};
  uint32_t m = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int k = 0; k < 4; k++) {
    const uint32_t t = ~(((f[k] & 0x7f7f7f7fu) + 0x7f7f7f7fu) | f[k]) & 0x80808080u;  // bit 7 of every zero byte, exact
    m |= (((t >> 7) * 0x01020408u) >> 24 & 0xfu) << (4 * k);
  }
  return m;
}

struct SseSplit {
  uint32_t s;         // start of the current line
  uint32_t have;      // bytes of the line head captured so far (<= 16)
  uint64_t h0, h1;    // first 16 bytes of the current line, little endian
  uint32_t pend_off, pend_len;
  uint32_t flags;     // F_*
  enum : uint32_t { F_PEND = 1, F_PEND_DONE = 2, F_STOPPED = 4, F_IRREGULAR = 8 };

  ARKS_HD void init() { s = 0; have = 0; h0 = h1 = 0; pend_off = pend_len = 0; flags = 0; }
  ARKS_HD bool irregular() const { return flags & F_IRREGULAR; }

  // append the bytes of unit `ub` that belong to the head of the current line
  ARKS_HD void capture(uint32_t ub, uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3) {
    const uint32_t o = s + have - ub;  // first unit byte that is not captured yet (s + have >= ub by construction)
    if (o >= 16) return;
    uint64_t lo = (uint64_t)q0 | (uint64_t)q1 << 32, hi = (uint64_t)q2 | (uint64_t)q3 << 32;
    if (o >= 8) { lo = hi >> (8 * (o - 8)); hi = 0; }
    else if (o) { lo = (lo >> (8 * o)) | (hi << (64 - 8 * o)); hi >>= 8 * o; }
    // (lo, hi) now start at the first new byte; place them behind the `have` bytes already there
    if (have == 0) { h0 = lo; h1 = hi; }
    else if (have >= 8) { h1 |= lo << (8 * (have - 8)); }
    else { h0 |= lo << (8 * have); h1 |= (lo >> (64 - 8 * have)) | (hi << (8 * have)); }
    have += 16 - o;
    if (have > 16) have = 16;
  }
  template <class E>
  ARKS_HD void end_line(uint32_t p, E&& emit) {
    const uint32_t L = p - s;
    if (L >= 65536) { flags |= F_IRREGULAR; return; }  // bufio.Scanner: token too long
    if (L == 0) {                                      // blank line: dispatch
      if (flags & F_PEND) {
        if (!(flags & F_STOPPED)) {
          if (flags & F_PEND_DONE) flags |= F_STOPPED;
          else emit(pend_off, pend_len);
        }
        flags &= ~(uint32_t)(F_PEND | F_PEND_DONE);
      } else if (!(flags & F_STOPPED)) {
        flags |= F_IRREGULAR;  // an event without data: not JSON, the stream fails
      }
      return;
    }
    if ((uint8_t)h0 == ':') return;  // comment
    if (L >= 5 && (h0 & 0xFFFFFFFFFFull) == 0x3a61746164ull /* "data:" */) {
      if (flags & F_PEND) { flags |= F_IRREGULAR; return; }  // multi-line data
      const uint32_t sp = (L >= 6 && (uint8_t)(h0 >> 40) == ' ') ? 1u : 0u;
      pend_off = s + 5 + sp;
      pend_len = L - 5 - sp;
      // first six payload bytes = head bytes [5+sp, 11+sp)
      const uint64_t six = sp ? ((h0 >> 48) | (h1 << 16)) : ((h0 >> 40) | (h1 << 24));
      flags |= F_PEND;
      if (pend_len >= 6 && (six & 0xFFFFFFFFFFFFull) == 0x5d454e4f445bull /* "[DONE]" */) flags |= F_PEND_DONE;
      return;
    }
    flags |= F_IRREGULAR;  // any other field, or a line without a colon
  }
  // one 16-byte unit starting at byte `ub`, `nvalid` of its bytes inside the chunk
  template <class E>
  ARKS_HD void unit(uint32_t ub, uint32_t nvalid, uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3, E&& emit) {
    const uint32_t valid = nvalid >= 16 ? 0xffffu : ((1u << nvalid) - 1u);
    uint32_t nl = eq_mask16(q0, q1, q2, q3, 0x0a0a0a0au) & valid;
    if (eq_mask16(q0, q1, q2, q3, 0x0d0d0d0du) & valid) flags |= F_IRREGULAR;
    if (have < 16) capture(ub, q0, q1, q2, q3);
    while (nl) {
      const uint32_t p = ub + first_set(nl);
      nl &= nl - 1;
      end_line(p, emit);
      s = p + 1; have = 0; h0 = h1 = 0;
      capture(ub, q0, q1, q2, q3);
    }
  }
  ARKS_HD void finish(uint32_t len) {
    if (len - s >= 65536) flags |= F_IRREGULAR;  // unterminated over-long last line
  }
};

// verdict of one event parsed on its own (SseT::dispatch for a regular chunk)
struct SseEventVerdict {
  uint32_t fail, no_choices;
};
ARKS_HD SseEventVerdict sse_event_verdict(JsonT& ev, uint32_t end_pos) {
  if (!ev.dead()) ev.step('\n', end_pos);  // the decoder joins data lines with '\n'
  SseEventVerdict v;
  v.fail = !ev.ok_at_end() || ev.cold->has_error_key;
  v.no_choices = !v.fail && ev.cold->n_choices == 0;
  return v;
}

// ---------------------------------------------------------------------------------------------
// Feed bytes [pos, lim) of one document to machine `m`; `load(u)` returns its 16-byte unit u (bytes past the end may
// hold anything). Every iteration is the same for every lane: (1) if the machine sits in a string, swallow the plain
// bytes up to the next special byte of this unit; (2) push one byte through the table. The special-byte mask of a unit is
// computed once, when the unit is loaded.
// ---------------------------------------------------------------------------------------------
template <class M, class L, class K>
ARKS_HD void consume_t(M& m, uint32_t& pos, uint32_t lim, L&& load, K&& mask_of) {
  uint32_t cu = 0xffffffffu, q0 = 0, q1 = 0, q2 = 0, q3 = 0, umask = 0;
  while (pos < lim) {
    uint32_t o = pos & 15;
    if ((pos >> 4) != cu) {
      cu = pos >> 4;
      const Unit16 q = load(cu);
      q0 = q.w[0]; q1 = q.w[1]; q2 = q.w[2]; q3 = q.w[3];
      umask = mask_of(cu, q0, q1, q2, q3);
    }
    if (m.can_fast()) {
      const uint32_t rest = umask >> o;
      uint32_t run = rest ? first_set(rest) : 16u - o;
      const uint32_t avail = lim - pos;
      if (run > avail) run = avail;
      if (run) {
        m.skip(run, o, q0, q1, q2, q3);
        pos += run;
        o += run;
      }
      if ((o == 16) | (pos >= lim)) continue;
    }
    const uint32_t lo = (o & 8) ? q2 : q0, hi = (o & 8) ? q3 : q1;
    const uint32_t w = (o & 4) ? hi : lo;
    m.step((uint8_t)(w >> (8 * (o & 3))), pos);
    pos++;
    if (m.dead()) return;
  }
}

// Same contract as consume_t for a bare JsonT, different schedule: every lane first runs its ordinary transitions
// (and bulk skips) up to the next byte that raises an event, then the warp handles one event per lane together.
// When the 32 documents of a warp share a template (frames of one SSE stream format, completions of one server) the
// k-th event of every lane is the same kind, so event() runs with the warp converged instead of ~10 lanes wide;
// documents that do not line up only cost idle lanes, never a different result.
// ---------------------------------------------------------------------------------------------
// consume_rounds — the schedule the scan kernels use for heterogeneous documents. One round = up to R ordinary
// advances per lane (a bulk skip and / or one table step each), then ONE event per lane for the lanes that ran into
// one, then the warp re-converges (__syncwarp). Without the forced re-convergence the lanes of a warp whose documents
// differ drift apart for good (Volta+ schedules diverged lanes independently and a loop with early exits has no
// convergence point inside), so a warp of 32 different chat requests ran only a few lanes wide. With rounds, a lane that reaches an event early idles for at most R-1 short advances, and
// the expensive event code runs once per round instead of once per byte position of any lane.
// ALL 32 lanes of the warp must call this together (lanes without work pass pos >= lim). Host build: a plain loop.
// ---------------------------------------------------------------------------------------------
template <int R, class L, class K>
ARKS_HD void consume_rounds(JsonT& m, uint32_t& pos, uint32_t lim, L&& load, K&& mask_of) {
  uint32_t cu = 0xffffffffu, q0 = 0, q1 = 0, q2 = 0, q3 = 0, umask = 0;
#ifdef __CUDA_ARCH__
  while (__any_sync(0xffffffffu, pos < lim)) {
#else
  while (pos < lim) {
#endif
    uint32_t t = 0, k = 0;
    uint8_t c = 0;
    bool ev = false;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int r = 0; r < R; r++) {
      if (!ev && pos < lim) {
        uint32_t o = pos & 15;
        if ((pos >> 4) != cu) {
          cu = pos >> 4;
          const Unit16 q = load(cu);
          q0 = q.w[0]; q1 = q.w[1]; q2 = q.w[2]; q3 = q.w[3];
          umask = mask_of(cu, q0, q1, q2, q3);
        }
        bool more = true;
        if (m.can_fast()) {
          const uint32_t rest = umask >> o;
          uint32_t run = rest ? first_set(rest) : 16u - o;
          const uint32_t avail = lim - pos;
          if (run > avail) run = avail;
          if (run) {
            m.skip(run, o, q0, q1, q2, q3);
            pos += run;
            o += run;
          }
          more = (o < 16) & (pos < lim);
        }
        if (more) {
          const uint32_t lo = (o & 8) ? q2 : q0, hi = (o & 8) ? q3 : q1;
          const uint32_t w = (o & 4) ? hi : lo;
          c = (uint8_t)(w >> (8 * (o & 3)));
          k = m.cls[c];
          t = m.tab[m.ss * kJsonClasses + k];
          if (t >= EV_BASE) {
            ev = true;
          } else {
            const uint32_t ps = m.ss;
            m.ss = t;
            if (m.hb & JsonT::kSideMask) m.side_work(ps, c, pos);
            pos++;
            if (m.dead()) pos = lim;
          }
        }
      }
    }
    if (ev) {
      m.event(t, k, c, pos);
      pos++;
      if (m.dead()) pos = lim;
    }
#ifdef __CUDA_ARCH__
    __syncwarp();
#endif
  }
}

struct MaskOnTheSpot {
  ARKS_HD uint32_t operator()(uint32_t, uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3) const { return special_mask16(q0, q1, q2, q3); }
};
template <class M, class L>
ARKS_HD void consume_t(M& m, uint32_t& pos, uint32_t lim, L&& load) { consume_t(m, pos, lim, load, MaskOnTheSpot()); }

template <class L, class K>
ARKS_HD void consume_evsync(JsonT& m, uint32_t& pos, uint32_t lim, L&& load, K&& mask_of) {
  uint32_t cu = 0xffffffffu, q0 = 0, q1 = 0, q2 = 0, q3 = 0, umask = 0;
  while (pos < lim) {
    uint32_t t = 0, k = 0;
    uint8_t c = 0;
    bool ev = false;
    while (pos < lim) {
      uint32_t o = pos & 15;
      if ((pos >> 4) != cu) {
        cu = pos >> 4;
        const Unit16 q = load(cu);
        q0 = q.w[0]; q1 = q.w[1]; q2 = q.w[2]; q3 = q.w[3];
        umask = mask_of(cu, q0, q1, q2, q3);
      }
      if (m.can_fast()) {
        const uint32_t rest = umask >> o;
        uint32_t run = rest ? first_set(rest) : 16u - o;
        const uint32_t avail = lim - pos;
        if (run > avail) run = avail;
        if (run) {
          m.skip(run, o, q0, q1, q2, q3);
          pos += run;
          o += run;
        }
        if ((o == 16) | (pos >= lim)) continue;
      }
      const uint32_t lo = (o & 8) ? q2 : q0, hi = (o & 8) ? q3 : q1;
      const uint32_t w = (o & 4) ? hi : lo;
      c = (uint8_t)(w >> (8 * (o & 3)));
      k = m.cls[c];
      t = m.tab[m.ss * kJsonClasses + k];
      if (t >= EV_BASE) { ev = true; break; }
      const uint32_t ps = m.ss;
      m.ss = t;
      if (m.hb & JsonT::kSideMask) m.side_work(ps, c, pos);
      pos++;
      if (m.dead()) return;
    }
    if (!ev) return;
    m.event(t, k, c, pos);
    pos++;
    if (m.dead()) return;
  }
}

template <class L>
ARKS_HD void consume_evsync(JsonT& m, uint32_t& pos, uint32_t lim, L&& load) { consume_evsync(m, pos, lim, load, MaskOnTheSpot()); }

template <int R, class L>
ARKS_HD void consume_rounds(JsonT& m, uint32_t& pos, uint32_t lim, L&& load) { consume_rounds<R>(m, pos, lim, load, MaskOnTheSpot()); }

}  // namespace arks
