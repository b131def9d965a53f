// warp_scan.cuh — the LATENCY path of the scan: one WARP per document (device, sm_90a; host build for tests).
//
// A micro-batch of a few hundred requests leaves most of the GPU idle, and what the stream threads wait for is the time ONE
// document takes, and one lane walking 1 KiB of chat JSON alone is a long dependent chain; here the 32 lanes of a warp share
// the document:
//
//   phase 1  (per 1 KiB segment, 32 bytes per lane, bit masks)  quote / backslash masks -> escaped characters (carry
//            between lanes by shuffle) -> in-string mask (prefix XOR inside the word, ballot across lanes) -> string
//            content checks -> every byte OUTSIDE strings becomes a token (position, byte) in a per-warp array, placed by a
//            warp prefix sum: a compact, ordered list of the document's structure
//   phase 2  the token list is cut into 32 equal chunks, one per lane: (a) each lane folds its chunk's brackets into a
//            stack effect (pops, pushes, container bits), (b) a warp scan composes the effects so every lane knows the
//            container stack at its first token, (c) each lane derives its grammar state from the tokens just before its
//            chunk and walks its tokens through the JSON grammar, (d) the lanes that meet a member the gateway reads
//            (model / stream / stream_options / usage) extract it.
//
// As a THROUGHPUT path it loses: per document, its warp collectives cost more than a lane-per-document scan, and that holds
// with the single-lane tails taken out too (DESIGN.md §5, "Why large batches do not take it"). Large batches take
// mask_scan.cuh. Same contract as mask_scan.cuh: a
// FILTER in front of the exact engine (json_engine.cuh) that accepts a document only inside a conservative subset (valid
// RFC 8259, no control bytes in strings, depth <= 32, top-level object, the members the gateway reads of the expected type,
// not duplicated, spelled without escapes, <= kFastMaxLen bytes / kFastMaxTok structure bytes); everything else goes to
// the exact engine, so verdicts never depend on the path (tests/test_warp_scan.py).
#pragma once
#include "json_common.cuh"

namespace arks {
namespace wd {

constexpr uint32_t kFastMaxLen = 2048;   // bytes of a document this path keeps resident (longer ones: exact engine)
constexpr uint32_t kFastMaxTok = 512;    // bytes outside strings (structure, scalars, blanks)
constexpr uint32_t kFastMaxDepth = 32;   // one container bit per level in a 32-bit word
constexpr uint32_t kFastSeg = 1024;      // bytes per mask pass: 32 lanes x 32 bytes
constexpr uint32_t kFastMiniCap = 160;   // tokens a lane may walk alone inside stream_options / usage

// token entry: pos (16) | byte (8) | flags
constexpr uint32_t TK_OPEN = 1u << 24, TK_CLOSE = 1u << 25;
ARKS_HD uint32_t tk_pos(uint32_t t) { return t & 0xffffu; }
ARKS_HD uint32_t tk_byte(uint32_t t) { return (t >> 16) & 0xffu; }

struct FastOut {
  uint32_t m_start, m_rawlen, m_esc;  // raw span of the model string (0 / 0 / 0: null or absent)
  uint32_t stream3, so_present, iu3;  // K_REQ tri-states: 0 nil, 1 false, 2 true
  int64_t usage[3];                   // K_RESP
};

// ---- byte-plane SWAR: bit 7 of every byte that is zero, exact ----
ARKS_HD uint32_t zero_bytes(uint32_t x) { return ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x) & 0x80808080u; }
// the 4 flag bits (bit 7 of each byte) as a nibble
ARKS_HD uint32_t plane_nibble(uint32_t t) { return ((t >> 7) * 0x01020408u) >> 24; }

// ---- phase 1 lane state ----
struct FastMasks {
  uint32_t Q, B, V;  // quote, backslash, inside-the-document: bit j = byte j of the lane's 32
  uint32_t anyc;     // some byte < 0x20 among the lane's 32 (byte plane, unreduced)
  uint32_t w[8];
};

// masks of the lane's 32 bytes; `w` = the bytes as 8 little-endian words, `nvalid` = how many of them are inside the document
ARKS_HD void fast_masks(FastMasks& m, uint32_t nvalid) {
  uint32_t Q = 0, B = 0, anyc = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int j = 0; j < 8; j++) {
    const uint32_t x = m.w[j];
    Q |= plane_nibble(zero_bytes(x ^ 0x22222222u)) << (4 * j);
    B |= plane_nibble(zero_bytes(x ^ 0x5c5c5c5cu)) << (4 * j);
    anyc |= zero_bytes(x & 0xe0e0e0e0u);
  }
  m.V = nvalid >= 32 ? 0xffffffffu : ((1u << nvalid) - 1u);
  m.Q = Q & m.V;
  m.B = B & m.V;
  m.anyc = anyc;
}
// bytes < 0x20 as a bit mask (only computed when anyc says there is one)
ARKS_HD uint32_t fast_ctrl_mask(const FastMasks& m) {
  uint32_t C = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int j = 0; j < 8; j++) C |= plane_nibble(zero_bytes(m.w[j] & 0xe0e0e0e0u)) << (4 * j);
  return C & m.V;
}
// the lane's last backslash run has odd length (it escapes the next lane's first byte), for B != ~0
ARKS_HD uint32_t odd_tail(uint32_t B) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__clz((int)~B) & 1u;
#else
  return (~B ? (uint32_t)__builtin_clz(~B) : 32u) & 1u;
#endif
}
// characters escaped by a backslash (simdjson's find_escaped on 32-bit words); prev = the previous lane's odd_tail
ARKS_HD uint32_t find_escaped(uint32_t bs, uint32_t prev) {
  bs &= ~prev;
  const uint32_t follows = (bs << 1) | prev;
  const uint32_t even = 0x55555555u;
  const uint32_t odd_starts = bs & ~even & ~follows;
  const uint32_t invert = (odd_starts + bs) << 1;
  return (even ^ invert) & follows;
}
ARKS_HD uint32_t prefix_xor32(uint32_t x) {
  x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16;
  return x;
}
ARKS_HD uint32_t popc32(uint32_t x) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__popc(x);
#else
  return (uint32_t)__builtin_popcount(x);
#endif
}

// string content checks for the lane's bytes; doc = the whole document (shared memory on the device).
// E: escaped characters, R: inside-a-string (opening quote included), Qu: unescaped quotes. false = not in the subset.
ARKS_HD bool fast_string_checks(const uint8_t* doc, uint32_t len, uint32_t base, const FastMasks& m, uint32_t E, uint32_t R) {
  if (m.B & ~R) return false;                           // a backslash outside a string
  if (m.anyc && (fast_ctrl_mask(m) & R)) return false;  // a control byte inside a string
  uint32_t e = E;
  while (e) {
    const uint32_t p = base + first_set(e);
    e &= e - 1;
    const uint8_t c = doc[p];
    if (c == 'u') {
      if (p + 4 >= len) return false;
      if ((hexval(doc[p + 1]) | hexval(doc[p + 2]) | hexval(doc[p + 3]) | hexval(doc[p + 4])) < 0) return false;
    } else if (!(c == '"' || c == '\\' || c == '/' || c == 'b' || c == 'f' || c == 'n' || c == 'r' || c == 't')) {
      return false;
    }
  }
  return true;
}
// append the lane's tokens (bytes outside strings: TB) at tok[off...]
ARKS_HD void fast_emit(const uint8_t* doc, uint32_t base, uint32_t TB, uint32_t Qu, uint32_t R, uint32_t* tok, uint32_t off) {
  while (TB) {
    const uint32_t j = first_set(TB);
    TB &= TB - 1;
    const uint32_t p = base + j;
    uint32_t t = p | (uint32_t)doc[p] << 16;
    if ((Qu >> j) & 1u) t |= ((R >> j) & 1u) ? TK_OPEN : TK_CLOSE;
    tok[off++] = t;
  }
}

// ---- phase 2: grammar over the token list ----
enum : uint32_t {
  G_VAL = 0, G_ARR0, G_OBJ0, G_KEY, G_COLON, G_AFTER, G_STRK, G_STRV, G_TOP, G_END,
  G_T1, G_T2, G_T3, G_F1, G_F2, G_F3, G_F4, G_N1, G_N2, G_N3,         // literals in progress
  G_NM, G_NZ, G_NI, G_ND, G_NF, G_NE, G_NS, G_NX,                     // RFC 8259 number
  G_ERR
};
ARKS_HD bool tk_ws(uint32_t b) { return b == ' ' || b == '\t' || b == '\n' || b == '\r'; }
ARKS_HD bool g_scalar_state(uint32_t g) { return g >= G_T1 && g <= G_NX; }
ARKS_HD bool g_number_accepting(uint32_t g) { return g == G_NZ || g == G_NI || g == G_NF || g == G_NX; }

// one byte of a literal / number in progress: next state, G_AFTER when the literal is complete, G_ERR, or 0xff when the
// byte does not belong to the scalar (the caller ends an accepting number and dispatches the byte again)
ARKS_HD uint32_t scalar_step(uint32_t g, uint32_t b) {
  const bool dig = (b - '0') <= 9u;
  switch (g) {
    case G_T1: return b == 'r' ? G_T2 : G_ERR;
    case G_T2: return b == 'u' ? G_T3 : G_ERR;
    case G_T3: return b == 'e' ? G_AFTER : G_ERR;
    case G_F1: return b == 'a' ? G_F2 : G_ERR;
    case G_F2: return b == 'l' ? G_F3 : G_ERR;
    case G_F3: return b == 's' ? G_F4 : G_ERR;
    case G_F4: return b == 'e' ? G_AFTER : G_ERR;
    case G_N1: return b == 'u' ? G_N2 : G_ERR;
    case G_N2: return b == 'l' ? G_N3 : G_ERR;
    case G_N3: return b == 'l' ? G_AFTER : G_ERR;
    case G_NM: return b == '0' ? G_NZ : dig ? G_NI : G_ERR;
    case G_NZ: return b == '.' ? G_ND : (b == 'e' || b == 'E') ? G_NE : dig ? G_ERR : 0xffu;
    case G_NI: return dig ? G_NI : b == '.' ? G_ND : (b == 'e' || b == 'E') ? G_NE : 0xffu;
    case G_ND: return dig ? G_NF : G_ERR;
    case G_NF: return dig ? G_NF : (b == 'e' || b == 'E') ? G_NE : 0xffu;
    case G_NE: return dig ? G_NX : (b == '+' || b == '-') ? G_NS : G_ERR;
    case G_NS: return dig ? G_NX : G_ERR;
    default:   return dig ? G_NX : 0xffu;  // G_NX
  }
}
// first byte of a value
ARKS_HD uint32_t value_start(uint32_t t) {
  const uint32_t b = tk_byte(t);
  if (t & TK_OPEN) return G_STRV;
  if (b == 't') return G_T1;
  if (b == 'f') return G_F1;
  if (b == 'n') return G_N1;
  if (b == '-') return G_NM;
  if (b == '0') return G_NZ;
  if ((b - '1') <= 8u) return G_NI;
  return G_ERR;  // brackets are handled by the caller
}

struct FastWalk {
  uint32_t g, depth, stack;  // stack: bit d = level d+1 is an object
  ARKS_HD bool top_obj() const { return depth && ((stack >> (depth - 1)) & 1u); }
  // consume one token; false = grammar error / outside the subset
  ARKS_HD bool step(uint32_t t) {
    const uint32_t b = tk_byte(t);
    if (g_scalar_state(g)) {
      const uint32_t n = scalar_step(g, b);
      if (n != 0xffu) { g = n; return n != G_ERR; }
      g = G_AFTER;  // an accepting number ended before this byte (0xff is only returned from accepting states)
    }
    if (g == G_STRK) { g = G_COLON; return (t & TK_CLOSE) != 0; }
    if (g == G_STRV) { g = depth ? G_AFTER : G_END; return (t & TK_CLOSE) != 0; }
    if (tk_ws(b)) return true;
    switch (g) {
      case G_TOP:
        if (b != '{') return false;
        depth = 1; stack = 1u; g = G_OBJ0;
        return true;
      case G_VAL: case G_ARR0:
        if (b == '{' || b == '[') {
          if (depth >= kFastMaxDepth) return false;
          stack = (stack & ~(1u << depth)) | ((b == '{' ? 1u : 0u) << depth);
          depth++;
          g = b == '{' ? G_OBJ0 : G_ARR0;
          return true;
        }
        if (b == ']' && g == G_ARR0 && depth) { depth--; g = depth ? G_AFTER : G_END; return true; }
        g = value_start(t);
        return g != G_ERR;
      case G_OBJ0:
        if (t & TK_OPEN) { g = G_STRK; return true; }
        if (b == '}' && depth) { depth--; g = depth ? G_AFTER : G_END; return true; }
        return false;
      case G_KEY:
        if (t & TK_OPEN) { g = G_STRK; return true; }
        return false;
      case G_COLON:
        g = G_VAL;
        return b == ':';
      case G_AFTER:
        if (b == ',') { g = top_obj() ? G_KEY : G_VAL; return true; }
        if (b == '}' || b == ']') {
          if (depth == 0 || top_obj() != (b == '}')) return false;
          depth--;
          g = depth ? G_AFTER : G_END;
          return true;
        }
        return false;
      default:  // G_END: only blanks may follow the document
        return false;
    }
  }
};

// a chunk's brackets as a stack effect: pop `npop` levels (their closers' kinds in ptypes, first pop in bit 0), then push
// `npush` levels (kinds in pword, first push in bit 0)
struct FastEffect {
  uint32_t npop, npush, pword, ptypes;
  uint32_t bad;  // a closer did not match the opener it closes inside the chunk, or more than 32 levels
};
ARKS_HD void effect_token(FastEffect& e, uint32_t t) {
  if (t & (TK_OPEN | TK_CLOSE)) return;
  const uint32_t b = tk_byte(t);
  if (b == '{' || b == '[') {
    if (e.npush >= kFastMaxDepth) { e.bad = 1; return; }
    e.pword = (e.pword & ~(1u << e.npush)) | ((b == '{' ? 1u : 0u) << e.npush);
    e.npush++;
  } else if (b == '}' || b == ']') {
    const uint32_t kind = b == '}' ? 1u : 0u;
    if (e.npush) {
      e.npush--;
      if (((e.pword >> e.npush) & 1u) != kind) e.bad = 1;
    } else {
      if (e.npop >= kFastMaxDepth) { e.bad = 1; return; }
      e.ptypes |= kind << e.npop;
      e.npop++;
    }
  }
}
// effect of A followed by B (pop kinds of the outer levels are checked by the lanes themselves, not carried)
ARKS_HD FastEffect effect_compose(const FastEffect& a, const FastEffect& b) {
  FastEffect r;
  r.bad = a.bad | b.bad;
  r.ptypes = 0;
  if (b.npop <= a.npush) {
    const uint32_t k = a.npush - b.npop;
    r.npop = a.npop;
    r.npush = k + b.npush;
    if (r.npush > kFastMaxDepth) { r.bad = 1; r.npush = kFastMaxDepth; }
    r.pword = (k >= 32 ? a.pword : (a.pword & ((1u << k) - 1u))) | (k >= 32 ? 0u : (b.pword << k));
  } else {
    r.npop = a.npop + (b.npop - a.npush);
    r.npush = b.npush;
    r.pword = b.pword;
  }
  return r;
}

// last token before k that is not a blank, or -1
ARKS_HD int prev_sig(const uint32_t* tok, int k) {
  for (int j = k - 1; j >= 0; j--)
    if (!tk_ws(tk_byte(tok[j])) || (tok[j] & (TK_OPEN | TK_CLOSE))) return j;
  return -1;
}
ARKS_HD int next_sig(const uint32_t* tok, int k, int ntok) {
  for (int j = k + 1; j < ntok; j++)
    if (!tk_ws(tk_byte(tok[j])) || (tok[j] & (TK_OPEN | TK_CLOSE))) return j;
  return ntok;
}
ARKS_HD bool tk_is(uint32_t t, uint8_t c) { return tk_byte(t) == c && !(t & (TK_OPEN | TK_CLOSE)); }
// a byte of a literal or number (anything outside strings that is neither blank nor punctuation)
ARKS_HD bool tk_scalar(uint32_t t) {
  const uint32_t b = tk_byte(t);
  return !(t & (TK_OPEN | TK_CLOSE)) && !tk_ws(b) && b != ',' && b != ':' && b != '[' && b != ']' && b != '{' && b != '}';
}

// grammar state in front of token k0, given the container stack there; valid whenever tokens [0, k0) are a valid prefix
ARKS_HD uint32_t fast_state_before(const uint32_t* tok, int k0, uint32_t depth, uint32_t stack) {
  const bool top_obj = depth && ((stack >> (depth - 1)) & 1u);
  const int p = prev_sig(tok, k0);
  if (p < 0) return G_TOP;
  const uint32_t t = tok[p];
  auto key_position = [&](int q) {  // does a string whose opening quote is token q sit in key position?
    const int pp = prev_sig(tok, q);
    if (pp < 0) return false;
    return tk_is(tok[pp], '{') || (tk_is(tok[pp], ',') && top_obj);
  };
  if (t & TK_OPEN) return key_position(p) ? G_STRK : G_STRV;
  if (t & TK_CLOSE) return key_position(p - 1) ? G_COLON : (depth ? G_AFTER : G_END);
  const uint32_t b = tk_byte(t);
  if (b == '{') return G_OBJ0;
  if (b == '[') return G_ARR0;
  if (b == ':') return G_VAL;
  if (b == ',') return top_obj ? G_KEY : G_VAL;
  if (b == '}' || b == ']') return depth ? G_AFTER : G_END;
  // a literal or number ends at p. Blanks in between: whoever owns the first blank ended it. Otherwise replay the run.
  if (p != k0 - 1) return G_AFTER;
  int s = p;
  while (s > 0 && tk_scalar(tok[s - 1])) {
    if (p - s >= 64) return G_ERR;  // a literal / number longer than this: exact engine
    s--;
  }
  uint32_t g = value_start(tok[s]);
  for (int j = s + 1; j <= p && g != G_ERR; j++) {
    if (!g_scalar_state(g)) return G_ERR;  // bytes glued to a finished literal
    const uint32_t n = scalar_step(g, tk_byte(tok[j]));
    g = n == 0xffu ? G_ERR : n;
  }
  return g;
}

// any backslash among bytes [s, e) of the document? bmap: the lanes' backslash masks, word i = bytes [32 i, 32 i + 32)
ARKS_HD bool any_backslash(const uint32_t* bmap, uint32_t s, uint32_t e) {
  if (e <= s) return false;
  for (uint32_t w = s >> 5; w <= (e - 1) >> 5; w++) {
    uint32_t m = bmap[w];
    if (w == (s >> 5)) m &= 0xffffffffu << (s & 31);
    if (w == ((e - 1) >> 5)) m &= 0xffffffffu >> (31 - ((e - 1) & 31));
    if (m) return true;
  }
  return false;
}

// ---- extraction (run by the lane whose chunk holds the member's key) ----
ARKS_HD uint64_t key_fhash(const uint8_t* doc, uint32_t pos, uint32_t n) {
  uint64_t h = 0x811c9dc5ull;
  for (uint32_t i = 0; i < n; i++) h = fhash_step(h, doc[pos + i]);
  return h;
}
ARKS_HD bool key_equals(const uint8_t* doc, uint32_t pos, uint32_t n, const char* lit) {
  for (uint32_t i = 0; i < n; i++)
    if (doc[pos + i] != (uint8_t)lit[i]) return false;
  return true;
}

struct FastFound {
  uint32_t n_model, n_stream, n_so, n_iu, n_usage, n_u[3];  // how many times each member was met (more than once: exact engine)
  uint32_t bad;
  FastOut o;
};

// value of a member read as string-or-null (model)
ARKS_HD void take_model(const uint32_t* bmap, const uint32_t* tok, int v, int ntok, FastFound& f) {
  f.n_model++;
  if (v >= ntok) { f.bad = 1; return; }
  const uint32_t t = tok[v];
  if (t & TK_OPEN) {
    const uint32_t s = tk_pos(t) + 1, e = tk_pos(tok[v + 1]);  // the closing quote is the next token
    const uint32_t esc = any_backslash(bmap, s, e) ? 1u : 0u;
    f.o.m_start = e > s ? s : 0;
    f.o.m_rawlen = e - s;
    f.o.m_esc = e > s ? esc : 0;
  } else if (tk_byte(t) == 'n') {
    f.o.m_start = f.o.m_rawlen = f.o.m_esc = 0;
  } else {
    f.bad = 1;  // a model of another JSON type is a decode error: the exact engine reports it
  }
}
ARKS_HD uint32_t take_opt_bool(const uint32_t* tok, int v, int ntok, FastFound& f) {
  if (v >= ntok) { f.bad = 1; return 0; }
  const uint32_t b = tk_byte(tok[v]);
  if ((tok[v] & (TK_OPEN | TK_CLOSE)) || !(b == 't' || b == 'f' || b == 'n')) { f.bad = 1; return 0; }
  return b == 'n' ? 0u : b == 'f' ? 1u : 2u;
}
// the members of the object that opens at token v, one lane on its own: fn(key token index, key pos, key len, value token index)
template <class F>
ARKS_HD void mini_members(const uint32_t* tok, int v, int ntok, FastFound& f, F&& fn) {
  uint32_t rel = 1;
  bool expect_key = true;
  int j = v + 1;
  for (uint32_t it = 0; j < ntok; it++, j++) {
    if (it >= kFastMiniCap) { f.bad = 1; return; }
    const uint32_t t = tok[j];
    if (t & TK_OPEN) {
      if (rel == 1 && expect_key) {
        const int c = next_sig(tok, j + 1, ntok);
        fn(j, tk_pos(t) + 1, tk_pos(tok[j + 1]) - tk_pos(t) - 1, next_sig(tok, c, ntok));
        expect_key = false;
      }
      j++;  // the closing quote
      continue;
    }
    const uint32_t b = tk_byte(t);
    if (b == '{' || b == '[') rel++;
    else if (b == '}' || b == ']') { if (--rel == 0) return; }
    else if (b == ',' && rel == 1) expect_key = true;
  }
  f.bad = 1;
}
// a usage counter written as a plain non-negative integer of at most 18 digits; anything else: exact engine (gjson rules)
ARKS_HD bool take_uint(const uint32_t* tok, int v, int ntok, int64_t* out) {
  int64_t acc = 0;
  int n = 0;
  for (int j = v; j < ntok; j++, n++) {
    const uint32_t t = tok[j];
    const uint32_t b = tk_byte(t);
    if ((t & (TK_OPEN | TK_CLOSE)) || (b - '0') > 9u) {
      if (b == '.' || b == 'e' || b == 'E' || b == '-' || b == '+') return false;
      break;
    }
    if (n >= 18) return false;
    acc = acc * 10 + (int64_t)(b - '0');
  }
  if (n == 0) return false;
  *out = acc;
  return true;
}

// a key string met by the walk with `depth` levels open (the key's own object included); k = its opening-quote token
template <int KIND>
ARKS_HD void fast_on_key(const uint8_t* doc, const uint32_t* bmap, const uint32_t* tok, int k, int ntok, uint32_t depth, FastFound& f) {
  if (depth != 1) return;  // only members of the top-level object are read here; nested ones by the mini walks
  if (k + 1 >= ntok) { f.bad = 1; return; }
  const uint32_t kpos = tk_pos(tok[k]) + 1, klen = tk_pos(tok[k + 1]) - kpos;
  // a key with an escape may DECODE to a field name whatever its raw length: exact engine (json-iterator decodes, then hashes)
  if (any_backslash(bmap, kpos, kpos + klen)) { f.bad = 1; return; }
  if (KIND == K_REQ ? !(klen == 5 || klen == 6 || klen == 14) : klen != 5) return;
  const uint64_t h = key_fhash(doc, kpos, klen);
  const int c = next_sig(tok, k + 1, ntok);
  const int v = next_sig(tok, c, ntok);  // (that token c is the colon is checked by the walk)
  if (h == H_MODEL && klen == 5) { take_model(bmap, tok, v, ntok, f); return; }
  if (KIND == K_REQ) {
    if (h == H_STREAM && klen == 6) { f.n_stream++; f.o.stream3 = take_opt_bool(tok, v, ntok, f); return; }
    if (h == H_SO && klen == 14) {
      f.n_so++;
      if (v >= ntok) { f.bad = 1; return; }
      if (tk_is(tok[v], 'n')) { f.o.so_present = 0; f.o.iu3 = 0; return; }
      if (!tk_is(tok[v], '{')) { f.bad = 1; return; }
      f.o.so_present = 1;
      mini_members(tok, v, ntok, f, [&](int, uint32_t p, uint32_t n, int vv) {
        if (any_backslash(bmap, p, p + n)) { f.bad = 1; return; }
        if (n != 13) return;
        if (key_fhash(doc, p, n) == H_IU) { f.n_iu++; f.o.iu3 = take_opt_bool(tok, vv, ntok, f); }
      });
    }
  } else {
    if (h == H_USAGE && klen == 5) {
      f.n_usage++;
      if (v >= ntok) { f.bad = 1; return; }
      if (!tk_is(tok[v], '{')) return;  // null or any other type: the counters stay 0 (apijson decodes objects only)
      mini_members(tok, v, ntok, f, [&](int, uint32_t p, uint32_t n, int vv) {
        if (any_backslash(bmap, p, p + n)) { f.bad = 1; return; }  // may be an escaped spelling of a counter's name
        int which = -1;
        if (n == 13 && key_equals(doc, p, n, "prompt_tokens")) which = 0;
        else if (n == 17 && key_equals(doc, p, n, "completion_tokens")) which = 1;
        else if (n == 12 && key_equals(doc, p, n, "total_tokens")) which = 2;
        else return;
        f.n_u[which]++;
        if (vv >= ntok || !take_uint(tok, vv, ntok, &f.o.usage[which])) f.bad = 1;
      });
    }
  }
}

// ---- one lane's share of phase 2 (after the effect scan): tokens [k0, k1) with `depth` / `stack` in front of k0 ----
template <int KIND>
ARKS_HD bool fast_walk_chunk(const uint8_t* doc, const uint32_t* bmap, const uint32_t* tok, int k0, int k1, int ntok, uint32_t depth,
                             uint32_t stack, const FastEffect& own, FastFound& f) {
  if (own.npop > depth) return false;  // more closers than open levels (their kinds are checked by the walk below)
  FastWalk w;
  w.depth = depth;
  w.stack = stack;
  w.g = fast_state_before(tok, k0, depth, stack);
  if (w.g == G_ERR) return false;
  for (int k = k0; k < k1; k++) {
    const uint32_t before = w.g;
    if (!w.step(tok[k])) return false;
    if (w.g == G_STRK && before != G_STRK) fast_on_key<KIND>(doc, bmap, tok, k, ntok, w.depth, f);
  }
  if (k1 == ntok) {  // the lane that owns the last token also owns the end of the document
    if (g_scalar_state(w.g)) return false;  // (a top-level scalar is not in the subset anyway)
    if (w.g != G_END) return false;
  }
  return !f.bad;
}

// ---- host reference driver: the same phases with the warp collectives written as loops (tests; the device driver is in
// arks_gateway.cu and uses shuffles / ballots for exactly these steps) ----
#if !defined(__CUDA_ARCH__)
template <int KIND>
inline bool fast_scan_host(const uint8_t* doc, uint32_t len, FastOut& out, uint32_t* tok /* kFastMaxTok + 32 */) {
  if (len == 0 || len > kFastMaxLen) return false;
  uint32_t ntok = 0, carry_esc = 0, carry_str = 0;
  uint32_t bmap[kFastMaxLen / 32];
  for (uint32_t seg = 0; seg * kFastSeg < len; seg++) {
    FastMasks m[32];
    uint32_t co[32], E[32], Qu[32], R[32], TB[32];
    for (int l = 0; l < 32; l++) {
      const uint32_t base = seg * kFastSeg + 32u * l;
      for (int j = 0; j < 8; j++) {
        uint32_t w = 0;
        for (int b = 0; b < 4; b++) {  // a lane that starts inside the document reads 32 bytes of shared memory, past the end too
          const uint32_t p = base + 4 * j + b;
          w |= (uint32_t)(p < len ? doc[p] : base < len ? ARKS_HOST_PAST_END(doc, len, p, (uint8_t)0) : (uint8_t)0) << (8 * b);
        }
        m[l].w[j] = w;
      }
      fast_masks(m[l], base < len ? (len - base < 32 ? len - base : 32) : 0);
      if (m[l].B == 0xffffffffu) return false;  // 32 backslashes in a row: exact engine
      co[l] = odd_tail(m[l].B);
      bmap[seg * 32 + l] = m[l].B;
    }
    uint32_t par = carry_str;
    for (int l = 0; l < 32; l++) {
      E[l] = find_escaped(m[l].B, l ? co[l - 1] : carry_esc);
      Qu[l] = m[l].Q & ~E[l];
      R[l] = prefix_xor32(Qu[l]) ^ (par ? 0xffffffffu : 0u);
      par ^= popc32(Qu[l]) & 1u;
    }
    carry_esc = co[31];
    carry_str = par;
    for (int l = 0; l < 32; l++) {
      const uint32_t base = seg * kFastSeg + 32u * l;
      if (!fast_string_checks(doc, len, base, m[l], E[l], R[l])) return false;
      TB[l] = m[l].V & ~(R[l] & ~Qu[l]);
      if (ntok + popc32(TB[l]) > kFastMaxTok) return false;
      fast_emit(doc, base, TB[l], Qu[l], R[l], tok, ntok);
      ntok += popc32(TB[l]);
    }
  }
  if (carry_str || ntok == 0) return false;
  const int c = (int)((ntok + 31) / 32);
  FastEffect eff[32], pre[32];
  for (int l = 0; l < 32; l++) {
    eff[l] = FastEffect{0, 0, 0, 0, 0};
    for (int k = l * c; k < (l + 1) * c && k < (int)ntok; k++) effect_token(eff[l], tok[k]);
  }
  FastEffect run{0, 0, 0, 0, 0};
  for (int l = 0; l < 32; l++) { pre[l] = run; run = effect_compose(run, eff[l]); }
  if (run.bad) return false;
  FastFound tot{};
  for (int l = 0; l < 32; l++) {
    const int k0 = l * c, k1 = (l + 1) * c < (int)ntok ? (l + 1) * c : (int)ntok;
    if (k0 >= k1) continue;
    if (pre[l].npop) return false;  // more closers than openers
    FastFound f{};
    if (!fast_walk_chunk<KIND>(doc, bmap, tok, k0, k1, (int)ntok, pre[l].npush, pre[l].pword, eff[l], f)) return false;
    // combine: every member at most once in the whole document
    tot.n_model += f.n_model; tot.n_stream += f.n_stream; tot.n_so += f.n_so; tot.n_iu += f.n_iu; tot.n_usage += f.n_usage;
    for (int q = 0; q < 3; q++) tot.n_u[q] += f.n_u[q];
    if (f.n_model) { tot.o.m_start = f.o.m_start; tot.o.m_rawlen = f.o.m_rawlen; tot.o.m_esc = f.o.m_esc; }
    if (f.n_stream) tot.o.stream3 = f.o.stream3;
    if (f.n_so) { tot.o.so_present = f.o.so_present; tot.o.iu3 = f.o.iu3; }
    if (f.n_usage) for (int q = 0; q < 3; q++) tot.o.usage[q] = f.o.usage[q];
  }
  if (tot.n_model > 1 || tot.n_stream > 1 || tot.n_so > 1 || tot.n_iu > 1 || tot.n_usage > 1 || tot.n_u[0] > 1 || tot.n_u[1] > 1 ||
      tot.n_u[2] > 1)
    return false;
  out = tot.o;
  return true;
}
#endif

}  // namespace wd
}  // namespace arks
