// mask_scan.cuh — the fast path of the scan kernels: one lane per document, two CONVERGENT passes (device, sm_90a; host
// build for tests).
//
// json_engine.cuh walks every document through one loop that mixes string skipping, table steps and member hooks, window
// by window: 32 different documents per warp then execute the union of their code paths and wait for the densest one in
// every 128-byte window, with only a third of the lanes active. A warp-per-document formulation (token-balanced, prefix
// scans across lanes, warp_scan.cuh) is correct but slower in bulk — its serial single-lane sections and warp collectives
// cost more than they save. This file keeps a lane per
// document and instead makes every loop body the same for every lane, whatever its document looks like:
//
//   pass A  (32 bytes per step, branch-free)  quote / backslash byte masks (SWAR) -> escaped characters (carry in a
//           register) -> in-string mask (prefix XOR) -> string content checks -> the bitmap of TOKENS (the bytes outside
//           strings plus the opening quote of every string: a string is one token, its closing quote is "next token - 1")
//           goes to a per-lane array. Same instructions for prose, escapes, UTF-8, structure.
//   pass B  one table step per token (about fifty per KiB of chat JSON, not per byte of text):
//           class = CLS[byte]; entry = TAB[state][class] -> next state, push / pop / comma actions on a 32-level bit stack,
//           and three flags that log the members of the top-level object (key span, first byte of the value).
//   pass C  the logged members are matched against the names the gateway reads and their values extracted; the
//           stream_options / usage objects are read by a short token walk.
//   Lanes only differ in trip counts (document length in A, tokens in B, members in C); every block orders its own 128
//   documents by length so that the lanes of a warp get similar ones (the batch itself stays in arrival order).
//
// This path is a FILTER in front of the exact engine, not a second definition of the decoders: it accepts a document only
// if it lies in a conservative subset on which json-iterator (and encoding/json) agree with RFC 8259 — no control bytes
// in strings, valid escapes, RFC numbers and literals, depth <= 32, the top-level value an object, at most kFastMaxLen
// bytes, the members the gateway reads of the expected JSON type, not duplicated and spelled without escapes. Anything
// else (every malformed or unusual document) is handed to json_engine.cuh's automaton, which restates the reference's
// decoders quirk by quirk; so verdicts never depend on which path ran (fuzzed against the engine and the oracle:
// tests/test_mask_scan.py). One theoretical difference: json-iterator matches struct fields by a 64-bit hash of the
// lower-cased key; this path compares the bytes, so a different key colliding with a field's hash (2^-64) is not matched.
#pragma once
#include "json_common.cuh"

namespace arks {

constexpr uint32_t kFastMaxLen = 2048;             // longer documents: exact engine
constexpr uint32_t kFastChunks = kFastMaxLen / 32;
constexpr uint32_t kFastMaxMembers = 8;            // logged members of the top-level object: only keys as long as a name that is
                                                   // read (more of those than this: exact engine)
// key lengths pass C looks at, as a bit mask: model, stream, stream_options / model, usage
constexpr uint32_t kFastKeyLensReq = 1u << 5 | 1u << 6 | 1u << 14, kFastKeyLensResp = 1u << 5;
constexpr uint32_t kFastMiniCap = 192;             // structure bytes read inside stream_options / usage

struct FastOut {
  uint32_t m_start, m_rawlen, m_esc;  // raw span of the model string (0 / 0 / 0: null or absent)
  uint32_t stream3, so_present, iu3;  // K_REQ tri-states: 0 nil, 1 false, 2 true
  int64_t usage[3];                   // K_RESP
};

// Per-lane scratch between the passes, as a strided view: element j of this lane lives at base[j * stride]. On the device
// the arrays are in shared memory, lane-interleaved (stride = threads per block: every access of a warp is conflict-free
// when the lanes use the same j, and no lane ever touches local memory); on the host stride is 1.
struct FastScratch {
  uint32_t* tb_;    // kFastChunks words: the tokens (bytes outside strings + the opening quote of every string)
  uint32_t* mem_;   // 2 * kFastMaxMembers words: key pos | key len << 16, value pos
  uint32_t stride;
  uint32_t bs_lo, bs_hi;  // chunk j contains a backslash (bit j): lets the key / model checks skip the byte scan
  uint32_t nz_lo, nz_hi;  // chunk j has bytes outside strings (tb(j) != 0): the token cursor jumps over the others
  // When two lanes scan one document (the second half is scanned before anybody knows whether it starts inside a string),
  // the words from `flip_from` on were written under the assumption "outside" and are read complemented if that was wrong:
  // for every byte — quote or not — "is a token" is exactly the opposite under the other assumption.
  uint32_t flip_from = 0xffffffffu, last_w = 0, vlast = 0xffffffffu;  // last_w / vlast: last chunk and its valid-byte mask
  ARKS_HD uint32_t& tb(uint32_t j) const { return tb_[j * stride]; }  // the stored word (pass A writes it)
  ARKS_HD uint32_t tbv(uint32_t j) const {                            // the word as passes B / C read it
    const uint32_t raw = tb_[j * stride];
    return j >= flip_from ? (j == last_w ? vlast : 0xffffffffu) & ~raw : raw;
  }
  ARKS_HD uint32_t& mem(uint32_t j) const { return mem_[j * stride]; }
};
// the two chunks pass A has at hand (the current one and the next), as words a lane can index dynamically: shared memory
// on the device (registers cannot be indexed), element k of slot c & 1 at ring[((c & 1) * 8 + k) * stride]
struct FastRing {
  uint32_t* ring;
  uint32_t stride;
  ARKS_HD void put(uint32_t chunk, const uint32_t w[8]) const {
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int k = 0; k < 8; k++) ring[((chunk & 1u) * 8 + k) * stride] = w[k];
  }
  ARKS_HD uint32_t word_at(uint32_t p) const { return ring[((((p >> 5) & 1u) * 8) + ((p >> 2) & 7u)) * stride]; }
  ARKS_HD uint8_t byte_at(uint32_t p) const {  // p inside the current or the next chunk
    return (uint8_t)(word_at(p) >> (8 * (p & 3u)));
  }
  // the four bytes at p .. p+3 as a little-endian word (p + 3 may reach into the next chunk)
  ARKS_HD uint32_t four_at(uint32_t p) const {
    const uint32_t lo = word_at(p), hi = word_at(p + 3), sh = 8 * (p & 3u);
    return sh ? (lo >> sh) | (hi << (32 - sh)) : lo;
  }
};
// are the four bytes of x all hexadecimal digits? SWAR, exact (checked over all 2^32 words): bit 7 of every byte is
// forced on before the subtractions, so no borrow crosses a byte
ARKS_HD bool four_hex(uint32_t x) {
  const uint32_t H = 0x80808080u;
  const uint32_t xs = x | H, ys = x | 0x20202020u | H;
  const uint32_t dig = (xs - 0x30303030u) & ~(xs - 0x3a3a3a3au);  // bit 7: '0' <= byte < ':'
  const uint32_t let = (ys - 0x61616161u) & ~(ys - 0x67676767u);  // bit 7: 'a' <= (byte | 0x20) < 'g'
  return !(x & H) && (((dig | let) & H) == H);
}

// ---- byte-plane SWAR: bit 7 of every byte that is zero, exact ----
ARKS_HD uint32_t zero_bytes(uint32_t x) { return ~(((x & 0x7f7f7f7fu) + 0x7f7f7f7fu) | x) & 0x80808080u; }
ARKS_HD uint32_t plane_nibble(uint32_t t) { return ((t >> 7) * 0x01020408u) >> 24; }  // the 4 flag bits as a nibble

// characters escaped by a backslash (simdjson's find_escaped on 32-bit words); prev: the first byte is escaped from before
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
ARKS_HD uint32_t clz32(uint32_t x) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__clz((int)x);
#else
  return x ? (uint32_t)__builtin_clz(x) : 32u;
#endif
}

// ---- pass A: one 32-byte chunk. w: the bytes as 8 little-endian words; carries live in the caller's registers ----
struct FastCarry {
  uint32_t esc;     // the next chunk's first byte is escaped
  uint32_t in_str;  // the next chunk starts inside a string
  uint32_t bad;
  uint32_t bad_flip;  // the same verdict if the scan had started INSIDE a string instead (second lane of a split document)
};
ARKS_HD void fast_chunk(const uint32_t w[8], uint32_t nvalid, const FastRing& ring, uint32_t len, uint32_t base, FastCarry& c,
                        uint32_t* tb_out, uint32_t* bm_out) {
  uint32_t Q = 0, B = 0, anyc = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int j = 0; j < 8; j++) {
    const uint32_t x = w[j];
    Q |= plane_nibble(zero_bytes(x ^ 0x22222222u)) << (4 * j);
    B |= plane_nibble(zero_bytes(x ^ 0x5c5c5c5cu)) << (4 * j);
    anyc |= (x - 0x20202020u) & ~x;  // bit 7 of a byte < 0x20 (and maybe of a neighbour: only a filter for the exact test)
  }
  anyc &= 0x80808080u;
  const uint32_t V = nvalid >= 32 ? 0xffffffffu : ((1u << nvalid) - 1u);
  Q &= V;
  B &= V;
  // a backslash run that fills the whole chunk keeps the carry as it is (32 is even); otherwise the carry out is the
  // parity of the run that touches the chunk's end (its first backslash cannot be escaped: something else precedes it)
  const uint32_t E = find_escaped(B, c.esc);
  // the byte after the chunk is escaped iff the chunk ends in a backslash that is not itself escaped (find_escaped has the
  // carry in it: this is the parity of the backslash run that touches the chunk's end, without counting it)
  c.esc = (B >> 31) & ~(E >> 31) & 1u;
  const uint32_t Qu = Q & ~E;
  const uint32_t Rraw = prefix_xor32(Qu);
  const uint32_t R = Rraw ^ (c.in_str ? 0xffffffffu : 0u);  // inside a string, opening quote included
  c.in_str ^= Rraw >> 31;                                  // the prefix XOR's top bit is the parity of all quotes
  uint32_t bad = B & ~R;  // a backslash outside a string
  uint32_t bad_flip = B & R;
  if (anyc) {             // rare: some byte < 0x20 in the chunk; inside a string it takes the document off this path
    uint32_t C = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int j = 0; j < 8; j++) C |= plane_nibble(zero_bytes(w[j] & 0xe0e0e0e0u)) << (4 * j);
    bad |= C & V & R;
    bad_flip |= C & V & ~R;
  }
  uint32_t e = E & V;
  while (e) {  // rare: what follows each backslash must be an escape RFC 8259 knows
    const uint32_t p = base + first_set(e);
    e &= e - 1;
    const uint32_t ch = ring.byte_at(p);
    // " \ / b f n r t as one bit test (bytes 0x20..0x7f: a bit per byte in three words); u needs four hex digits
    const uint32_t okw = ch < 0x40 ? 0x00008004u : ch < 0x60 ? 0x10000000u : ch < 0x80 ? 0x00144044u : 0u;  // 0x20-0x3f | 0x40-0x5f | 0x60-0x7f
    const bool simple = ch >= 0x20 && ((okw >> (ch & 31u)) & 1u);
    if (ch == 'u') {
      if (p + 4 >= len || !four_hex(ring.four_at(p + 1))) bad = bad_flip = 1;
    } else if (!simple) {
      bad = bad_flip = 1;
    }
  }
  c.bad |= bad;
  c.bad_flip |= bad_flip;
  // bytes outside strings, plus the OPENING quote of every string (R covers a string from its opening quote to the byte
  // before its closing quote; the closing quote is not a token: whatever follows it is, so "closing quote = next token - 1")
  *tb_out = V & ~(R & ~Qu) & ~(Qu & ~R);
  *bm_out = B;
}

// ---- one document, two lanes (pass A only) ----
// A lane per document means a 64 Ki-document wave is 2 048 warps, 14 per SM, each a dependent chain: the kernel runs at the
// speed of that chain. Pass A's chain is cut in two: lane L scans chunks [0, h), lane H chunks [h, nch) AT THE SAME TIME.
// What H does not know is whether chunk h starts inside a string. It does not need to: it scans as if it started outside,
//   * the escape carry into chunk h only depends on the backslash run at the end of chunk h-1 (H looks at that one chunk),
//   * under the other assumption every byte's "is a token" bit is exactly the complement (see FastScratch::tbv), so H keeps
//     one bitmap and both non-empty-chunk maps, both token counts and both verdicts (FastCarry::bad / bad_flip),
// and when L arrives with the true parity the right variant is picked. Exact, not speculative.
struct FastHalf {  // what lane H hands over
  uint32_t bs_lo, bs_hi;                      // chunks with a backslash
  uint32_t nz0_lo, nz0_hi, nz1_lo, nz1_hi;    // non-empty chunks under either assumption
  uint32_t ntok0, ntok1, bad0, bad1, parity;  // parity: quotes seen are odd
};
// H's first chunk; nch when the document is too short to be worth splitting
ARKS_HD uint32_t fast_split_point(uint32_t nch) { return nch >= 4 ? (nch + 1) / 2 : nch; }
// backslash mask of a chunk (for the escape carry out of chunk h-1)
ARKS_HD uint32_t fast_backslash_mask(const uint32_t w[8], uint32_t nvalid) {
  uint32_t B = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int j = 0; j < 8; j++) B |= plane_nibble(zero_bytes(w[j] ^ 0x5c5c5c5cu)) << (4 * j);
  return B & (nvalid >= 32 ? 0xffffffffu : ((1u << nvalid) - 1u));
}
// escape carry into the chunk after one whose backslash mask is Bprev; a chunk of 32 backslashes would need the chunk
// before it as well: such a document is left to the exact engine
ARKS_HD uint32_t fast_esc_after(uint32_t Bprev, uint32_t* bad) {
  if (Bprev == 0xffffffffu) { *bad = 1; return 0; }
  return clz32(~Bprev) & 1u;
}
// L's own result is in `s` (bs / nz bits of its chunks) and cL; returns false if the document is off this path
ARKS_HD bool fast_split_merge(FastScratch& s, uint32_t len, uint32_t h, const FastCarry& cL, const FastHalf& H, uint32_t* ntok) {
  const uint32_t nch = (len + 31) >> 5, flip = cL.in_str;
  if (cL.bad || (flip ? H.bad1 : H.bad0) || (cL.in_str ^ H.parity)) return false;  // ... or the document ends inside a string
  s.bs_lo |= H.bs_lo; s.bs_hi |= H.bs_hi;
  s.nz_lo |= flip ? H.nz1_lo : H.nz0_lo;
  s.nz_hi |= flip ? H.nz1_hi : H.nz0_hi;
  *ntok += flip ? H.ntok1 : H.ntok0;
  s.flip_from = flip ? h : 0xffffffffu;
  s.last_w = nch - 1;
  const uint32_t tail = len - 32 * (nch - 1);
  s.vlast = tail >= 32 ? 0xffffffffu : ((1u << tail) - 1u);
  return true;
}
// what H accumulates per chunk besides the stored word
ARKS_HD void fast_half_note(FastHalf& H, uint32_t j, uint32_t tbw, uint32_t bm, uint32_t V) {
  const uint32_t bit = 1u << (j & 31), alt = V & ~tbw;
  if (j < 32) { H.bs_lo |= bm ? bit : 0u; H.nz0_lo |= tbw ? bit : 0u; H.nz1_lo |= alt ? bit : 0u; }
  else { H.bs_hi |= bm ? bit : 0u; H.nz0_hi |= tbw ? bit : 0u; H.nz1_hi |= alt ? bit : 0u; }
  H.ntok0 += popc32(tbw);
  H.ntok1 += popc32(alt);
}

// ---- pass B: the grammar as a table ----
enum : uint32_t {
  G_TOP = 0, G_VAL, G_ARR0, G_OBJ0, G_KEY, G_COLON, G_AFTER, G_STRK, G_STRV,
  G_T1, G_T2, G_T3, G_F1, G_F2, G_F3, G_F4, G_N1, G_N2, G_N3,   // literals in progress
  G_NM, G_NZ, G_NI, G_ND, G_NF, G_NE, G_NS, G_NX,               // RFC 8259 number
  G_ERR, G_NSTATES
};
enum : uint32_t {
  C_QUOTE = 0, C_LBRACE, C_RBRACE, C_LBRACK, C_RBRACK, C_COLON, C_COMMA, C_WS, C_MINUS, C_PLUS, C_ZERO, C_DIG19, C_DOT, C_e, C_E,
  C_t, C_r, C_u, C_f, C_a, C_l, C_s, C_n, C_OTHER, C_NCLASSES
};
constexpr uint32_t kFastTabStride = 32;  // classes per row, padded
// entry: next state (5 bits) | action << 5 | flags
enum : uint32_t { A_NONE = 0, A_PUSH_OBJ, A_PUSH_ARR, A_POP_OBJ, A_POP_ARR, A_COMMA, A_ERR };
constexpr uint32_t F_VALSTART = 1u << 8, F_KEYSTART = 1u << 9, F_KEYEND = 1u << 10;

struct FastTables {
  uint8_t cls[256];
  uint16_t tab[G_NSTATES * kFastTabStride];
};
constexpr uint32_t fast_class_of(int b) {
  return b == '"' ? C_QUOTE : b == '{' ? C_LBRACE : b == '}' ? C_RBRACE : b == '[' ? C_LBRACK : b == ']' ? C_RBRACK
       : b == ':' ? C_COLON : b == ',' ? C_COMMA : (b == ' ' || b == '\t' || b == '\n' || b == '\r') ? C_WS
       : b == '-' ? C_MINUS : b == '+' ? C_PLUS : b == '0' ? C_ZERO : (b >= '1' && b <= '9') ? C_DIG19 : b == '.' ? C_DOT
       : b == 'e' ? C_e : b == 'E' ? C_E : b == 't' ? C_t : b == 'r' ? C_r : b == 'u' ? C_u : b == 'f' ? C_f : b == 'a' ? C_a
       : b == 'l' ? C_l : b == 's' ? C_s : b == 'n' ? C_n : C_OTHER;
}
constexpr uint16_t fast_entry(uint32_t next, uint32_t action = A_NONE, uint32_t flags = 0) {
  return (uint16_t)(next | action << 5 | flags);
}
// what a finished value (string, literal, number, container) may be followed by
constexpr uint16_t fast_after(uint32_t c) {
  return c == C_WS ? fast_entry(G_AFTER) : c == C_COMMA ? fast_entry(G_AFTER, A_COMMA) : c == C_RBRACE ? fast_entry(G_AFTER, A_POP_OBJ)
       : c == C_RBRACK ? fast_entry(G_AFTER, A_POP_ARR) : fast_entry(G_ERR, A_ERR);
}
constexpr uint16_t fast_value_start(uint32_t c) {
  return c == C_QUOTE ? fast_entry(G_AFTER, A_NONE, F_VALSTART) : c == C_LBRACE ? fast_entry(G_OBJ0, A_PUSH_OBJ, F_VALSTART)
       : c == C_LBRACK ? fast_entry(G_ARR0, A_PUSH_ARR, F_VALSTART) : c == C_t ? fast_entry(G_T1, A_NONE, F_VALSTART)
       : c == C_f ? fast_entry(G_F1, A_NONE, F_VALSTART) : c == C_n ? fast_entry(G_N1, A_NONE, F_VALSTART)
       : c == C_MINUS ? fast_entry(G_NM, A_NONE, F_VALSTART) : c == C_ZERO ? fast_entry(G_NZ, A_NONE, F_VALSTART)
       : c == C_DIG19 ? fast_entry(G_NI, A_NONE, F_VALSTART) : fast_entry(G_ERR, A_ERR);
}
constexpr uint16_t fast_transition(uint32_t g, uint32_t c) {
  const bool dig = c == C_ZERO || c == C_DIG19, exp = c == C_e || c == C_E;
  switch (g) {
    case G_TOP:   return c == C_WS ? fast_entry(G_TOP) : c == C_LBRACE ? fast_entry(G_OBJ0, A_PUSH_OBJ) : fast_entry(G_ERR, A_ERR);
    case G_VAL:   return c == C_WS ? fast_entry(G_VAL) : fast_value_start(c);
    case G_ARR0:  return c == C_WS ? fast_entry(G_ARR0) : c == C_RBRACK ? fast_entry(G_AFTER, A_POP_ARR) : fast_value_start(c);
    case G_OBJ0:  return c == C_WS ? fast_entry(G_OBJ0) : c == C_QUOTE ? fast_entry(G_COLON, A_NONE, F_KEYSTART)
                       : c == C_RBRACE ? fast_entry(G_AFTER, A_POP_OBJ) : fast_entry(G_ERR, A_ERR);
    case G_KEY:   return c == C_WS ? fast_entry(G_KEY) : c == C_QUOTE ? fast_entry(G_COLON, A_NONE, F_KEYSTART) : fast_entry(G_ERR, A_ERR);
    case G_COLON: return c == C_WS ? fast_entry(G_COLON) : c == C_COLON ? fast_entry(G_VAL) : fast_entry(G_ERR, A_ERR);
    case G_AFTER: return fast_after(c);
    // a string is ONE token, its opening quote (pass A leaves the closing quote out): G_STRK / G_STRV are never entered
    case G_T1: return c == C_r ? fast_entry(G_T2) : fast_entry(G_ERR, A_ERR);
    case G_T2: return c == C_u ? fast_entry(G_T3) : fast_entry(G_ERR, A_ERR);
    case G_T3: return c == C_e ? fast_entry(G_AFTER) : fast_entry(G_ERR, A_ERR);
    case G_F1: return c == C_a ? fast_entry(G_F2) : fast_entry(G_ERR, A_ERR);
    case G_F2: return c == C_l ? fast_entry(G_F3) : fast_entry(G_ERR, A_ERR);
    case G_F3: return c == C_s ? fast_entry(G_F4) : fast_entry(G_ERR, A_ERR);
    case G_F4: return c == C_e ? fast_entry(G_AFTER) : fast_entry(G_ERR, A_ERR);
    case G_N1: return c == C_u ? fast_entry(G_N2) : fast_entry(G_ERR, A_ERR);
    case G_N2: return c == C_l ? fast_entry(G_N3) : fast_entry(G_ERR, A_ERR);
    case G_N3: return c == C_l ? fast_entry(G_AFTER) : fast_entry(G_ERR, A_ERR);
    case G_NM: return c == C_ZERO ? fast_entry(G_NZ) : c == C_DIG19 ? fast_entry(G_NI) : fast_entry(G_ERR, A_ERR);
    case G_NZ: return c == C_DOT ? fast_entry(G_ND) : exp ? fast_entry(G_NE) : dig ? fast_entry(G_ERR, A_ERR) : fast_after(c);
    case G_NI: return dig ? fast_entry(G_NI) : c == C_DOT ? fast_entry(G_ND) : exp ? fast_entry(G_NE) : fast_after(c);
    case G_ND: return dig ? fast_entry(G_NF) : fast_entry(G_ERR, A_ERR);
    case G_NF: return dig ? fast_entry(G_NF) : exp ? fast_entry(G_NE) : fast_after(c);
    case G_NE: return dig ? fast_entry(G_NX) : (c == C_PLUS || c == C_MINUS) ? fast_entry(G_NS) : fast_entry(G_ERR, A_ERR);
    case G_NS: return dig ? fast_entry(G_NX) : fast_entry(G_ERR, A_ERR);
    case G_NX: return dig ? fast_entry(G_NX) : fast_after(c);
    default:   return fast_entry(G_ERR, A_ERR);
  }
}
struct FastTablesInit {
  FastTables t;
  constexpr FastTablesInit() : t() {
    for (int b = 0; b < 256; b++) t.cls[b] = (uint8_t)fast_class_of(b);
    for (uint32_t g = 0; g < G_NSTATES; g++)
      for (uint32_t c = 0; c < kFastTabStride; c++) t.tab[g * kFastTabStride + c] = c < C_NCLASSES ? fast_transition(g, c) : fast_entry(G_ERR, A_ERR);
  }
};

// position of the first byte outside strings at or after `from` (an absolute byte position), or `none`
ARKS_HD uint32_t next_token(const FastScratch& s, uint32_t nch, uint32_t from, uint32_t none) {
  uint32_t w = from >> 5;
  if (w >= nch) return none;
  uint32_t m = s.tbv(w) & (0xffffffffu << (from & 31));
  while (!m) {
    if (++w >= nch) return none;
    m = s.tbv(w);
  }
  return w * 32 + first_set(m);
}
// any backslash among bytes [b, e)? The per-chunk summary answers "no" without touching the document in the usual case.
// the three helpers below are called from a dozen places with loops inside: inlined they were 3 300 of the request kernel's
// 9 000 SASS instructions, and a kernel whose warps each sit somewhere else in 144 KB of code waits for the instruction
// cache more than for anything else (ncu: stall_no_instruction on top). One copy each.
ARKS_OUTLINE bool any_backslash_bytes(const uint8_t* doc, uint32_t b, uint32_t e) {
  uint32_t d = 0;
  for (uint32_t i = b; i < e; i++) d |= doc[i] == '\\';
  return d != 0;
}
ARKS_HD bool any_backslash(const uint8_t* doc, const FastScratch& s, uint32_t b, uint32_t e) {
  if (e <= b) return false;
  const uint32_t c0 = b >> 5, c1 = (e - 1) >> 5;  // the chunks the span lies in, tested without a loop
  const uint64_t m = (~0ull << c0) & (~0ull >> (63 - c1));
  if (!(((uint64_t)s.bs_hi << 32 | s.bs_lo) & m)) return false;
  return any_backslash_bytes(doc, b, e);
}
// case-folded comparison with a lower-case literal (json-iterator's struct fields), exact comparison (gjson's Map())
// Key comparison against a literal of at most 24 bytes: the document's bytes are fetched with 24 independent (predicated) loads
// and compared as three 64-bit words — one trip to memory instead of a loop that pays one per byte (ncu had the byte loop
// as the kernel's hottest source line). The literal travels as packed words made at compile time.
struct KeyLit {
  uint64_t w[3];
};
ARKS_HD constexpr KeyLit key_lit(const char* s, int n) {
  KeyLit k{{0, 0, 0}};
  for (int i = 0; i < n; i++) k.w[i >> 3] |= (uint64_t)(uint8_t)s[i] << (8 * (i & 7));
  return k;
}
// fold: ASCII letters of the document compare case-insensitively with a lower-case literal (json-iterator's struct fields);
// otherwise exact (gjson's Map())
ARKS_OUTLINE bool key_equals(const uint8_t* doc, uint32_t pos, uint32_t n, uint64_t l0, uint64_t l1, uint64_t l2, bool fold) {
  uint64_t d[3] = {0, 0, 0};
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (uint32_t i = 0; i < 24; i++) {
    uint32_t c = i < n ? doc[pos + i] : 0u;
    if (fold && (c - 'A') <= 25u) c += 32;
    d[i >> 3] |= (uint64_t)c << (8 * (i & 7));
  }
  return ((d[0] ^ l0) | (d[1] ^ l1) | (d[2] ^ l2)) == 0;
}
#define ARKS_KEY_IS(doc, pos, n, lit, fold) \
  ([&]() { constexpr KeyLit k_ = key_lit(lit, (int)sizeof(lit) - 1); return key_equals(doc, pos, n, k_.w[0], k_.w[1], k_.w[2], fold); }())
#define key_is_fold(doc, pos, n, lit) ARKS_KEY_IS(doc, pos, n, lit, true)
#define key_is(doc, pos, n, lit) ARKS_KEY_IS(doc, pos, n, lit, false)

// ---- pass B: walk the bytes outside strings through the grammar; logs the members of the top-level object ----
// Which byte comes next depends only on the bitmap, not on the grammar state, so the bytes are fetched kFastAhead at a time
// (independent loads: the lane's memory latency is paid once per group, not once per byte) and then stepped in order.
constexpr int kFastAhead = 8;
struct TokCursor {  // iterates the set bits of the tb bitmap, jumping over empty chunks with the nz bitmap
  uint32_t w, cur, nz_lo, nz_hi;
  ARKS_HD void init(const FastScratch& s, uint32_t nch, uint32_t from) {
    w = from >> 5;
    cur = w < nch ? (s.tbv(w) & (0xffffffffu << (from & 31))) : 0;
    // chunks after w that are not empty
    const uint64_t nz = ((uint64_t)s.nz_hi << 32 | s.nz_lo) & (w >= 63 ? 0ull : ~0ull << (w + 1));
    nz_lo = (uint32_t)nz;
    nz_hi = (uint32_t)(nz >> 32);
  }
  ARKS_HD bool next(const FastScratch& s, uint32_t* pos) {
    if (!cur) {
      if (nz_lo) { w = first_set(nz_lo); nz_lo &= nz_lo - 1; }
      else if (nz_hi) { w = 32 + first_set(nz_hi); nz_hi &= nz_hi - 1; }
      else return false;
      cur = s.tbv(w);
    }
    *pos = w * 32 + first_set(cur);
    cur &= cur - 1;
    return true;
  }
};
// kFastAhead tokens fetched together: the byte loads go out back to back (which byte comes next depends only on the bitmap),
// then the grammar steps run over them in a loop that exists ONCE — positions and bytes travel packed in four registers,
// because eight inlined copies of the step were 24 KB of code and the warps of this kernel stall on instruction fetch more
// than on anything else (they are few and each sits somewhere else in the code).
struct TokBatch {
  uint64_t by, p0, p1;  // 8 bytes; 8 positions of 16 bits
  ARKS_HD int fetch(TokCursor& tc, const FastScratch& s, const uint8_t* doc) {
    uint32_t pos[kFastAhead], b[kFastAhead];
    int n = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int q = 0; q < kFastAhead; q++) {
      pos[q] = 0;
      const bool have = tc.next(s, &pos[q]);
      b[q] = have ? doc[pos[q]] : 0u;
      n += have;
    }
    by = (uint64_t)(b[0] | b[1] << 8 | b[2] << 16 | b[3] << 24) | (uint64_t)(b[4] | b[5] << 8 | b[6] << 16 | b[7] << 24) << 32;
    p0 = (uint64_t)(pos[0] | pos[1] << 16) | (uint64_t)(pos[2] | pos[3] << 16) << 32;
    p1 = (uint64_t)(pos[4] | pos[5] << 16) | (uint64_t)(pos[6] | pos[7] << 16) << 32;
    return n;
  }
  ARKS_HD uint32_t byte(int q) const { return (uint32_t)(by >> (8 * q)) & 0xffu; }
  ARKS_HD uint32_t pos(int q) const { return (uint32_t)((q < 4 ? p0 : p1) >> (16 * (q & 3))) & 0xffffu; }
};
static_assert(kFastAhead == 8 && kFastMaxLen <= 65536, "TokBatch packs 8 positions of 16 bits");
// returns the number of members logged, or -1 (not in the subset)
// key_lens: only members whose raw key length has its bit set are logged (the others cannot spell a name that is read —
// unless they contain an escape, which sends the document to the exact engine here as it would in pass C)
// WALK: 8 = the step inlined eight times behind the eight loads (no packing, 24 KB of code); 0 = one copy of the step in a
// loop over a packed batch (the instruction cache's friend). Same results; which one is faster is a measurement (DESIGN.md).
template <int WALK>
ARKS_HD int fast_walk(const uint8_t* doc, const FastTables& T, const FastScratch& s, uint32_t nch, uint32_t key_lens) {
  uint32_t g = G_TOP, depth = 0, stack = 0, nmem = 0, nsus = 0, kstart = 0, pending = 0, bad = 0, keyopen = 0;
  const uint64_t bs64 = (uint64_t)s.bs_hi << 32 | s.bs_lo;
  TokCursor tc;
  tc.init(s, nch, 0);
  // (A version of this step without branches — selects and predicated stores only — was measured too: same time for
  // requests, 5 % slower for completions; the kernel is bound by the latency of each lane's dependent chain, not by the
  // instructions the diverged branches add. DESIGN.md section 5.)
  auto step = [&](uint32_t pq, uint32_t byte) {
    const uint32_t e = T.tab[g * kFastTabStride + T.cls[byte]];
    const uint32_t act = (e >> 5) & 7u;
    g = e & 31u;
    const bool top_obj = depth && ((stack >> (depth - 1)) & 1u);
    // members of the top-level object: key span and the first byte of the value (depth is still the one BEFORE a push).
    // A key is one token (its opening quote); it ends one byte before whatever token comes next.
    if (keyopen) {  // this token is the first after a top-level key: the key's closing quote sits right before it
      keyopen = 0;
      const uint32_t klen = pq - 1 - kstart;
      if (klen < 32 && (key_lens >> klen & 1u)) {  // pass C compares it (and checks it for escapes)
        if (nmem + nsus >= kFastMaxMembers) bad = 1;
        else { s.mem(2 * nmem) = kstart | klen << 16; pending = 1; }
      } else if (klen) {
        // another length: only an escape could make it spell a name that is read. The chunks it lies in are tested
        // here without a loop; the few keys that share a chunk with a backslash are parked (from the top of the
        // member log down) and looked at byte by byte after the walk, outside this loop
        const uint32_t c0 = kstart >> 5, c1 = (pq - 2) >> 5;
        const uint64_t m = (~0ull << c0) & (~0ull >> (63 - c1));
        if (bs64 & m) {
          if (nmem + nsus >= kFastMaxMembers) bad = 1;
          else { s.mem(2 * (kFastMaxMembers - 1 - nsus)) = kstart | klen << 16; nsus++; }
        }
      }
    }
    if ((e & (F_KEYSTART | F_VALSTART)) && depth == 1) {
      if (e & F_KEYSTART) { kstart = pq + 1; keyopen = 1; pending = 0; }
      if ((e & F_VALSTART) && pending) { s.mem(2 * nmem + 1) = pq; nmem++; pending = 0; }
    }
    if (act == A_PUSH_OBJ || act == A_PUSH_ARR) {
      if (depth >= 32) bad = 1;
      else { stack = (stack & ~(1u << depth)) | ((act == A_PUSH_OBJ ? 1u : 0u) << depth); depth++; }
    } else if (act == A_POP_OBJ || act == A_POP_ARR) {
      if (!depth || top_obj != (act == A_POP_OBJ)) bad = 1;
      else depth--;
    } else if (act == A_COMMA) {
      if (!depth) bad = 1;
      g = top_obj ? G_KEY : G_VAL;
    } else if (act == A_ERR) {
      bad = 1;
    }
  };
  for (;;) {
    int n = 0;
    if (WALK == 8) {
      uint32_t pos[kFastAhead], by[kFastAhead];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
      for (int q = 0; q < kFastAhead; q++) {
        pos[q] = 0;
        const bool have = tc.next(s, &pos[q]);
        by[q] = have ? doc[pos[q]] : 0u;
        n += have;
      }
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
      for (int q = 0; q < kFastAhead; q++)
        if (q < n) step(pos[q], by[q]);
    } else {
      TokBatch tk;
      n = tk.fetch(tc, s, doc);
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
      for (int q = 0; q < n; q++) step(tk.pos(q), tk.byte(q));
    }
    if (bad) return -1;
    if (n < kFastAhead) break;
  }
  // the document is one complete object (numbers cannot be open here: the top-level value is an object)
  if (g != G_AFTER || depth != 0) return -1;
  for (uint32_t k = 0; k < nsus; k++) {  // a top-level key with an escape: the exact engine decodes and compares it
    const uint32_t kk = s.mem(2 * (kFastMaxMembers - 1 - k));
    if (any_backslash_bytes(doc, kk & 0xffffu, (kk & 0xffffu) + (kk >> 16))) return -1;
  }
  return (int)nmem;
}

// ---- pass C: the logged members -> what the gateway reads ----
// the members of the object whose '{' is at `open`, for stream_options (K_REQ) / usage (K_RESP); false: not in the subset
template <int KIND>
ARKS_HD bool fast_inner_object(const uint8_t* doc, const FastScratch& s, uint32_t nch, uint32_t open, FastOut& o) {
  uint32_t rel = 1, keyopen = 0, expect_key = 1, ks = 0, seen = 0, nd = 0, ok = 1, done = 0;
  int which = -1;  // the member whose value is being read: 0..2 usage counters, 3 include_usage
  int64_t acc = 0;
  TokCursor tc;
  tc.init(s, nch, open + 1);
  for (uint32_t it = 0; !done; it += kFastAhead) {
    if (it >= kFastMiniCap) return false;
    TokBatch tk;
    const int n = tk.fetch(tc, s, doc);
    if (n == 0) return false;
#ifdef __CUDA_ARCH__
#pragma unroll 1
#endif
    for (int q = 0; q < n; q++) {
      if (done || !ok) continue;
      const uint32_t p = tk.pos(q);
      const uint8_t b = (uint8_t)tk.byte(q);
      if (keyopen) {  // the first token after a key of this object: the key ended one byte before its closing quote
        keyopen = 0;
        const uint32_t len = p - 1 - ks;
        if (any_backslash(doc, s, ks, p - 1)) { ok = 0; continue; }  // may be an escaped spelling of a name that is read
        which = -1;
        if (KIND == K_REQ) {
          if (len == 13 && key_is_fold(doc, ks, len, "include_usage")) which = 3;
        } else {
          if (len == 13 && key_is(doc, ks, len, "prompt_tokens")) which = 0;
          else if (len == 17 && key_is(doc, ks, len, "completion_tokens")) which = 1;
          else if (len == 12 && key_is(doc, ks, len, "total_tokens")) which = 2;
        }
        if (which >= 0) {
          if (seen & (1u << which)) { ok = 0; continue; }  // duplicates: exact engine
          seen |= 1u << which;
          acc = 0; nd = 0;
        }
      }
      if (b == '"') {  // a whole string (strings are one token)
        if (rel == 1 && expect_key) { expect_key = 0; keyopen = 1; ks = p + 1; }
        else if (rel == 1 && which >= 0) ok = 0;  // a counter / flag written as a string: exact engine (gjson rules)
        continue;
      }
      if (b == '{' || b == '[') {
        if (rel == 1 && which >= 0) ok = 0;
        rel++;
        continue;
      }
      const bool closes = b == '}' || b == ']';
      if (closes || (b == ',' && rel == 1)) {
        if (rel == 1 && which >= 0) {  // the value of a member that is read ends here
          if (which == 3) { if (nd == 0) ok = 0; }
          else if (nd == 0 || nd > 18) ok = 0;
          else if (which == 0) o.usage[0] = acc;  // (no dynamic index: the counters stay in registers)
          else if (which == 1) o.usage[1] = acc;
          else o.usage[2] = acc;
          which = -1;
        }
        if (closes) { if (--rel == 0) done = 1; }
        else expect_key = 1;
        continue;
      }
      if (rel == 1 && which >= 0 && b != ':' && !(b == ' ' || b == '\t' || b == '\n' || b == '\r')) {
        if (which == 3) {  // OptionalDecoder{boolCodec}: true / false / null (the grammar pass checked the spelling)
          if (nd == 0) {
            if (!(b == 't' || b == 'f' || b == 'n')) ok = 0;
            o.iu3 = b == 'n' ? 0u : b == 'f' ? 1u : 2u;
          }
          nd++;
        } else {  // a plain non-negative integer; anything else (sign, fraction, exponent, literal): exact engine
          if ((uint32_t)(b - '0') > 9u) ok = 0;
          acc = (int64_t)((uint64_t)acc * 10u + (uint64_t)(b - '0'));  // wraps past 18 digits; such a value is declined below
          nd++;
        }
      }
    }
    if (!ok) return false;
    if (n < kFastAhead && !done) return false;
  }
  return true;
}

template <int KIND>
ARKS_HD bool fast_members(const uint8_t* doc, const FastScratch& s, uint32_t nch, int nmem, FastOut& o) {
  o.m_start = o.m_rawlen = o.m_esc = 0;
  o.stream3 = o.so_present = o.iu3 = 0;
  o.usage[0] = o.usage[1] = o.usage[2] = 0;
  uint32_t seen = 0;  // bit 0 model, 1 stream, 2 stream_options, 3 usage
  for (int m = 0; m < nmem; m++) {
    const uint32_t kk = s.mem(2 * m), vpos = s.mem(2 * m + 1);
    const uint32_t kpos = kk & 0xffffu, klen = kk >> 16;
    // a key with an escape may DECODE to a field name whatever its raw length: exact engine (json-iterator decodes, then hashes)
    if (any_backslash(doc, s, kpos, kpos + klen)) return false;
    int what = -1;
    if (klen == 5 && key_is_fold(doc, kpos, 5, "model")) what = 0;
    else if (KIND == K_REQ && klen == 6 && key_is_fold(doc, kpos, 6, "stream")) what = 1;
    else if (KIND == K_REQ && klen == 14 && key_is_fold(doc, kpos, 14, "stream_options")) what = 2;
    else if (KIND == K_RESP && klen == 5 && key_is_fold(doc, kpos, 5, "usage")) what = 3;
    if (what < 0) continue;
    if (seen & (1u << what)) return false;  // duplicated members: exact engine (last-wins / pointer-reuse rules)
    seen |= 1u << what;
    const uint8_t vb = doc[vpos];
    if (what == 0) {  // stringCodec: string or null
      if (vb == '"') {
        const uint32_t after = next_token(s, nch, vpos + 1, 0xffffffffu);  // the first token behind the string ...
        if (after == 0xffffffffu) return false;
        const uint32_t end = after - 1;                                      // ... and its closing quote right before it
        o.m_rawlen = end - vpos - 1;
        o.m_start = o.m_rawlen ? vpos + 1 : 0;
        o.m_esc = o.m_rawlen && any_backslash(doc, s, vpos + 1, end) ? 1u : 0u;
      } else if (vb != 'n') {
        return false;  // a model of another JSON type is a decode error: the exact engine reports it
      }
    } else if (what == 1) {
      if (!(vb == 't' || vb == 'f' || vb == 'n')) return false;
      o.stream3 = vb == 'n' ? 0u : vb == 'f' ? 1u : 2u;
    } else if (what == 2) {
      if (vb == '{') {
        o.so_present = 1;
        if (!fast_inner_object<K_REQ>(doc, s, nch, vpos, o)) return false;
      } else if (vb != 'n') {
        return false;
      }
    } else {
      if (vb == '{' && !fast_inner_object<K_RESP>(doc, s, nch, vpos, o)) return false;
      // null or any other type: the counters stay 0 (apijson decodes objects only)
    }
  }
  return true;
}

// ---- host reference driver: exactly what one lane does (tests) ----
#if !defined(__CUDA_ARCH__)
static const FastTablesInit kFastTablesHost{};
template <int KIND>
inline bool fast_scan_host(const uint8_t* doc, uint32_t len, FastOut& out) {
  if (len == 0 || len > kFastMaxLen) return false;
  static thread_local uint32_t tb[kFastChunks], mem[2 * kFastMaxMembers], ringw[16];
  FastScratch s{tb, mem, 1, 0, 0, 0, 0};
  const FastRing ring{ringw, 1};
  const uint32_t nch = (len + 31) / 32;
  FastCarry c{0, 0, 0, 0};
  auto words_of = [&](uint32_t j, uint32_t w[8]) {
    for (int q = 0; q < 8; q++) {
      uint32_t v = 0;
      for (int b = 0; b < 4; b++) {
        const uint32_t p = 32 * j + 4 * q + b;
        v |= (uint32_t)(p < len ? doc[p] : ARKS_HOST_PAST_END(doc, len, p, (uint8_t)(0xA5 ^ p))) << (8 * b);  // garbage past the end, as on the device
      }
      w[q] = v;
    }
  };
  uint32_t w[8], wn[8];
  words_of(0, w);
  ring.put(0, w);
  for (uint32_t j = 0; j < nch; j++) {
    uint32_t bm;
    words_of(j + 1, wn);
    ring.put(j + 1, wn);  // the chunk after the current one is at hand too (a \uXXXX may straddle the boundary)
    fast_chunk(w, len - 32 * j < 32 ? len - 32 * j : 32, ring, len, 32 * j, c, &s.tb(j), &bm);
    if (bm) { if (j < 32) s.bs_lo |= 1u << j; else s.bs_hi |= 1u << (j - 32); }
    if (s.tb(j)) { if (j < 32) s.nz_lo |= 1u << j; else s.nz_hi |= 1u << (j - 32); }
    for (int q = 0; q < 8; q++) w[q] = wn[q];
  }
  if (c.bad || c.in_str) return false;
  const int nmem = fast_walk<0>(doc, kFastTablesHost.t, s, nch, KIND == K_REQ ? kFastKeyLensReq : kFastKeyLensResp);
  if (nmem < 0) return false;
  return fast_members<KIND>(doc, s, nch, nmem, out);
}
// the same with pass A done the way two lanes do it (first half, second half under the "outside a string" assumption, merge)
template <int KIND>
inline bool fast_scan_host_split(const uint8_t* doc, uint32_t len, FastOut& out) {
  if (len == 0 || len > kFastMaxLen) return false;
  static thread_local uint32_t tb[kFastChunks], mem[2 * kFastMaxMembers], ringw[16];
  FastScratch s{tb, mem, 1, 0, 0, 0, 0};
  const FastRing ring{ringw, 1};
  const uint32_t nch = (len + 31) / 32, h = fast_split_point(nch);
  auto words_of = [&](uint32_t j, uint32_t w[8]) {
    for (int q = 0; q < 8; q++) {
      uint32_t v = 0;
      for (int b = 0; b < 4; b++) {
        const uint32_t p = 32 * j + 4 * q + b;
        v |= (uint32_t)(p < len ? doc[p] : ARKS_HOST_PAST_END(doc, len, p, (uint8_t)(0xA5 ^ p))) << (8 * b);
      }
      w[q] = v;
    }
  };
  auto nvalid = [&](uint32_t j) { return len - 32 * j < 32 ? len - 32 * j : 32u; };
  uint32_t w[8], wn[8], ntok = 0;
  FastCarry cL{0, 0, 0, 0};
  for (uint32_t j = 0; j < h; j++) {  // lane L
    uint32_t bm;
    words_of(j, w); words_of(j + 1, wn);
    ring.put(j, w); ring.put(j + 1, wn);
    fast_chunk(w, nvalid(j), ring, len, 32 * j, cL, &s.tb(j), &bm);
    if (bm) { if (j < 32) s.bs_lo |= 1u << j; else s.bs_hi |= 1u << (j - 32); }
    if (s.tb(j)) { if (j < 32) s.nz_lo |= 1u << j; else s.nz_hi |= 1u << (j - 32); }
    ntok += popc32(s.tb(j));
  }
  FastHalf H{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (h < nch) {  // lane H
    FastCarry cH{0, 0, 0, 0};
    words_of(h - 1, w);
    cH.esc = fast_esc_after(fast_backslash_mask(w, 32), &cH.bad);
    cH.bad_flip = cH.bad;
    for (uint32_t j = h; j < nch; j++) {
      uint32_t bm;
      words_of(j, w); words_of(j + 1, wn);
      ring.put(j, w); ring.put(j + 1, wn);
      fast_chunk(w, nvalid(j), ring, len, 32 * j, cH, &s.tb(j), &bm);
      fast_half_note(H, j, s.tb(j), bm, nvalid(j) >= 32 ? 0xffffffffu : ((1u << nvalid(j)) - 1u));
    }
    H.bad0 = cH.bad; H.bad1 = cH.bad_flip; H.parity = cH.in_str;
  }
  if (!fast_split_merge(s, len, h, cL, H, &ntok)) return false;
  const int nmem = fast_walk<0>(doc, kFastTablesHost.t, s, nch, KIND == K_REQ ? kFastKeyLensReq : kFastKeyLensResp);
  if (nmem < 0) return false;
  return fast_members<KIND>(doc, s, nch, nmem, out);
}
#endif

}  // namespace arks
