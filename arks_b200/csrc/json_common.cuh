// json_common.cuh — pieces shared by the JSON / SSE engine (json_engine.cuh): field hashes of the decoders the reference
// uses, escape decoding, the out-of-line slow paths, and the SWAR byte masks used to skip ordinary string bytes.
// Host + device: tests/ compiles the engine with g++ and fuzzes it against the oracle on CPU.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define ARKS_HD __host__ __device__ __forceinline__
// rare paths are kept out of line as PURE functions of plain values (never of the machine object, whose address must
// not be taken or its fields leave the register file): keeps them from being speculated into the per-byte path
#define ARKS_OUTLINE __host__ __device__ __noinline__
#else
#define ARKS_HD inline
#define ARKS_OUTLINE inline
#endif

// Host drivers of the scan filters (mask_scan.cuh, warp_scan.cuh; tests only): the byte they see at position p >= len of
// a document, where the device reads whatever the staging buffer holds (the padding, the next body, stale bytes). `dflt`
// is the driver's own fill; a test defines this to hand over the bytes that follow the body in its buffer instead.
#ifndef ARKS_HOST_PAST_END
#define ARKS_HOST_PAST_END(doc, len, p, dflt) (dflt)
#endif

namespace arks {

enum : uint8_t { K_REQ = 0, K_RESP = 1, K_EVT = 2 };
// how the next value of an S / X member is consumed
enum : uint8_t { VM_SKIP = 0, VM_MODEL, VM_BOOL_STREAM, VM_BOOL_IU, VM_SO, VM_USAGE, VM_UINT, VM_ECHOICES };
// special object one level below the top-level object
enum : uint8_t { L2_NONE = 0, L2_SO, L2_USAGE };

static constexpr uint32_t kMaxDepth = 10000;  // jsoniter maxDepth == encoding/json maxNestingDepth
static constexpr uint32_t kStackWords = (kMaxDepth + 15) / 16 + 1;  // 2 bits per level (json_engine.cuh)

// jsoniter readFieldHash: int64 0x811c9dc5, ^= lower(byte), *= 0x1000193 (iter_object.go)
ARKS_HD constexpr uint64_t fhash_step(uint64_t h, uint8_t b) {
  return (h ^ (uint64_t)((b >= 'A' && b <= 'Z') ? b + 32 : b)) * 0x1000193ull;
}
ARKS_HD constexpr uint64_t fhash_lit(const char* s, int n) {
  uint64_t h = 0x811c9dc5ull;
  for (int i = 0; i < n; i++) h = fhash_step(h, (uint8_t)s[i]);
  return h;
}
static constexpr uint64_t H_MODEL = fhash_lit("model", 5);
static constexpr uint64_t H_STREAM = fhash_lit("stream", 6);
static constexpr uint64_t H_SO = fhash_lit("stream_options", 14);
static constexpr uint64_t H_IU = fhash_lit("include_usage", 13);
static constexpr uint64_t H_USAGE = fhash_lit("usage", 5);

// exact-key candidates (gjson Map(): case-sensitive, unescaped)
ARKS_HD constexpr uint64_t xhash_step(uint64_t h, uint8_t b) { return (h ^ (uint64_t)b) * 0x100000001b3ull; }
ARKS_HD constexpr uint64_t xhash_lit(const char* s, int n) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (int i = 0; i < n; i++) h = xhash_step(h, (uint8_t)s[i]);
  return h;
}
// ids: 0 prompt_tokens 1 completion_tokens 2 total_tokens 3 error 4 choices 5 usage
ARKS_HD const char* xkey_str(int id) {
  switch (id) {
    case 0: return "prompt_tokens";
    case 1: return "completion_tokens";
    case 2: return "total_tokens";
    case 3: return "error";
    case 4: return "choices";
    default: return "usage";
  }
}
ARKS_HD constexpr int xkey_len(int id) { return id == 0 ? 13 : id == 1 ? 17 : id == 2 ? 12 : id == 3 ? 5 : id == 4 ? 7 : 5; }
// bytes [8w, 8w+8) of a key literal as a little-endian word (zero padded): exact comparison against immediates
ARKS_HD constexpr uint64_t lit_word(const char* s, int n, int w) {
  uint64_t v = 0;
  for (int i = 0; i < 8; i++)
    if (8 * w + i < n) v |= (uint64_t)(uint8_t)s[8 * w + i] << (8 * i);
  return v;
}
ARKS_HD constexpr uint64_t xkey_word(int id, int w) {
  return id == 0 ? lit_word("prompt_tokens", 13, w) : id == 1 ? lit_word("completion_tokens", 17, w)
       : id == 2 ? lit_word("total_tokens", 12, w) : id == 3 ? lit_word("error", 5, w)
       : id == 4 ? lit_word("choices", 7, w) : lit_word("usage", 5, w);
}
static constexpr uint64_t X_PROMPT = xhash_lit("prompt_tokens", 13);
static constexpr uint64_t X_COMPL = xhash_lit("completion_tokens", 17);
static constexpr uint64_t X_TOTAL = xhash_lit("total_tokens", 12);
static constexpr uint64_t X_ERROR = xhash_lit("error", 5);
static constexpr uint64_t X_CHOICES = xhash_lit("choices", 7);
static constexpr uint64_t X_USAGE = xhash_lit("usage", 5);

ARKS_HD bool is_ws(uint8_t c) { return c == ' ' || c == '\n' || c == '\t' || c == '\r'; }
ARKS_HD bool is_digit(uint8_t c) { return (uint8_t)(c - '0') <= 9; }
ARKS_HD int hexval(uint8_t c) {
  if (is_digit(c)) return c - '0';
  uint8_t l = c | 0x20;
  if (l >= 'a' && l <= 'f') return l - 'a' + 10;
  return -1;
}

// ---- slow paths over an already validated raw string span (only when the span contains a backslash) ----
// Decodes jsoniter-style (readEscapedChar: surrogate pairing, lone surrogates -> U+FFFD) and feeds every
// output byte to `f`. The span is known to be well-formed.
template <class F>
ARKS_HD void decode_span(const uint8_t* p, uint32_t n, F&& f) {
  auto put_rune = [&](uint32_t r) {
    if (r <= 0x7F) {
      f((uint8_t)r);
    } else if (r <= 0x7FF) {
      f((uint8_t)(0xC0 | (r >> 6)));
      f((uint8_t)(0x80 | (r & 0x3F)));
    } else {
      if (r > 0x10FFFF || (r >= 0xD800 && r <= 0xDFFF)) r = 0xFFFD;
      if (r <= 0xFFFF) {
        f((uint8_t)(0xE0 | (r >> 12)));
        f((uint8_t)(0x80 | ((r >> 6) & 0x3F)));
        f((uint8_t)(0x80 | (r & 0x3F)));
      } else {
        f((uint8_t)(0xF0 | (r >> 18)));
        f((uint8_t)(0x80 | ((r >> 12) & 0x3F)));
        f((uint8_t)(0x80 | ((r >> 6) & 0x3F)));
        f((uint8_t)(0x80 | (r & 0x3F)));
      }
    }
  };
  auto u4 = [&](uint32_t i) {
    return (uint32_t)((hexval(p[i]) << 12) | (hexval(p[i + 1]) << 8) | (hexval(p[i + 2]) << 4) | hexval(p[i + 3]));
  };
  uint32_t i = 0;
  while (i < n) {
    uint8_t c = p[i++];
    if (c != '\\') {
      f(c);
      continue;
    }
    uint8_t e = p[i++];
    for (;;) {  // readEscapedChar, with its tail call unrolled into this loop
      if (e == 'u') {
        uint32_t r = u4(i);
        i += 4;
        if (r >= 0xD800 && r <= 0xDFFF) {
          if (i >= n || p[i] != '\\') {
            put_rune(r);
            break;
          }
          i++;  // the backslash
          e = p[i++];
          if (e != 'u') {
            put_rune(r);
            continue;  // readEscapedChar(e)
          }
          uint32_t r2 = u4(i);
          i += 4;
          if (r < 0xDC00 && r2 >= 0xDC00 && r2 < 0xE000) {
            put_rune((((r - 0xD800) << 10) | (r2 - 0xDC00)) + 0x10000);
          } else {
            put_rune(r);
            put_rune(r2);
          }
        } else {
          put_rune(r);
        }
        break;
      }
      uint8_t o = e;  // " \ / stay themselves
      if (e == 'b') o = '\b';
      else if (e == 'f') o = '\f';
      else if (e == 'n') o = '\n';
      else if (e == 'r') o = '\r';
      else if (e == 't') o = '\t';
      f(o);
      break;
    }
  }
}

// ---- out-of-line slow paths (pure functions) ----
// exact comparison of a raw (validated) key span with candidate `id`
static ARKS_OUTLINE bool exact_verify_span(const uint8_t* p, uint32_t n, uint32_t has_esc, int id) {
  const char* s = xkey_str(id);
  int L = xkey_len(id);
  if (!has_esc) {
    if ((int)n != L) return false;
    // all (<= 17) byte loads are issued together and compared against immediates: a loop with an early exit makes
    // every byte wait for the previous one's round trip to L2 (the key was hashed on the fly, this only confirms it)
    uint64_t w0 = 0, w1 = 0, w2 = 0;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int i = 0; i < 17; i++) {
      const uint64_t b = i < L ? (uint64_t)p[i] : 0ull;
      if (i < 8) w0 |= b << (8 * i);
      else if (i < 16) w1 |= b << (8 * (i - 8));
      else w2 |= b;
    }
    uint64_t d = 0;
    switch (id) {
#define ARKS_XK(ID) case ID: d = (w0 ^ xkey_word(ID, 0)) | (w1 ^ xkey_word(ID, 1)) | (w2 ^ xkey_word(ID, 2)); break;
      ARKS_XK(0) ARKS_XK(1) ARKS_XK(2) ARKS_XK(3) ARKS_XK(4)
      default: d = (w0 ^ xkey_word(5, 0)) | (w1 ^ xkey_word(5, 1)) | (w2 ^ xkey_word(5, 2)); break;
#undef ARKS_XK
    }
    return d == 0;
  }
  int k = 0;
  bool ok = true;
  decode_span(p, n, [&](uint8_t b) {
    if (k >= L || (uint8_t)s[k] != b) ok = false;
    k++;
  });
  return ok && k == L;
}
// which exact-key candidate in [lo, hi) the span equals, or -1 (khash only valid when !has_esc)
static ARKS_OUTLINE int exact_key_match(const uint8_t* p, uint32_t n, uint32_t has_esc, uint64_t khash, int lo, int hi) {
  int hit = -1;
  for (int id = lo; id < hi; id++) {
    uint64_t want = id == 0 ? X_PROMPT : id == 1 ? X_COMPL : id == 2 ? X_TOTAL : id == 3 ? X_ERROR : id == 4 ? X_CHOICES : X_USAGE;
    if ((has_esc || khash == want) && exact_verify_span(p, n, has_esc, id)) hit = id;
  }
  return hit;
}
// readFieldHash slow path: the hash of a key that contains a backslash (restarts from the first byte)
static ARKS_OUTLINE uint64_t struct_key_hash_slow(const uint8_t* p, uint32_t n) {
  uint64_t h = 0x811c9dc5ull;
  uint32_t i = 0;
  while (p[i] != '\\') h = fhash_step(h, p[i++]);
  decode_span(p + i, n - i, [&](uint8_t b) { h = fhash_step(h, b); });
  return h;
}
// gjson Result.Int of a Number token with a fraction or an exponent, re-read from its raw bytes p[0, n) (the validated
// number, possibly followed by bytes that cannot belong to it): int64(strconv.ParseFloat(raw, 64)) as Go computes it on
// amd64. That is the exact decimal value rounded to the nearest double (ties to even) and truncated toward zero, or
// INT64_MIN when the double is outside [-2^63, 2^63). Computed exactly with integer arithmetic for numbers of any
// length; only the exponent saturates the way ParseFloat's does (it stops growing at 10000), which can change a result
// for numbers of thousands of bytes and more only.
ARKS_HD uint32_t clz64(uint64_t x) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__clzll((long long)x);
#else
  return (uint32_t)__builtin_clzll(x);
#endif
}
static ARKS_OUTLINE int64_t float_number_value(const uint8_t* p, uint32_t n) {
  uint32_t i = 0;
  const bool neg = n > 0 && p[0] == '-';
  if (neg) i++;
  const uint32_t i0 = i;  // integer digits [i0, i1), fraction digits [f0, f0 + (m - ni))
  while (i < n && is_digit(p[i])) i++;
  const uint32_t i1 = i, ni = i1 - i0;
  uint32_t f0 = i;
  if (i < n && p[i] == '.') {
    f0 = ++i;
    while (i < n && is_digit(p[i])) i++;
  }
  const int64_t m = (int64_t)ni + (int64_t)(i - f0);  // mantissa digits
  int64_t e = 0;
  if (i < n && (p[i] | 0x20) == 'e') {
    i++;
    const bool eneg = i < n && p[i] == '-';
    if (i < n && (p[i] == '-' || p[i] == '+')) i++;
    for (; i < n && is_digit(p[i]); i++)
      if (e < 10000) e = e * 10 + (p[i] - '0');
    if (eneg) e = -e;
  }
  // k-th mantissa digit (0 outside the mantissa)
  auto dig = [&](int64_t k) -> uint32_t {
    if (k < 0 || k >= m) return 0;
    return (uint32_t)(k < ni ? p[i0 + k] : p[f0 + (k - ni)]) - '0';
  };
  int64_t z = 0, l = m - 1;  // first and last nonzero mantissa digit
  while (z < m && dig(z) == 0) z++;
  if (z == m) return 0;
  while (dig(l) == 0) l--;
  // value = 0.d_z d_z+1 ... d_l * 10^P: the integer part is mantissa digits [z, z + P), the fraction the ones after
  const int64_t P = (int64_t)ni + e - z;
  if (P > 19) return INT64_MIN;  // >= 10^19 > 2^63
  uint64_t N = 0;
  for (int64_t k = z; k < z + P; k++) N = N * 10 + dig(k);
  if (N >> 63) return INT64_MIN;
  const int64_t f = z + P;    // index of the first fraction digit
  const bool frac = l >= f;   // the fraction is not zero
  uint64_t r;
  if (N >> 53) {
    // doubles here are the multiples of 2^s: round the low s bits plus the fraction to nearest, ties to even
    const uint32_t s = 63 - clz64(N) - 52;
    const uint64_t low = N & ((1ull << s) - 1), half = 1ull << (s - 1), q = N >> s;
    const bool up = low > half || (low == half && (frac || (q & 1)));
    r = (q + up) << s;
    if (r >> 63) return INT64_MIN;
  } else {
    // the result is N or N + 1. N + 1 = n with 2^k < n <= 2^(k+1) is a double, and so is its predecessor n - 2^(k-52):
    // the value rounds to n iff its fraction is >= 1 - 2^-j with j = 53 - k, on a tie iff n's mantissa is even, which
    // holds for every n up to 2^52 and for even n above
    const uint32_t bl = N ? 64 - clz64(N) : 0, j = 54 - bl;  // k = bl - 1
    const uint64_t den = 1ull << j;
    uint64_t rem = den - 1;  // the digits of (2^j - 1) / 2^j by long division: exactly j of them
    int cmp = 0;
    int64_t k = f;
    for (; rem != 0 && cmp == 0; k++) {
      rem *= 10;
      const uint32_t t = (uint32_t)(rem >> j), d = dig(k);
      rem &= den - 1;
      cmp = d > t ? 1 : d < t ? -1 : 0;
    }
    if (cmp == 0) cmp = l >= k ? 1 : 0;  // digits beyond the threshold's last one
    r = N + (cmp > 0 || (cmp == 0 && (j >= 2 || (N & 1))));
  }
  return neg ? (int64_t)(0 - r) : (int64_t)r;
}
// gjson Result.Int for a Number token: a plain integer from its streamed capture (safeInt and parseInt both agree with a
// wrapping parse), anything else from its raw bytes
static ARKS_OUTLINE int64_t captured_number_value(uint64_t nacc, uint32_t nneg, uint32_t nplain, const uint8_t* p, uint32_t n) {
  if (nplain) return nneg ? (int64_t)(0 - nacc) : (int64_t)nacc;
  return float_number_value(p, n);
}

// ---------------------------------------------------------------------------------------------
// 16-byte units, SWAR search for the next byte a string cares about
// ---------------------------------------------------------------------------------------------
struct Unit16 {
  uint32_t w[4];
};

// bit 7 of byte k set  <=>  byte k of the word may be '"', '\\' or < 0x20 (other bits are garbage). The lowest flagged
// byte is always exact; higher bytes can be false positives (borrow of the subtract), which only costs a step() call on
// an ordinary byte. x ^ 0x02 maps {0x00..0x1f, '"'} onto the contiguous range 0x00..0x20, so two range tests suffice.
ARKS_HD uint32_t special_flags(uint32_t w) {
  uint32_t a = w ^ 0x02020202u, b = w ^ 0x5c5c5c5cu;
  return ((a - 0x21212121u) & ~a) | ((b - 0x01010101u) & ~b);
}
ARKS_HD uint32_t special_mask16(uint32_t q0, uint32_t q1, uint32_t q2, uint32_t q3) {
  uint32_t f0 = (special_flags(q0) >> 7) & 0x01010101u, f1 = (special_flags(q1) >> 7) & 0x01010101u;
  uint32_t f2 = (special_flags(q2) >> 7) & 0x01010101u, f3 = (special_flags(q3) >> 7) & 0x01010101u;
  return ((f0 * 0x01020408u) >> 24 & 0xfu) | ((f1 * 0x01020408u) >> 20 & 0xf0u) | ((f2 * 0x01020408u) >> 16 & 0xf00u) |
         ((f3 * 0x01020408u) >> 12 & 0xf000u);
}
ARKS_HD uint32_t first_set(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__ffs((int)x) - 1u;
#else
  return (uint32_t)__builtin_ffs((int)x) - 1u;
#endif
}

}  // namespace arks
