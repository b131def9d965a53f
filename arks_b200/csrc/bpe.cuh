// bpe.cuh — the on-device BPE token counter (device, sm_90a; host build for tests).
//
// The north star asks for the prompt / completion text to be BPE-counted on the GPU. The reference has no tokenizer
// (SURVEY.md §0 F1: it reads `usage` from the upstream's response), so this is a SIDE output: it never feeds admit / deny
// unless the host opts in, and its oracle is HF `tokenizers` (tests/test_bpe.py), not the Go code.
//
//   what is counted   every JSON string that is the value of a key named `content` (the messages of a chat request, the
//                     message / delta of a completion or SSE chunk), escapes decoded; on metered rows (N5,
//                     arks_set_stream_metering) also `text`, `reasoning_content` and `arguments`
//   pass 1  (bpe_scan_body, one lane per body)  a byte scanner finds those strings, decodes them into a scratch text
//           buffer and cuts them into pieces with the Qwen2 pre-tokenizer pattern
//           (transformers/models/qwen2/tokenization_qwen2.py:33) written out as a hand scanner over Unicode classes
//           (letter / number / white space / other: a nibble per code point, measured on the regex engine `tokenizers`
//           uses, tools/gen_bpe_unicode.py); every piece becomes one entry (text offset, length, body) of a work list
//   pass 2  (bpe_piece_tokens, one lane per PIECE — pieces, not bodies, are the unit of parallelism)  byte-level BPE: the
//           piece's bytes as base tokens, then merge the adjacent pair of lowest rank, leftmost first, until no pair is
//           in the merge table; the symbols left are the piece's tokens. Merge ranks live in an open-addressing hash table
//           in HBM (L2-resident: 8 MB at Qwen2.5 scale); the lowest-rank — i.e. most frequent — merges are also in a small
//           table that every block stages into shared memory with one 1-D bulk copy (TMA).
// A body is reported as ARKS_BPE_UNCOUNTED instead of a wrong number when it is outside what this path handles: invalid
// UTF-8 / escapes, a lone surrogate, a piece longer than kBpeMaxPiece bytes, NFC-unsafe code points when the tokenizer
// normalises (Qwen2 does), work-list overflow.
// Two pre-tokenizer families are handled: Qwen2 (one number character per piece) and Llama 3 (runs of up to three, `\p{N}{1,3}`;
// every other alternative of the two patterns is the same), chosen per vocabulary by kBpeFlagDigits3. A vocabulary with
// kBpeFlagIgnoreMerges (Llama 3's `"ignore_merges": true`) counts a piece that is itself a vocabulary entry as one token
// before any merge is tried: the piece's bytes are hashed and compared against the vocabulary's token strings.
#pragma once
#include "json_common.cuh"

namespace arks {

constexpr uint32_t kBpeMaxPiece = 128;      // bytes of one pre-token handled on the device
constexpr uint32_t kBpeHotSlots = 2048;     // shared-memory table: 32 KB, holds the kBpeHotMerges lowest-rank merges
// How many of the lowest-rank (most frequent) merges the shared-memory table holds. A lookup probes it first and most pairs a
// merge loop asks about are in no table at all, so what matters is the cost of a MISS: linear probing at 68 % load (1 400 of
// 2 048 slots) walked 5 slots per miss. Counted on the bench workload with the host build (ARKS_BPE_PROBE), slots read per
// pre-token in the shared table / in the full table: 1 400 entries 30.1 / 6.2, 1 024: 17.9 / 6.4, 768: 14.6 / 6.5, 512: 13.3 / 6.9,
// none: 11.2 / 13.5 — 768 halves the shared-memory walks for the same L2 traffic. Contents never change a result (the full
// table holds every merge).
#ifndef ARKS_BPE_HOT_MERGES
#define ARKS_BPE_HOT_MERGES 768
#endif
constexpr uint32_t kBpeHotMerges = ARKS_BPE_HOT_MERGES;
constexpr uint32_t kBpeUncounted = 0xFFFFFFFFu;
constexpr uint32_t kBpeFlagNfc = 1u;
constexpr uint32_t kBpeFlagDigits3 = 2u;        // the pre-tokenizer splits numbers as \p{N}{1,3} (Llama 3) instead of \p{N}
constexpr uint32_t kBpeFlagIgnoreMerges = 4u;   // a piece that is a vocabulary entry is one token (whole-piece lookup first)
constexpr uint32_t kBpeMaxVocabs = 8;           // vocabulary slots of a context (slot 0: the default)
enum : uint32_t { UC_OTHER = 0, UC_LETTER = 1, UC_NUMBER = 2, UC_SPACE = 3, UC_NFC_UNSAFE = 4 };

struct BpeSlot {  // one merge: key = left | right << 32; rank == 0xFFFFFFFF marks an empty slot
  uint32_t left, right, rank, merged;
};
struct BpeWholeSlot {  // tok == 0xFFFFFFFF marks an empty slot; fp: the high half of the string's hash
  uint32_t fp, tok;
};
struct BpeTablesDev {
  const uint32_t* byte_id;  // 256
  const BpeSlot* table;     // all merges
  uint32_t table_mask;
  const BpeSlot* hot;       // kBpeHotSlots slots (global image; blocks copy it to shared memory)
  const uint8_t* cp_class;  // 0x110000 / 2 (one table shared by every vocabulary: the classes belong to the pattern)
  uint32_t flags;
  // kBpeFlagIgnoreMerges only: the vocabulary's token byte strings of 2..kBpeMaxPiece bytes, an open-addressing table over them
  const BpeWholeSlot* whole = nullptr;
  uint32_t whole_mask = 0;
  const uint32_t* whole_off = nullptr;  // token k is whole_pool[whole_off[k], whole_off[k + 1])
  const uint8_t* whole_pool = nullptr;
};

// host test build only (tests/host_machine.cpp): counts the table slots a lookup reads, so that the bench can state the
// merge-table traffic of a workload next to its text bytes (SURVEY.md section 8d). Nothing on the device.
#ifndef ARKS_BPE_PROBE
#define ARKS_BPE_PROBE(kind)
#endif
ARKS_HD uint32_t bpe_hash(uint32_t left, uint32_t right, uint32_t mask) {
  const uint64_t k = ((uint64_t)right << 32 | left) * 0x9E3779B97F4A7C15ull;
  return (uint32_t)(k >> 40) & mask;
}
// rank and merged id of the pair, or false
ARKS_HD bool bpe_lookup(const BpeSlot* hot, const BpeTablesDev& T, uint32_t left, uint32_t right, uint32_t* rank, uint32_t* merged) {
  uint32_t s = bpe_hash(left, right, kBpeHotSlots - 1);
  for (;;) {
    ARKS_BPE_PROBE(0);
    const BpeSlot e = hot[s];
    if (e.rank == 0xFFFFFFFFu) break;
    if (e.left == left && e.right == right) { *rank = e.rank; *merged = e.merged; return true; }
    s = (s + 1) & (kBpeHotSlots - 1);
  }
  s = bpe_hash(left, right, T.table_mask);
  for (;;) {
    ARKS_BPE_PROBE(1);
    const BpeSlot e = T.table[s];
    if (e.rank == 0xFFFFFFFFu) return false;
    if (e.left == left && e.right == right) { *rank = e.rank; *merged = e.merged; return true; }
    s = (s + 1) & T.table_mask;
  }
}

// FNV-1a over a byte string: the whole-piece table's hash (low bits: the slot, high half: the fingerprint)
ARKS_HD uint64_t bpe_bytes_hash(const uint8_t* p, uint32_t n) {
  uint64_t h = 0xcbf29ce484222325ull;
  for (uint32_t i = 0; i < n; i++) h = (h ^ p[i]) * 0x100000001b3ull;
  return h;
}
// the piece is one of the vocabulary's token strings: exact (a fingerprint match is confirmed byte by byte)
ARKS_HD bool bpe_whole_token(const uint8_t* p, uint32_t n, const BpeTablesDev& T) {
  const uint64_t h = bpe_bytes_hash(p, n);
  const uint32_t fp = (uint32_t)(h >> 32);
  for (uint32_t s = (uint32_t)h & T.whole_mask;; s = (s + 1) & T.whole_mask) {
    const BpeWholeSlot e = T.whole[s];
    if (e.tok == 0xFFFFFFFFu) return false;
    if (e.fp != fp) continue;
    const uint32_t a = T.whole_off[e.tok];
    if (T.whole_off[e.tok + 1] - a != n) continue;
    uint32_t diff = 0;
    for (uint32_t k = 0; k < n; k++) diff |= (uint32_t)(T.whole_pool[a + k] ^ p[k]);
    if (diff == 0) return true;
  }
}

// tokens of one piece of `n` <= kBpeMaxPiece bytes. Every round looks all adjacent pairs up again instead of keeping their
// ranks: the same result, a third of the per-lane scratch (pieces are short: a word, a number, a run of punctuation).
// kIgnoreMerges (vocabularies with kBpeFlagIgnoreMerges): a piece that is a vocabulary entry is one token, merged or not.
template <bool kIgnoreMerges = false>
ARKS_HD uint32_t bpe_piece_tokens(const uint8_t* p, uint32_t n, const BpeSlot* hot, const BpeTablesDev& T) {
  if (kIgnoreMerges && n >= 2 && bpe_whole_token(p, n, T)) return 1;
  uint32_t sym[kBpeMaxPiece];
  for (uint32_t i = 0; i < n; i++) sym[i] = T.byte_id[p[i]];
  while (n > 1) {
    uint32_t best = 0xFFFFFFFFu, at = 0, into = 0;
    for (uint32_t i = 0; i + 1 < n; i++) {
      uint32_t r, m;
      if (bpe_lookup(hot, T, sym[i], sym[i + 1], &r, &m) && r < best) { best = r; at = i; into = m; }  // lowest rank, leftmost
    }
    if (best == 0xFFFFFFFFu) break;
    sym[at] = into;
    for (uint32_t i = at + 1; i + 1 < n; i++) sym[i] = sym[i + 1];
    n--;
  }
  return n;
}

// ---- UTF-8 / classes ----
ARKS_HD uint32_t bpe_class(const uint8_t* tbl, uint32_t cp) {
  const uint8_t b = tbl[cp >> 1];
  return (cp & 1u) ? (uint32_t)(b >> 4) : (uint32_t)(b & 15u);
}
// code point at text[pos] (valid UTF-8 is guaranteed by the decoder below); *len: its byte length
ARKS_HD uint32_t bpe_cp_at(const uint8_t* t, uint32_t pos, uint32_t* len) {
  const uint32_t b0 = t[pos];
  if (b0 < 0x80) { *len = 1; return b0; }
  if (b0 < 0xE0) { *len = 2; return (b0 & 0x1Fu) << 6 | (t[pos + 1] & 0x3Fu); }
  if (b0 < 0xF0) { *len = 3; return (b0 & 0x0Fu) << 12 | (t[pos + 1] & 0x3Fu) << 6 | (t[pos + 2] & 0x3Fu); }
  *len = 4;
  return (b0 & 0x07u) << 18 | (t[pos + 1] & 0x3Fu) << 12 | (t[pos + 2] & 0x3Fu) << 6 | (t[pos + 3] & 0x3Fu);
}
ARKS_HD uint32_t bpe_put_utf8(uint8_t* t, uint32_t w, uint32_t cp) {
  if (cp < 0x80) { t[w] = (uint8_t)cp; return 1; }
  if (cp < 0x800) { t[w] = (uint8_t)(0xC0 | cp >> 6); t[w + 1] = (uint8_t)(0x80 | (cp & 0x3F)); return 2; }
  if (cp < 0x10000) {
    t[w] = (uint8_t)(0xE0 | cp >> 12); t[w + 1] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F)); t[w + 2] = (uint8_t)(0x80 | (cp & 0x3F));
    return 3;
  }
  t[w] = (uint8_t)(0xF0 | cp >> 18); t[w + 1] = (uint8_t)(0x80 | ((cp >> 12) & 0x3F)); t[w + 2] = (uint8_t)(0x80 | ((cp >> 6) & 0x3F));
  t[w + 3] = (uint8_t)(0x80 | (cp & 0x3F));
  return 4;
}

// ---- the Qwen2 split pattern as a scanner over text[s, e) (valid UTF-8); emit(begin, end) per piece, in order ----
//   (?i:'s|'t|'re|'ve|'m|'ll|'d) | [^\r\n\p{L}\p{N}]?\p{L}+ | \p{N} | ?[^\s\p{L}\p{N}]+[\r\n]* | \s*[\r\n]+ | \s+(?!\S) | \s+
// Alternatives in order, each greedy with backtracking; checked against `tokenizers` on random Unicode (tests/test_bpe.py).
// kDigits: the longest run of number characters alternative 3 takes, 1 (Qwen2: \p{N}) or 3 (Llama 3: \p{N}{1,3}, the only
// difference between the two patterns; tests/test_model_vocab.py).
template <uint32_t kDigits = 1, class E>
ARKS_HD void bpe_pretokenize(const uint8_t* t, uint32_t s, uint32_t e, const uint8_t* cls_tbl, E&& emit) {
  uint32_t i = s;
  auto cls = [&](uint32_t pos, uint32_t* len) { return bpe_class(cls_tbl, bpe_cp_at(t, pos, len)) & 3u; };
  auto is_nl = [&](uint32_t pos) { return t[pos] == '\n' || t[pos] == '\r'; };
  while (i < e) {
    uint32_t l0;
    const uint32_t k0 = cls(i, &l0);
    const uint8_t c0 = t[i];
    // 1: contractions, case-insensitive (U+017F LATIN SMALL LETTER LONG S folds to s)
    if (c0 == '\'' && i + 1 < e) {
      const uint8_t a = t[i + 1] | 0x20;
      if (a == 's' || a == 't' || a == 'm' || a == 'd') { emit(i, i + 2); i += 2; continue; }
      if (t[i + 1] == 0xC5 && i + 2 < e && t[i + 2] == 0xBF) { emit(i, i + 3); i += 3; continue; }
      if (i + 2 < e) {
        const uint8_t b = t[i + 2] | 0x20;
        if ((a == 'r' && b == 'e') || (a == 'v' && b == 'e') || (a == 'l' && b == 'l')) { emit(i, i + 3); i += 3; continue; }
      }
    }
    // 2: an optional single non-letter, non-number, non-newline character, then letters
    {
      uint32_t j = i, lj = l0, kj = k0;
      if (k0 != UC_LETTER && k0 != UC_NUMBER && !is_nl(i) && i + l0 < e) {
        uint32_t l1;
        if (cls(i + l0, &l1) == UC_LETTER) { j = i + l0; lj = l1; kj = UC_LETTER; }
      }
      if (kj == UC_LETTER) {
        uint32_t q = j + lj;
        while (q < e) {
          uint32_t lq;
          if (cls(q, &lq) != UC_LETTER) break;
          q += lq;
        }
        emit(i, q);
        i = q;
        continue;
      }
    }
    // 3: one number character (up to kDigits of them)
    if (k0 == UC_NUMBER) {
      uint32_t q = i + l0;
      for (uint32_t d = 1; d < kDigits && q < e; d++) {
        uint32_t lq;
        if (cls(q, &lq) != UC_NUMBER) break;
        q += lq;
      }
      emit(i, q);
      i = q;
      continue;
    }
    // 4: an optional space, then characters that are neither white space, letters nor numbers, then newlines
    {
      uint32_t j = i, kj = k0, lj = l0;
      if (c0 == ' ' && i + 1 < e) {
        uint32_t l1;
        if (cls(i + 1, &l1) == UC_OTHER) { j = i + 1; kj = UC_OTHER; lj = l1; }
      }
      if (kj == UC_OTHER) {
        uint32_t q = j + lj;
        while (q < e) {
          uint32_t lq;
          if (cls(q, &lq) != UC_OTHER) break;
          q += lq;
        }
        while (q < e && is_nl(q)) q++;
        emit(i, q);
        i = q;
        continue;
      }
    }
    // 5-7: a run of white space
    {
      uint32_t q = i, last_nl_end = 0, last_start = i;
      bool has_nl = false;
      while (q < e) {
        uint32_t lq;
        if (cls(q, &lq) != UC_SPACE) break;
        if (is_nl(q)) { has_nl = true; last_nl_end = q + 1; }
        last_start = q;
        q += lq;
      }
      if (has_nl) { emit(i, last_nl_end); i = last_nl_end; continue; }   // \s*[\r\n]+ : through the run's last newline
      if (q == e || last_start == i) { emit(i, q); i = q; continue; }    // \s+(?!\S) at the end of the text; or a single \s
      emit(i, last_start);                                              // \s+(?!\S): all but the run's last character
      i = last_start;
    }
  }
}

// ---- key sets: the names whose string values are counted. Bit k selects name k; all candidates are matched at once ----
constexpr uint32_t kBpeKeysContent = 1u;  // `content` only: every row that is not metered
constexpr uint32_t kBpeKeysWide = 15u;    // + `text` (content parts), `reasoning_content`, `arguments` (tool calls): metered rows
// The names are packed little-endian into 64-bit immediates (no loads, no pointers held in registers); bytes past a name
// are 0. A candidate that survives past its length is harmless: bpe_key_done wants the exact length.
ARKS_HD constexpr uint64_t bpe_pack8(const char* s, uint32_t n) {
  uint64_t v = 0;
  for (uint32_t i = n; i-- > 0;) v = v << 8 | (uint8_t)s[i];
  return v;
}
constexpr uint64_t kKeyContent = bpe_pack8("content", 7), kKeyText = bpe_pack8("text", 4);
constexpr uint64_t kKeyReason0 = bpe_pack8("reasoning_content", 8), kKeyReason1 = bpe_pack8("reasoning_content" + 8, 8), kKeyReason2 = 't';
constexpr uint64_t kKeyArgs0 = bpe_pack8("arguments", 8), kKeyArgs1 = 's';
// candidates still equal to the decoded key after its character `cp` at position `pos`
ARKS_HD uint32_t bpe_key_step(uint32_t cand, uint32_t pos, uint32_t cp) {
  if (cp >= 0x80 || pos >= 17) return 0;
  const uint32_t sh = 8 * (pos & 7);
  const bool lo = pos < 8, mid = pos >= 8 && pos < 16;
  const uint32_t c0 = lo ? (uint32_t)(kKeyContent >> sh) & 0xffu : 0u;
  const uint32_t c1 = lo ? (uint32_t)(kKeyText >> sh) & 0xffu : 0u;
  const uint32_t c2 = (uint32_t)((lo ? kKeyReason0 : mid ? kKeyReason1 : kKeyReason2) >> sh) & 0xffu;
  const uint32_t c3 = (uint32_t)((lo ? kKeyArgs0 : mid ? kKeyArgs1 : 0ull) >> sh) & 0xffu;
  return cand & ((c0 == cp ? 1u : 0u) | (c1 == cp ? 2u : 0u) | (c2 == cp ? 4u : 0u) | (c3 == cp ? 8u : 0u));
}
// a candidate of exactly `pos` characters is left
ARKS_HD bool bpe_key_done(uint32_t cand, uint32_t pos) {
  return ((cand & 1u) && pos == 7) || ((cand & 2u) && pos == 4) || ((cand & 4u) && pos == 17) || ((cand & 8u) && pos == 9);
}

// ---- pass 1: one body ----
struct BpeScanOut {
  uint32_t pieces;  // emitted
  uint32_t bad;     // the body is reported as uncounted
};
// text: scratch for the decoded strings of this body (capacity >= len bytes). keys: kBpeKeysContent or kBpeKeysWide.
// emit(text offset, length) per piece. kDigits: the pre-tokenizer family (bpe_pretokenize).
template <uint32_t kDigits = 1, class E>
ARKS_HD BpeScanOut bpe_scan_body(const uint8_t* b, uint32_t len, uint8_t* text, const BpeTablesDev& T, uint32_t keys, E&& emit) {
  BpeScanOut o{0, 0};
  uint32_t i = 0, wr = 0;
  bool last_string = false, last_is_key = false, expect = false;
  while (i < len && !o.bad) {
    const uint8_t c = b[i];
    if (c == '"') {
      const bool count_it = expect;
      expect = false;
      const uint32_t w0 = wr;
      uint32_t cand = keys, pos = 0;  // key names still equal to the decoded string, its decoded length
      bool closed = false, unsafe = false;
      i++;
      while (i < len) {
        uint32_t ch = b[i];
        uint32_t cp;
        if (ch == '"') { closed = true; i++; break; }
        if (ch == '\\') {
          if (i + 1 >= len) { o.bad = 1; break; }
          const uint8_t x = b[i + 1];
          i += 2;
          if (x == 'u') {
            if (i + 4 > len) { o.bad = 1; break; }
            const int h = hexval(b[i]) << 12 | hexval(b[i + 1]) << 8 | hexval(b[i + 2]) << 4 | hexval(b[i + 3]);
            if ((hexval(b[i]) | hexval(b[i + 1]) | hexval(b[i + 2]) | hexval(b[i + 3])) < 0) { o.bad = 1; break; }
            i += 4;
            cp = (uint32_t)h;
            if (cp >= 0xD800 && cp < 0xDC00) {  // high surrogate: must be followed by \uDC00..\uDFFF
              if (i + 6 <= len && b[i] == '\\' && b[i + 1] == 'u') {
                const int lo = hexval(b[i + 2]) << 12 | hexval(b[i + 3]) << 8 | hexval(b[i + 4]) << 4 | hexval(b[i + 5]);
                if ((hexval(b[i + 2]) | hexval(b[i + 3]) | hexval(b[i + 4]) | hexval(b[i + 5])) >= 0 && lo >= 0xDC00 && lo < 0xE000) {
                  cp = 0x10000u + ((cp - 0xD800u) << 10) + ((uint32_t)lo - 0xDC00u);
                  i += 6;
                } else { o.bad = 1; break; }
              } else { o.bad = 1; break; }
            } else if (cp >= 0xDC00 && cp < 0xE000) { o.bad = 1; break; }  // a lone low surrogate
          } else {
            cp = x == 'n' ? '\n' : x == 't' ? '\t' : x == 'r' ? '\r' : x == 'b' ? '\b' : x == 'f' ? '\f'
               : (x == '"' || x == '\\' || x == '/') ? x : 0xFFFFFFFFu;
            if (cp == 0xFFFFFFFFu) { o.bad = 1; break; }
          }
        } else if (ch < 0x80) {
          if (ch < 0x20) { o.bad = 1; break; }  // not JSON
          cp = ch;
          i++;
        } else {  // raw UTF-8: validate (no overlongs, no surrogates, <= U+10FFFF)
          const uint32_t need = ch >= 0xF0 ? 4 : ch >= 0xE0 ? 3 : ch >= 0xC2 ? 2 : 0;
          if (!need || ch > 0xF4 || i + need > len) { o.bad = 1; break; }
          cp = ch & (need == 2 ? 0x1Fu : need == 3 ? 0x0Fu : 0x07u);
          bool okc = true;
          for (uint32_t k = 1; k < need; k++) { okc &= (b[i + k] & 0xC0) == 0x80; cp = cp << 6 | (b[i + k] & 0x3Fu); }
          if (!okc || (need == 3 && cp < 0x800) || (need == 4 && (cp < 0x10000 || cp > 0x10FFFF)) || (cp >= 0xD800 && cp < 0xE000)) { o.bad = 1; break; }
          i += need;
        }
        if (bpe_class(T.cp_class, cp) & UC_NFC_UNSAFE) unsafe = true;
        if (cand) cand = bpe_key_step(cand, pos, cp);
        pos++;
        wr += bpe_put_utf8(text, wr, cp);
      }
      if (!closed) { o.bad = 1; break; }
      if (count_it) {
        if (unsafe && (T.flags & kBpeFlagNfc)) { o.bad = 1; break; }
        bpe_pretokenize<kDigits>(text, w0, wr, T.cp_class, [&](uint32_t s, uint32_t e) {
          if (e - s > kBpeMaxPiece) o.bad = 1;
          else { emit(s, e - s); o.pieces++; }
        });
      } else {
        wr = w0;  // not counted: the scratch is reused
      }
      last_string = true;
      last_is_key = bpe_key_done(cand, pos);
      continue;
    }
    if (c == ' ' || c == '\t' || c == '\n' || c == '\r') { i++; continue; }
    if (c == ':' && last_string && last_is_key) expect = true;
    else expect = false;
    last_string = false;
    i++;
  }
  return o;
}
template <class E>
ARKS_HD BpeScanOut bpe_scan_body(const uint8_t* b, uint32_t len, uint8_t* text, const BpeTablesDev& T, E&& emit) {
  return bpe_scan_body(b, len, text, T, kBpeKeysContent, emit);
}

// ---- host: the merge list as the two hash tables the lookups use (also used by the CPU test build) ----
}  // namespace arks
#include <vector>
namespace arks {
// slots: a power of two; merges [0, n) inserted in rank order (a pair that occurs twice keeps its lowest rank, as in the
// tokenizer's dictionary)
inline void bpe_fill_table(std::vector<BpeSlot>& tab, uint32_t slots, const uint32_t* left, const uint32_t* right, const uint32_t* merged,
                           uint32_t n) {
  tab.assign(slots, BpeSlot{0, 0, 0xFFFFFFFFu, 0});
  for (uint32_t r = 0; r < n; r++) {
    uint32_t s = bpe_hash(left[r], right[r], slots - 1);
    bool dup = false;
    while (tab[s].rank != 0xFFFFFFFFu) {
      if (tab[s].left == left[r] && tab[s].right == right[r]) { dup = true; break; }
      s = (s + 1) & (slots - 1);
    }
    if (!dup) tab[s] = BpeSlot{left[r], right[r], r, merged[r]};
  }
}
inline uint32_t bpe_table_slots(uint32_t n_merges) {
  uint32_t s = 1024;
  while (s < 2 * n_merges + 16) s <<= 1;
  return s;
}
// the whole-piece table of a vocabulary with kBpeFlagIgnoreMerges: token k is bytes[off[k], off[k + 1]); only strings of
// 2..kBpeMaxPiece bytes are entered (shorter or longer pieces never look it up). Returns the slot count (a power of two).
inline uint32_t bpe_fill_whole(std::vector<BpeWholeSlot>& tab, const uint8_t* bytes, const uint32_t* off, uint32_t n) {
  uint32_t slots = 1024;
  while (slots < 2 * n + 16) slots <<= 1;
  tab.assign(slots, BpeWholeSlot{0, 0xFFFFFFFFu});
  for (uint32_t k = 0; k < n; k++) {
    const uint32_t len = off[k + 1] - off[k];
    if (len < 2 || len > kBpeMaxPiece) continue;
    const uint64_t h = bpe_bytes_hash(bytes + off[k], len);
    uint32_t s = (uint32_t)h & (slots - 1);
    while (tab[s].tok != 0xFFFFFFFFu) s = (s + 1) & (slots - 1);
    tab[s] = BpeWholeSlot{(uint32_t)(h >> 32), k};
  }
  return slots;
}

}  // namespace arks
