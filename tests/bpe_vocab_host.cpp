// bpe_vocab_host.cpp — TEST-ONLY host build of the BPE counter (arks_b200/csrc/bpe.cuh) for one vocabulary slot with its
// flags: the pre-tokenizer family (kBpeFlagDigits3) and the whole-piece lookup of `ignore_merges` vocabularies
// (kBpeFlagIgnoreMerges, with the token strings), for tests/test_model_vocab.py.
#include "../arks_b200/csrc/bpe.cuh"
#include <type_traits>
#include <vector>
using namespace arks;

struct Slot {  // one vocabulary slot and everything its BpeTablesDev points into
  std::vector<BpeSlot> table, hot;
  std::vector<BpeWholeSlot> whole;
  std::vector<uint32_t> byte_id, tok_off;
  std::vector<uint8_t> cls, tok_bytes;
  BpeTablesDev t{};
};
static Slot g_slot[kBpeMaxVocabs];
extern "C" {
void bv_load(uint32_t slot, const uint32_t* byte_id, uint32_t n, const uint32_t* left, const uint32_t* right, const uint32_t* merged,
             const uint8_t* cp_class, uint32_t flags, const uint8_t* tok_bytes, const uint32_t* tok_off, uint32_t n_tok) {
  Slot& S = g_slot[slot];
  S.byte_id.assign(byte_id, byte_id + 256);
  S.cls.assign(cp_class, cp_class + 0x110000 / 2);
  const uint32_t slots = bpe_table_slots(n);
  bpe_fill_table(S.table, slots, left, right, merged, n);
  bpe_fill_table(S.hot, kBpeHotSlots, left, right, merged, n < kBpeHotMerges ? n : kBpeHotMerges);
  S.t = BpeTablesDev{S.byte_id.data(), S.table.data(), slots - 1, S.hot.data(), S.cls.data(), flags};
  if (flags & kBpeFlagIgnoreMerges) {
    S.tok_off.assign(tok_off, tok_off + n_tok + 1);
    S.tok_bytes.assign(tok_bytes, tok_bytes + tok_off[n_tok]);
    S.tok_bytes.push_back(0);
    S.t.whole_mask = bpe_fill_whole(S.whole, S.tok_bytes.data(), S.tok_off.data(), n_tok) - 1;
    S.t.whole = S.whole.data();
    S.t.whole_off = S.tok_off.data();
    S.t.whole_pool = S.tok_bytes.data();
  }
}
// `content` tokens of a body or SSE chunk with the slot's vocabulary and flags, or 0xFFFFFFFF
uint32_t bv_count(uint32_t slot, const uint8_t* body, size_t len) {
  const BpeTablesDev& T = g_slot[slot].t;
  std::vector<uint8_t> text(len + 8);
  uint32_t total = 0;
  auto count = [&](auto digits, auto ignore) {
    return bpe_scan_body<decltype(digits)::value>(body, (uint32_t)len, text.data(), T, kBpeKeysContent, [&](uint32_t off, uint32_t n) {
      total += bpe_piece_tokens<decltype(ignore)::value>(text.data() + off, n, T.hot, T);
    });
  };
  using D1 = std::integral_constant<uint32_t, 1>;
  using D3 = std::integral_constant<uint32_t, 3>;
  const bool d3 = T.flags & kBpeFlagDigits3, im = T.flags & kBpeFlagIgnoreMerges;
  const BpeScanOut o = d3 ? (im ? count(D3{}, std::true_type{}) : count(D3{}, std::false_type{}))
                          : (im ? count(D1{}, std::true_type{}) : count(D1{}, std::false_type{}));
  return o.bad ? kBpeUncounted : total;
}
// piece ends (byte offsets) of text[0, len) under the slot's pre-tokenizer; returns how many (at most cap written)
uint32_t bv_pretokenize(uint32_t slot, const uint8_t* text, uint32_t len, uint32_t* ends, uint32_t cap) {
  uint32_t k = 0;
  auto put = [&](uint32_t, uint32_t e) {
    if (k < cap) ends[k] = e;
    k++;
  };
  const BpeTablesDev& T = g_slot[slot].t;
  if (T.flags & kBpeFlagDigits3) bpe_pretokenize<3>(text, 0, len, T.cp_class, put);
  else bpe_pretokenize<1>(text, 0, len, T.cp_class, put);
  return k;
}
}
