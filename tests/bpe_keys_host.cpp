// bpe_keys_host.cpp — TEST-ONLY host build of the BPE counter (arks_b200/csrc/bpe.cuh) with the key set chosen per call:
// `content` only, or the wider set of metered rows (N5, arks_set_stream_metering), for tests/test_stream_metering.py.
#include "../arks_b200/csrc/bpe.cuh"
#include <vector>
using namespace arks;

static std::vector<BpeSlot> g_table, g_hot;
static std::vector<uint32_t> g_byte_id;
static std::vector<uint8_t> g_cls;
static BpeTablesDev g_bpe{};
extern "C" {
void bk_load(const uint32_t* byte_id, uint32_t n, const uint32_t* left, const uint32_t* right, const uint32_t* merged,
             const uint8_t* cp_class, uint32_t flags) {
  g_byte_id.assign(byte_id, byte_id + 256);
  g_cls.assign(cp_class, cp_class + 0x110000 / 2);
  const uint32_t slots = bpe_table_slots(n);
  bpe_fill_table(g_table, slots, left, right, merged, n);
  bpe_fill_table(g_hot, kBpeHotSlots, left, right, merged, n < kBpeHotMerges ? n : kBpeHotMerges);
  g_bpe = BpeTablesDev{g_byte_id.data(), g_table.data(), slots - 1, g_hot.data(), g_cls.data(), flags};
}
// tokens of the body's strings under the key set (wide != 0: content, text, reasoning_content, arguments), or 0xFFFFFFFF
uint32_t bk_count(const uint8_t* body, size_t len, int wide) {
  std::vector<uint8_t> text(len + 8);
  uint32_t total = 0;
  const BpeScanOut o = bpe_scan_body(body, (uint32_t)len, text.data(), g_bpe, wide ? kBpeKeysWide : kBpeKeysContent,
                                     [&](uint32_t off, uint32_t n) { total += bpe_piece_tokens(text.data() + off, n, g_bpe.hot, g_bpe); });
  return o.bad ? kBpeUncounted : total;
}
}
