// sortkey.cuh — the order-preserving key words of the sort (sort.cu) and of the range push that routes rows by them
// (partition.cu: k_range_dest).  One definition, so that the router and the sort agree by construction on every edge the
// comparator has: -0.0 == +0.0, BIGINT UNSIGNED >= 2^63 above every BIGINT, "" != NULL, a proper prefix below its extensions.
// A ByItem orders by its words most significant first: the NULL flag, then the value word — or, for a string, the zero-padded
// 8-byte big-endian chunks first to last and then the length — each inverted when Desc.
#pragma once
#include "common.cuh"

namespace tq {

// types.CompareInt64 / CompareUint64 / CompareFloat64 (types/compare.go) as unsigned comparisons of one word
__device__ __forceinline__ uint64_t enc_word(uint64_t v, int type) {
  if (type == TQ_TYPE_INT64) return v ^ 0x8000000000000000ull;
  if (type == TQ_TYPE_FLOAT64) {
    if ((v << 1) == 0) return 0x8000000000000000ull;          // -0.0 == +0.0
    return (v >> 63) ? ~v : (v | 0x8000000000000000ull);
  }
  return v;  // BIGINT UNSIGNED
}

enum { KS_COL8 = 0, KS_F32 = 1, KS_STR_CHUNK = 2, KS_STR_LEN = 3, KS_NULL_FLAG = 4, KS_MIX_CLASS = 5, KS_MIX_VALUE = 6 };
struct KeySrc {
  int mode;             // KS_*
  int type;             // KS_COL8 / KS_MIX_*: TQ_TYPE_* of the column
  int word;             // KS_STR_CHUNK: which 8-byte chunk of the cell
  int desc;             // ByItems.Desc: the word is inverted
  const uint64_t *d8;   // 8-byte slots
  const uint32_t *d4;   // FLOAT slots
  const int64_t *off;   // var-len: offsets[n + 1] (relative to `base`) and bytes
  const uint8_t *bytes;
  int64_t base;
  const uint32_t *bm;   // NOT-NULL bitmap or nullptr
};

__device__ __forceinline__ uint64_t key_word(const KeySrc &k, uint32_t r) {
  const bool nn = tqd::bm_not_null(k.bm, r);
  uint64_t w = 0;
  switch (k.mode) {
    case KS_COL8: if (nn) w = enc_word(k.d8[r], k.type); break;
    case KS_F32: if (nn) w = enc_word((uint64_t)__double_as_longlong((double)__uint_as_float(k.d4[r])), TQ_TYPE_FLOAT64); break;
    case KS_STR_CHUNK:
      if (nn) {
        const int64_t s0 = k.off[r] - k.base, len = k.off[r + 1] - k.off[r];
        const int64_t b0 = (int64_t)k.word * 8;
#pragma unroll
        for (int j = 0; j < 8; j++) w = (w << 8) | (uint64_t)((b0 + j < len) ? k.bytes[s0 + b0 + j] : 0);
      }
      break;
    case KS_STR_LEN: if (nn) w = (uint64_t)(k.off[r + 1] - k.off[r]); break;
    case KS_NULL_FLAG: w = nn ? 1 : 0; break;
    // a BIGINT compared with a BIGINT UNSIGNED (types.CompareInt with mixed flags): (class, value) pairs order and
    // equate the two domains exactly — negative < [0, 2^63) < unsigned >= 2^63
    case KS_MIX_CLASS:
      if (nn) { const uint64_t v = k.d8[r]; w = (k.type == TQ_TYPE_INT64) ? ((v >> 63) ? 0 : 1) : ((v >> 63) ? 2 : 1); }
      break;
    default: if (nn) w = k.d8[r]; break;   // KS_MIX_VALUE: inside a class the raw two's-complement word orders both domains
  }
  return k.desc ? ~w : w;
}

}  // namespace tq
