// topk_keys.cuh -- the total order every selection over page scores uses (topk.cu, topk_docs.cu): a page's score is the
// sum of its query's group scores, mapped to an order-preserving 32-bit key; ties break towards the lower page (slot).
#pragma once
#include <stdint.h>

namespace bms {

__device__ __forceinline__ uint32_t key_of(float s) {
  const uint32_t u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ uint32_t key_of(int s) { return uint32_t(s) ^ 0x80000000u; }
// key_of of a caller's float: -0 -> +0 and every NaN -> the canonical NaN 0x7fffffff (the device's fadd returns it), so
// that -0 ties with +0 and every NaN ranks above +inf, tied with the other NaNs.  The sums page_key forms from T(0) are
// canonical already; raw floats handed to the merge are not (a NaN with its sign bit set would key below -inf, and
// 0xffffffff would get key 0, the key of an invalid entry).
__device__ __forceinline__ uint32_t key_of_canonical(float s) { return key_of(s + 0.0f); }
__device__ __forceinline__ float score_of_key(uint32_t k, float) {
  const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}
__device__ __forceinline__ float score_of_key(uint32_t k, int) { return float(int(k ^ 0x80000000u)); }

template <typename T>
__device__ __forceinline__ bool page_key(const T* __restrict__ gs, int64_t ld, int g0, int g1, const uint32_t* allow,
                                         int64_t p, uint32_t* key) {
  if (allow && !((__ldg(allow + (p >> 5)) >> (p & 31)) & 1u)) return false;
  T acc = T(0);
  for (int g = g0; g < g1; ++g) acc += __ldg(gs + int64_t(g) * ld + p);
  *key = key_of(acc);
  return true;
}

}  // namespace bms
