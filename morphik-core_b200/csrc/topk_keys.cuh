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

// The type a page's group scores are added in: float32 for float scores; int64 for I32 scores, whose sum can pass int32
// (an int8 token scores up to 128 * 127^2, so a query of 1041 tokens can).  finish_sum saturates that int64 sum to
// +-(2^31 - 1): the order stays exact inside the range, pages beyond it tie at the bound, and no sum wraps to the other
// sign.  The bound is symmetric, so a sum never reaches INT32_MIN, whose key is 0.
template <typename T> struct SumOf { using type = T; };
template <> struct SumOf<int> { using type = int64_t; };
constexpr int64_t kI32SumBound = 2147483647;
__device__ __forceinline__ float finish_sum(float s) { return s; }
__device__ __forceinline__ int finish_sum(int64_t s) {
  return int(s < -kI32SumBound ? -kI32SumBound : s > kI32SumBound ? kI32SumBound : s);
}

template <typename T>
__device__ __forceinline__ bool page_key(const T* __restrict__ gs, int64_t ld, int g0, int g1, const uint32_t* allow,
                                         int64_t p, uint32_t* key) {
  if (allow && !((__ldg(allow + (p >> 5)) >> (p & 31)) & 1u)) return false;
  typename SumOf<T>::type acc = 0;
  for (int g = g0; g < g1; ++g) acc += __ldg(gs + int64_t(g) * ld + p);
  *key = key_of(finish_sum(acc));
  return true;
}

}  // namespace bms
