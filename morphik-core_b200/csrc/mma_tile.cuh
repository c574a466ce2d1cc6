// mma_tile.cuh -- tile geometry and accumulator helpers of the wgmma MaxSim kernel (maxsim_wgmma.cu).
#pragma once
#include <type_traits>

#include "common.cuh"
#include "ptx.cuh"

namespace bms {

constexpr uint32_t kSubtileBytes = 128 * 128;    // 128 rows x 128 B (one swizzle-128B panel)
constexpr uint32_t kSmemLimit = 232448;          // 227 KB opt-in maximum per CTA
constexpr uint32_t kBarrierBytes = 2048;         // mbarriers

// KIND 0: bf16 rows (256 B = two 128 B K-panels), wgmma .bf16 (k16), fp32 accumulators
// KIND 1: int8 rows (128 B = one panel),           wgmma .s8 (k32),    int32 accumulators (exact)
// KIND 2: fp8 e4m3 rows (128 B in HBM), widened to f16 in shared memory (two panels, exact), wgmma .f16 (k16), fp32
//         accumulators.  Hopper's e4m3 wgmma adds its products with less than fp32 precision (relative errors of 1e-3 were
//         measured against the oracle on an H100); e4m3 -> f16 is exact, so the f16 products are exact and sum in fp32.
// Every wgmma step consumes 32 B of K per row of shared memory.
template <int KIND>
struct Kind {
  static constexpr int kPanels = KIND == 1 ? 1 : 2;
  static constexpr uint32_t kTileBytes = kPanels * kSubtileBytes;
  static constexpr int kPanelElems = KIND == 1 ? 128 : 64;  // TMA x-coordinate step per panel (elements)
  static constexpr int kKSteps = KIND == 1 ? 4 : 8;         // wgmma K steps per 128-d row
  static constexpr int kMaxNM = KIND == 1 ? 8 : 4;          // query tiles one CTA can keep resident in shared memory
  using Acc = typename std::conditional<KIND == 1, int, float>::type;
};

// corpus dtype (include/b200ms.h) -> kernel KIND, or -1
__host__ __device__ constexpr int kind_of_dtype(int dtype) {
  return dtype == B200MS_BF16 ? 0 : dtype == B200MS_I8 ? 1 : dtype == B200MS_F8 ? 2 : -1;
}

// e4m3 x 8 (one 8-byte word) -> 8 f16 (exact)
__device__ __forceinline__ uint4 e4m3x8_to_f16x8(uint32_t lo, uint32_t hi) {
  uint4 o;
  asm("{\n\t.reg .b16 a, b, c, d;\n\t"
      "mov.b32 {a, b}, %4;\n\tmov.b32 {c, d}, %5;\n\t"
      "cvt.rn.f16x2.e4m3x2 %0, a;\n\tcvt.rn.f16x2.e4m3x2 %1, b;\n\t"
      "cvt.rn.f16x2.e4m3x2 %2, c;\n\tcvt.rn.f16x2.e4m3x2 %3, d;\n\t}"
      : "=r"(o.x), "=r"(o.y), "=r"(o.z), "=r"(o.w)
      : "r"(lo), "r"(hi));
  return o;
}

__device__ __forceinline__ float acc_max(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ int acc_max(int a, int b) { return max(a, b); }
__device__ __forceinline__ float acc_max3(float a, float b, float c) { return fmax3(a, b, c); }
__device__ __forceinline__ int acc_max3(int a, int b, int c) { return imax3(a, b, c); }

// m64n128 accumulator fragment (ptx.cuh) -> r0[c] / r1[c] = max over this thread's 8 of the 32 columns of chunk c (columns
// 32c .. 32c+31) of its token row l/4 (r0) and l/4 + 8 (r1).  The other 24 columns live in the other lanes of the quad: max
// is exact and order-free, so callers keep per-lane partial maxima and combine the quad once, with quad_max.
template <typename Acc>
__device__ __forceinline__ void chunk_maxima(const Acc (&d)[64], Acc (&r0)[4], Acc (&r1)[4]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    Acc a = acc_max(d[16 * c + 0], d[16 * c + 1]);
    Acc b = acc_max(d[16 * c + 2], d[16 * c + 3]);
#pragma unroll
    for (int j = 4 * c + 1; j < 4 * c + 4; ++j) {
      a = acc_max3(a, d[4 * j + 0], d[4 * j + 1]);
      b = acc_max3(b, d[4 * j + 2], d[4 * j + 3]);
    }
    r0[c] = a;
    r1[c] = b;
  }
}

// max over the four lanes of a quad (the lanes that share an accumulator row)
template <typename Acc>
__device__ __forceinline__ Acc quad_max(Acc v) {
  v = acc_max(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return acc_max(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// zero_pad_compat (option "zero_pad_compat"): colpali_engine's score_multi_vector pads every batch of pages with zero rows
// up to the longest page of the batch and lets them take part in the max (transformers port processing_colpali.py:350-362),
// so a page shorter than its batch's longest scores sum_t max(true max_t, 0).  clamp_bits bit i = "page (or candidate slot) i
// is shorter than the longest of its batch"; NULL = clean MaxSim (the default).
template <typename Acc>
__device__ __forceinline__ Acc clamp_token_max(const uint32_t* __restrict__ clamp_bits, int idx, Acc rm) {
  if (clamp_bits != nullptr && ((__ldg(clamp_bits + (idx >> 5)) >> (idx & 31)) & 1u)) return acc_max(rm, Acc(0));
  return rm;
}

}  // namespace bms
