// scan.cuh -- the one-block prefix sum the planning kernels share (host_tier.cu, scan_plan.cu).
#pragma once
#include <stdint.h>

namespace bms {

constexpr int kScanThreads = 1024;

// Exclusive prefix sum of val(0..n) into out[0..n] (out[n] = total) by one block of kScanThreads threads, each summing a
// contiguous span: the order of additions is fixed, so the result is deterministic.
template <class F>
__device__ void block_scan(F val, int64_t n, int64_t* __restrict__ out) {
  __shared__ int64_t part[kScanThreads];
  const int t = threadIdx.x;
  const int64_t per = (n + kScanThreads - 1) / kScanThreads;
  const int64_t i0 = min(n, int64_t(t) * per), i1 = min(n, i0 + per);
  int64_t sum = 0;
  for (int64_t i = i0; i < i1; ++i) sum += val(i);
  part[t] = sum;
  __syncthreads();
  for (int off = 1; off < kScanThreads; off <<= 1) {
    const int64_t v = t >= off ? part[t - off] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int64_t run = part[t] - sum;
  for (int64_t i = i0; i < i1; ++i) {
    out[i] = run;
    run += val(i);
  }
  if (t == kScanThreads - 1) out[n] = part[t];
}

}  // namespace bms
