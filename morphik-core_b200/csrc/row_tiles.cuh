// row_tiles.cuh -- one 64-row block of packed rows (the wgmma A operand) against every 128-row tile of a page (B), on the
// scan's own tensor-core instructions (mma_tile.cuh): bf16 k16 / fp32, s8 k32 / int32, e4m3 widened to f16 k16 / fp32, in
// the scan's K order, so every row x row product is the value the scan takes its max over, bit for bit.
//
// Used by b200ms_explain_device (A = 64 query tokens, maxsim_explain.cu) and, through row_block_maxsim, by page-to-page
// MaxSim: b200ms_mmr_device (maxsim_mmr.cu) and b200ms_pair_maxsim_device (duplicates.cu).  One warpgroup (128 threads) runs
// it; thread r stages row r of every B tile with plain 16-byte loads, the next tile in flight while the current one is on
// the tensor pipe.  Shared memory: the B tile ([kPanels][128 rows x 128 B]) at b_addr, the A block ([kPanels][64 rows x
// 128 B]) right behind it, both 1024-byte aligned.
//
// Page-to-page MaxSim, sim(a -> b) = score_scale * S / len_a with S the sum over a's true rows of each row's max over b's
// true rows, is computed here only, so that every caller's value is the same bit for bit: row_block_maxsim (dense dtypes)
// or row_block_maxsim_b1 (1-bit rows) gives one 64-row block's sum, ordered_sum adds the blocks, page_sim finishes.
#pragma once
#include "common.cuh"
#include "mma_tile.cuh"
#include "ptx.cuh"

namespace bms {

constexpr int kRowTileThreads = 128;         // one warpgroup
constexpr int kABlockRows = 64;              // rows of the A block (one wgmma M block)
constexpr uint32_t kABlockPanel = 64 * 128;  // one 128-byte K panel of the 64-row A block

// dynamic shared memory a kernel that runs rows_vs_page_tiles<KIND> asks for (B tile + A block + alignment slack)
template <int KIND>
constexpr int row_tiles_smem() {
  return 1024 + 3 * Kind<KIND>::kPanels * int(kABlockPanel);
}

// one 128-byte-row K-major SWIZZLE_128B atom: row r, 16-byte chunk c (0..7) of a panel
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return uint32_t(r >> 3) * 1024u + uint32_t(r & 7) * 128u + ((uint32_t(c) ^ uint32_t(r & 7)) << 4);
}

// 16-byte piece c of a stored row -> shared memory (e4m3: two f16 pieces)
template <int KIND>
__device__ __forceinline__ void put_piece(uint32_t base, uint32_t panel_bytes, int row, int c, const uint4& v) {
  if constexpr (KIND == 2) {
    const uint4 lo = e4m3x8_to_f16x8(v.x, v.y), hi = e4m3x8_to_f16x8(v.z, v.w);
    st_shared_v4(base + uint32_t((2 * c) >> 3) * panel_bytes + sw128_off(row, (2 * c) & 7), lo);
    st_shared_v4(base + uint32_t((2 * c + 1) >> 3) * panel_bytes + sw128_off(row, (2 * c + 1) & 7), hi);
  } else {
    st_shared_v4(base + uint32_t(c >> 3) * panel_bytes + sw128_off(row, c & 7), v);
  }
}

// 16-byte pieces of one stored row
template <int KIND>
constexpr int row_chunks() {
  return KIND == 0 ? 16 : 8;
}

// rows [row0, row0 + 64) of `rows` -> the A block; a row at or past `limit` (the end of what `rows` holds) is zero
template <int KIND>
__device__ __forceinline__ void load_a_block(uint32_t a_addr, const uint4* rows, int64_t row0, int64_t limit) {
  constexpr int kSrcChunks = row_chunks<KIND>();
  constexpr int kPieces = kABlockRows * kSrcChunks / kRowTileThreads;
#pragma unroll
  for (int k = 0; k < kPieces; ++k) {
    const int p = int(threadIdx.x) + k * kRowTileThreads;
    const int row = p / kSrcChunks, c = p % kSrcChunks;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row0 + row < limit) v = __ldg(rows + (row0 + row) * kSrcChunks + c);
    put_piece<KIND>(a_addr, kABlockPanel, row, c, v);
  }
}

// The tile loop.  B = rows [row0, row0 + padded) of `prows` (padded: the page's rows rounded up to 32; rows past it are
// zero), in tiles of 128.  Fetches tile 0, waits until the previous work item's wgmmas have read shared memory, runs
// load_a() (which fills the A block), then per tile n: one m64n128 chain over the 128-d rows and epi(d, n) with the
// accumulators d (ptx.cuh fragment layout: d[4 jb + 2 h + e] is A row 16 warp + lane/4 + 8 h, B row 128 n + 8 jb +
// 2 (lane & 3) + e).  Every thread of the warpgroup calls it with the same arguments.
template <int KIND, class LoadA, class Epi>
__device__ __forceinline__ void rows_vs_page_tiles(uint32_t a_addr, uint32_t b_addr, const uint4* prows, int64_t row0,
                                                   int padded, LoadA&& load_a, Epi&& epi) {
  using K = Kind<KIND>;
  using Acc = typename K::Acc;
  constexpr int kSrcChunks = row_chunks<KIND>();
  const int r = threadIdx.x;  // B: row r of every page tile
  const int n_tiles = (padded + kTileN - 1) / kTileN;
  uint4 nxt[kSrcChunks];
  auto fetch = [&](int n) {
    const int row = n * kTileN + r;
#pragma unroll
    for (int c = 0; c < kSrcChunks; ++c) nxt[c] = make_uint4(0, 0, 0, 0);
    if (row < padded) {
#pragma unroll
      for (int c = 0; c < kSrcChunks; ++c) nxt[c] = __ldg(prows + (row0 + row) * kSrcChunks + c);
    }
  };
  fetch(0);
  __syncthreads();  // the previous item's wgmmas have read the A block
  load_a();
  for (int n = 0; n < n_tiles; ++n) {
    if (n > 0) __syncthreads();  // the previous tile's wgmmas have read the B tile
#pragma unroll
    for (int c = 0; c < kSrcChunks; ++c) put_piece<KIND>(b_addr, kSubtileBytes, r, c, nxt[c]);
    fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core's async-proxy reads
    __syncthreads();
    Acc d[64];
    wgmma_fence();
    {
      const uint64_t ad = wgmma_desc_kmajor_sw128(a_addr), bd = wgmma_desc_kmajor_sw128(b_addr);
#pragma unroll
      for (int ks = 0; ks < K::kKSteps; ++ks) {  // 32 B of K per step, 4 steps per 128 B panel: the scan's order
        const uint32_t ao = ((ks >> 2) * kABlockPanel + (ks & 3) * 32) >> 4;
        const uint32_t bo = ((ks >> 2) * kSubtileBytes + (ks & 3) * 32) >> 4;
        if constexpr (KIND == 0) {
          wgmma_m64n128k16_bf16(d, ad + ao, bd + bo, ks != 0);
        } else if constexpr (KIND == 1) {
          wgmma_m64n128k32_s8(d, ad + ao, bd + bo, ks != 0);
        } else {
          wgmma_m64n128k16_f16(d, ad + ao, bd + bo, ks != 0);
        }
      }
      wgmma_commit();
    }
    if (n + 1 < n_tiles) fetch(n + 1);  // in flight while the chain runs
    wgmma_wait<0>();
    reg_fence_all(d);
    epi(d, n);
  }
}

// ------------------------------------------------------------------ page-to-page MaxSim
// The sum type of a page's row maxima: float, or long long for int8 and 1-bit rows (int32 maxima)
template <int KIND>
using RowSum = typename std::conditional<KIND == 1, long long, float>::type;

// The max over no row yet: fmaxf's identity (a NaN row max stays NaN only when every row is NaN) / the least int
template <typename Acc>
__device__ __forceinline__ Acc max_none() {
  if constexpr (std::is_same<Acc, float>::value) {
    return __int_as_float(0x7fffffff);
  } else {
    return INT32_MIN;
  }
}

// The one summation order of page-to-page MaxSim: term(0) + term(1) + ... from P(0).  A 64-row block adds its rows' maxima
// so, and a page adds its blocks' sums so.
template <typename P, class Term>
__device__ __forceinline__ P ordered_sum(int n, Term&& term) {
  P s = P(0);
  for (int i = 0; i < n; ++i) s += term(i);
  return s;
}

// v[0 .. len) in that order: each 64-row block in row order, the blocks in order
template <typename P, typename V>
__device__ __forceinline__ P block_ordered_sum(const V* v, int len) {
  return ordered_sum<P>((len + kABlockRows - 1) / kABlockRows, [&](int t) {
    const int r0 = t * kABlockRows;
    return ordered_sum<P>(len - r0 < kABlockRows ? len - r0 : kABlockRows, [&](int r) { return P(v[r0 + r]); });
  });
}

// sim = score_scale * S / len in fp32, every operation rounded (no contraction)
template <typename P>
__device__ __forceinline__ float page_sim(P s, float scale, int len) {
  float sf;
  if constexpr (std::is_same<P, float>::value) {
    sf = s;
  } else {
    sf = __ll2float_rn(s);
  }
  return __fdiv_rn(__fmul_rn(sf, scale), float(len));
}

struct NoHook {
  template <class... T>
  __device__ __forceinline__ void operator()(T&&...) const {}
};

// One 64-row block of page a against page b (dense dtypes, one warpgroup): A = rows [a_row0, a_row0 + 64) of prows (reads at
// or past a_limit are zero), of which the first `rows` are a's; B = b's len_b true rows from b_row0.  Per A row the max over
// b's true rows; returns in thread 0 the sum of the first `rows` maxima in row order.  hook(d, n) sees each tile's
// accumulators (row_tiles layout) before the row maxima are taken from them.  rowmax is rewritten only after the next call's first
// barrier, so calls may follow each other without one.
template <int KIND, class Hook = NoHook>
__device__ __forceinline__ RowSum<KIND> row_block_maxsim(uint32_t a_addr, uint32_t b_addr, const uint4* prows,
                                                         int64_t a_row0, int rows, int64_t a_limit, int64_t b_row0,
                                                         int len_b, Hook&& hook = Hook()) {
  using Acc = typename Kind<KIND>::Acc;
  using P = RowSum<KIND>;
  __shared__ Acc rowmax[kABlockRows];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = 16 * warp + (lane >> 2);
  Acc mx0 = max_none<Acc>(), mx1 = max_none<Acc>();  // A rows m0 and m0 + 8: this lane's max over its columns
  rows_vs_page_tiles<KIND>(
      a_addr, b_addr, prows, b_row0, (len_b + kGroup - 1) & ~(kGroup - 1),
      [&] { load_a_block<KIND>(a_addr, prows, a_row0, a_limit); },
      [&](const Acc(&d)[64], int n) {
        hook(d, n);
        const int rbase = n * kTileN + 2 * (lane & 3);
#pragma unroll
        for (int jb = 0; jb < 16; ++jb) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (rbase + 8 * jb + e < len_b) {
              mx0 = acc_max(mx0, d[4 * jb + e]);
              mx1 = acc_max(mx1, d[4 * jb + 2 + e]);
            }
          }
        }
      });
  mx0 = quad_max(mx0);
  mx1 = quad_max(mx1);
  if ((lane & 3) == 0) {
    rowmax[m0] = mx0;
    rowmax[m0 + 8] = mx1;
  }
  __syncthreads();
  P s = P(0);
  if (threadIdx.x == 0) s = ordered_sum<P>(rows, [&](int r) { return P(rowmax[r]); });
  return s;
}

constexpr int kRowBlockB1Threads = 256;  // 1-bit row block: 8 warps, 8 A rows each
constexpr int kB1RowsPerWarp = kABlockRows / (kRowBlockB1Threads / 32);

// row_block_maxsim for 1-bit rows (kRowBlockB1Threads threads): 128 - popc(a ^ b), exact.  Lane l of every warp walks b's
// rows l, l + 32, ...; hook(row, v) sees v[k], the value of this warp's A row k against that b row (rows past `rows` are
// zero rows).  Ends with a barrier, after which the next call may rewrite rowmax.
template <class Hook = NoHook>
__device__ __forceinline__ long long row_block_maxsim_b1(const uint4* prows, int64_t a_row0, int rows, int64_t b_row0,
                                                         int len_b, Hook&& hook = Hook()) {
  __shared__ int rowmax[kABlockRows];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint4 av[kB1RowsPerWarp];
  int mx[kB1RowsPerWarp];
#pragma unroll
  for (int k = 0; k < kB1RowsPerWarp; ++k) {
    const int r = warp * kB1RowsPerWarp + k;
    av[k] = r < rows ? __ldg(prows + a_row0 + r) : make_uint4(0, 0, 0, 0);
    mx[k] = INT32_MIN;
  }
  for (int row = lane; row < len_b; row += 32) {
    const uint4 dv = __ldg(prows + b_row0 + row);
    int v[kB1RowsPerWarp];
#pragma unroll
    for (int k = 0; k < kB1RowsPerWarp; ++k) {
      v[k] = 128 - (__popc(av[k].x ^ dv.x) + __popc(av[k].y ^ dv.y) + __popc(av[k].z ^ dv.z) + __popc(av[k].w ^ dv.w));
      mx[k] = max(mx[k], v[k]);
    }
    hook(row, v);
  }
#pragma unroll
  for (int k = 0; k < kB1RowsPerWarp; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx[k] = max(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
    if (lane == 0) rowmax[warp * kB1RowsPerWarp + k] = mx[k];
  }
  __syncthreads();
  long long s = 0;
  if (threadIdx.x == 0) s = ordered_sum<long long>(rows, [&](int r) { return (long long)rowmax[r]; });
  __syncthreads();  // rowmax is read before the next call writes it
  return s;
}

// ------------------------------------------------------------------ host side
// The kernel of a row-tile family that scores a corpus dtype: wgmma<kind_of_dtype(dtype)> on one warpgroup with
// row_tiles_smem<kind>() bytes of dynamic shared memory, or b1 on b1_threads threads for 1-bit rows
template <class Args>
struct RowTileKernel {
  void (*fn)(Args) = nullptr;
  int threads = 0, smem = 0;
};

// *k = that kernel, with its shared-memory opt-in raised (ensure_smem); `what` names the family in errors
template <class Args>
int row_tile_kernel(b200ms_t* h, int dtype, void (*wgmma0)(Args), void (*wgmma1)(Args), void (*wgmma2)(Args),
                    void (*b1)(Args), int b1_threads, const char* what, RowTileKernel<Args>* k) {
  if (dtype == B200MS_B1) {
    *k = {b1, b1_threads, 0};
    return B200MS_OK;
  }
  switch (kind_of_dtype(dtype)) {
    case 0: *k = {wgmma0, kRowTileThreads, row_tiles_smem<0>()}; break;
    case 1: *k = {wgmma1, kRowTileThreads, row_tiles_smem<1>()}; break;
    case 2: *k = {wgmma2, kRowTileThreads, row_tiles_smem<2>()}; break;
    default: return set_error(h, B200MS_ESTATE, std::string(what) + ": corpus dtype has no scorer");
  }
  return ensure_smem(h, reinterpret_cast<const void*>(k->fn), k->smem, what);
}

// One launch of k on stream s, counted in h->launches
template <class Args>
int launch_row_tiles(b200ms_t* h, const RowTileKernel<Args>& k, dim3 grid, const Args& a, cudaStream_t s, const char* what) {
  void* args[] = {const_cast<Args*>(&a)};
  if (int e = check_cuda(h, cudaLaunchKernel(reinterpret_cast<const void*>(k.fn), grid, dim3(k.threads), args,
                                             size_t(k.smem), s),
                         what))
    return e;
  h->launches++;
  return check_cuda(h, cudaGetLastError(), what);
}

}  // namespace bms
