// duplicates.cu -- near-duplicate pages: both directions of page-to-page MaxSim for a list of page pairs
// (b200ms_pair_maxsim_device), and duplicate groups as the connected components of the pairs whose smaller direction
// reaches a threshold (b200ms_duplicate_groups_device).
//
// Pair kernel.  sim(a -> b) needs, per true row of a, the max over b's true rows; sim(b -> a) needs, per true row of b, the
// max over a's true rows.  Both are reductions of the same row x row product, so one CTA (one warpgroup) runs a against b
// once through row_tiles.cuh's row_block_maxsim (A = 64-row blocks of a, B = 128-row tiles of b), the routine
// mmr_round_wgmma runs: it gives the row maxima, and its per-tile hook takes the column maxima, folded over a's blocks into
// one value per row of b (shared memory for pages up to kPairSmemCols rows, else a slice of global scratch owned by the
// CTA).  Maxima commute, so neither depends on the schedule.  Both sums take b200ms_mmr_device's order from the same
// helpers (ordered_sum, page_sim).  1-bit corpora run row_block_maxsim_b1 (128 - popc on the CUDA cores), as mmr_round_b1
// does, its per-row hook taking the column maxima.
//
// Groups.  Lock-free union-find on the labels: every edge hooks the larger of its two roots onto the smaller with a CAS
// and retries while its endpoints have different roots, so after one pass every component is one tree whose root is its
// smallest page; a second pass points every page at its root.  Labels only ever decrease (atomicMin), so no racing write
// can move a page back down its path.
#include <cmath>

#include "common.cuh"
#include "mma_tile.cuh"
#include "ptx.cuh"
#include "row_tiles.cuh"

namespace bms {

constexpr int kPairSmemCols = 2048;  // column maxima of a page up to this many rows stay in shared memory
constexpr int kLabelThreads = 256;

struct PairArgs {
  const int64_t* pa = nullptr;  // [n_pairs] page ids
  const int64_t* pb = nullptr;
  int64_t n_pairs = 0;
  int64_t n_pages = 0;
  const int32_t* page_len = nullptr;    // [n_pages] TRUE row counts
  const void* rows = nullptr;           // packed rows of the corpus
  const int64_t* page_start = nullptr;  // first padded row per page
  int64_t n_rows = 0;
  float scale = 1.f;
  float* sim_ab = nullptr;
  float* sim_ba = nullptr;
  void* col_scratch = nullptr;  // [gridDim.x, col_stride] column maxima of pages past kPairSmemCols rows
  int64_t col_stride = 0;
};

// one pair: 0 = skip it (written already), else its ids and true lengths
__device__ __forceinline__ bool pair_item(const PairArgs& a, int64_t i, int64_t& pa, int64_t& pb, int& la, int& lb) {
  pa = __ldg(a.pa + i);
  pb = __ldg(a.pb + i);
  if (pa < 0 || pa >= a.n_pages || pb < 0 || pb >= a.n_pages) {
    if (threadIdx.x == 0) a.sim_ab[i] = a.sim_ba[i] = __int_as_float(0x7fffffff);
    return false;
  }
  la = __ldg(a.page_len + pa);
  lb = __ldg(a.page_len + pb);
  if (la == 0 || lb == 0) {  // a page without rows: 0 both ways, as b200ms_mmr_device
    if (threadIdx.x == 0) a.sim_ab[i] = a.sim_ba[i] = 0.f;
    return false;
  }
  return true;
}

// ------------------------------------------------------------------ dense dtypes on wgmma (row_tiles.cuh)
template <int KIND>
__global__ void __launch_bounds__(kRowTileThreads) pair_maxsim_wgmma(const __grid_constant__ PairArgs a) {
  using Acc = typename Kind<KIND>::Acc;
  using P = RowSum<KIND>;
  extern __shared__ uint8_t smem_raw[];
  __shared__ Acc tile_cols[4][kTileN];  // per warp: max over its 16 rows of a, per column of the current tile
  __shared__ Acc col_smem[kPairSmemCols];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t b_addr = smem_u32(smem);
  const uint32_t a_addr = b_addr + Kind<KIND>::kPanels * kSubtileBytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = 16 * warp + (lane >> 2);
  const uint4* prows = static_cast<const uint4*>(a.rows);
  const Acc none = max_none<Acc>();
  Acc* const col_global = static_cast<Acc*>(a.col_scratch) + int64_t(blockIdx.x) * a.col_stride;
  for (int64_t i = blockIdx.x; i < a.n_pairs; i += gridDim.x) {
    int64_t pa, pb;
    int la, lb;
    if (!pair_item(a, i, pa, pb, la, lb)) continue;
    Acc* col = lb <= kPairSmemCols ? col_smem : col_global;
    // column c is only ever touched by thread c % 128 until the sums below
    for (int c = threadIdx.x; c < lb; c += kRowTileThreads) col[c] = none;
    const int64_t a0 = __ldg(a.page_start + pa), b0 = __ldg(a.page_start + pb);
    const P s_ab = ordered_sum<P>((la + kABlockRows - 1) / kABlockRows, [&](int tt) {
      const int rows = la - tt * kABlockRows < kABlockRows ? la - tt * kABlockRows : kABlockRows;
      const bool ok0 = m0 < rows, ok1 = m0 + 8 < rows;
      return row_block_maxsim<KIND>(
          a_addr, b_addr, prows, a0 + int64_t(tt) * kABlockRows, rows, a.n_rows, b0, lb, [&](const Acc(&d)[64], int n) {
#pragma unroll
            for (int jb = 0; jb < 16; ++jb) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                // column 8 jb + 2 (lane & 3) + e of the tile over this warp's true rows of a
                Acc v = ok0 ? d[4 * jb + e] : none;
                if (ok1) v = acc_max(v, d[4 * jb + 2 + e]);
                v = acc_max(v, __shfl_xor_sync(0xffffffffu, v, 4));
                v = acc_max(v, __shfl_xor_sync(0xffffffffu, v, 8));
                v = acc_max(v, __shfl_xor_sync(0xffffffffu, v, 16));
                if (lane < 4) tile_cols[warp][8 * jb + 2 * lane + e] = v;
              }
            }
            __syncthreads();
            const int c = n * kTileN + int(threadIdx.x);
            if (c < lb) {
              const Acc v = acc_max(acc_max(tile_cols[0][threadIdx.x], tile_cols[1][threadIdx.x]),
                                    acc_max(tile_cols[2][threadIdx.x], tile_cols[3][threadIdx.x]));
              col[c] = acc_max(col[c], v);
            }
            // tile_cols is rewritten only after the tile loop's next barrier
          });
    });
    __syncthreads();  // every column maximum is final
    if (threadIdx.x == 0) {
      a.sim_ab[i] = page_sim<P>(s_ab, a.scale, la);
      a.sim_ba[i] = page_sim<P>(block_ordered_sum<P>(col, lb), a.scale, lb);
    }
    __syncthreads();  // col is read before the next pair initialises it
  }
}

// ------------------------------------------------------------------ 1-bit corpora: 128 - popc(a ^ b), exact
__global__ void __launch_bounds__(kRowBlockB1Threads) pair_maxsim_b1(const __grid_constant__ PairArgs a) {
  __shared__ int col_smem[kPairSmemCols];
  const int warp = threadIdx.x >> 5;
  const uint4* prows = static_cast<const uint4*>(a.rows);
  int* const col_global = static_cast<int*>(a.col_scratch) + int64_t(blockIdx.x) * a.col_stride;
  for (int64_t i = blockIdx.x; i < a.n_pairs; i += gridDim.x) {
    int64_t pa, pb;
    int la, lb;
    if (!pair_item(a, i, pa, pb, la, lb)) continue;
    int* col = lb <= kPairSmemCols ? col_smem : col_global;
    for (int c = threadIdx.x; c < lb; c += kRowBlockB1Threads) col[c] = INT32_MIN;
    __syncthreads();  // the column maxima are updated by every warp
    const int64_t a0 = __ldg(a.page_start + pa), b0 = __ldg(a.page_start + pb);
    const long long s_ab = ordered_sum<long long>((la + kABlockRows - 1) / kABlockRows, [&](int tt) {
      const int rows = la - tt * kABlockRows < kABlockRows ? la - tt * kABlockRows : kABlockRows;
      const int warp_rows = rows - warp * kB1RowsPerWarp;  // this warp's true rows of the block (may be <= 0)
      return row_block_maxsim_b1(prows, a0 + int64_t(tt) * kABlockRows, rows, b0, lb,
                                 [&](int row, const int (&v)[kB1RowsPerWarp]) {
                                   int cm = INT32_MIN;
#pragma unroll
                                   for (int k = 0; k < kB1RowsPerWarp; ++k)
                                     if (k < warp_rows) cm = max(cm, v[k]);
                                   if (warp_rows > 0) atomicMax(col + row, cm);
                                 });
    });
    // row_block_maxsim_b1 ends with a barrier (la > 0): every column maximum is final
    if (threadIdx.x == 0) {
      a.sim_ab[i] = page_sim<long long>(s_ab, a.scale, la);
      a.sim_ba[i] = page_sim<long long>(block_ordered_sum<long long>(col, lb), a.scale, lb);
    }
    __syncthreads();  // col is read before the next pair initialises it
  }
}

// ------------------------------------------------------------------ duplicate groups
__device__ __forceinline__ bool page_allowed(const uint32_t* allow, int64_t p) {
  return allow == nullptr || ((__ldg(allow + (p >> 5)) >> (p & 31)) & 1u);
}

__global__ void __launch_bounds__(kLabelThreads)
labels_init_kernel(int64_t* __restrict__ labels, int64_t n_pages, const uint32_t* __restrict__ allow) {
  for (int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; p < n_pages; p += int64_t(gridDim.x) * blockDim.x)
    labels[p] = page_allowed(allow, p) ? p : -1;
}

// the root of x's tree, pointing each page on the way at its grandparent.  Every page's ancestors have smaller ids, so
// the pointer is lowered with atomicMin: a racing thread holding an older ancestor can never undo a higher one (a plain
// store could, and after the last pass it could leave a page pointing below its root).
__device__ __forceinline__ int64_t find_root(volatile int64_t* L, int64_t x) {
  int64_t p = L[x];
  while (p != x) {
    const int64_t g = L[p];
    if (g != p) atomicMin(reinterpret_cast<long long*>(const_cast<int64_t*>(L + x)), static_cast<long long>(g));
    x = p;
    p = g;
  }
  return x;
}

__global__ void __launch_bounds__(kLabelThreads)
hook_edges_kernel(const int64_t* __restrict__ pa, const int64_t* __restrict__ pb, const float* __restrict__ sab,
                  const float* __restrict__ sba, int64_t n_pairs, float threshold, int64_t n_pages,
                  const uint32_t* __restrict__ allow, int64_t* labels) {
  volatile int64_t* L = labels;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n_pairs; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t u = __ldg(pa + i), v = __ldg(pb + i);
    if (u < 0 || u >= n_pages || v < 0 || v >= n_pages || u == v) continue;
    // dup = min of the two directions >= threshold; a NaN in either direction fails the comparison
    if (!(__ldg(sab + i) >= threshold && __ldg(sba + i) >= threshold)) continue;
    if (!page_allowed(allow, u) || !page_allowed(allow, v)) continue;
    while (true) {
      int64_t ru = find_root(L, u), rv = find_root(L, v);
      if (ru == rv) break;
      if (ru > rv) {
        const int64_t t = ru;
        ru = rv;
        rv = t;
      }
      // rv is still a root: it becomes a child of ru; else another edge hooked it first and the roots are found again
      if (atomicCAS(reinterpret_cast<unsigned long long*>(labels + rv), static_cast<unsigned long long>(rv),
                    static_cast<unsigned long long>(ru)) == static_cast<unsigned long long>(rv))
        break;
    }
  }
}

__global__ void __launch_bounds__(kLabelThreads) labels_finish_kernel(int64_t* labels, int64_t n_pages) {
  volatile int64_t* L = labels;
  for (int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; p < n_pages; p += int64_t(gridDim.x) * blockDim.x)
    if (L[p] >= 0) atomicMin(reinterpret_cast<long long*>(labels + p), static_cast<long long>(find_root(L, p)));
}

}  // namespace bms

using namespace bms;

#define B200MS_API extern "C" __attribute__((visibility("default")))

B200MS_API int b200ms_pair_maxsim_device(b200ms_t* h, const int64_t* pair_a_dev, const int64_t* pair_b_dev, int64_t n_pairs,
                                         float score_scale, float* sim_ab_dev, float* sim_ba_dev, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  if (n_pairs < 0 || (n_pairs > 0 && (!pair_a_dev || !pair_b_dev || !sim_ab_dev || !sim_ba_dev)) ||
      !(score_scale > 0.f && score_scale < INFINITY))
    return set_error(h, B200MS_EINVAL,
                     "pair_maxsim_device: bad arguments (n_pairs >= 0, NULL arrays, score_scale finite and > 0)");
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "pair_maxsim: no corpus attached (call b200ms_set_corpus first)");
  if (c.host) return set_error(h, B200MS_ESTATE, "pair_maxsim: a host-resident corpus is not supported (HBM corpora only)");
  if (c.dtype != B200MS_B1 && kind_of_dtype(c.dtype) < 0)
    return set_error(h, B200MS_ESTATE, "pair_maxsim: corpus dtype has no scorer");
  if (n_pairs == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  RowTileKernel<PairArgs> k;
  if (int e = row_tile_kernel(h, c.dtype, pair_maxsim_wgmma<0>, pair_maxsim_wgmma<1>, pair_maxsim_wgmma<2>, pair_maxsim_b1,
                              kRowBlockB1Threads, "pair_maxsim", &k))
    return e;
  // one CTA per pair in a grid-stride loop: as many CTAs as fit on the card at once
  int per_sm = 0;
  if (int e = check_cuda(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, reinterpret_cast<const void*>(k.fn),
                                                                          k.threads, size_t(k.smem)),
                         "pair_maxsim: occupancy"))
    return e;
  const int64_t cap = int64_t(h->num_sms) * (per_sm > 0 ? per_sm : 1);
  const int grid = int(n_pairs < cap ? n_pairs : cap);
  PairArgs a;
  a.pa = pair_a_dev;
  a.pb = pair_b_dev;
  a.n_pairs = n_pairs;
  a.n_pages = c.n_pages;
  a.page_len = static_cast<const int32_t*>(h->page_len.p);
  const CorpusView v = corpus_view(h);
  a.rows = v.rows;
  a.page_start = v.page_start;
  a.n_rows = v.n_rows;
  a.scale = score_scale;
  a.sim_ab = sim_ab_dev;
  a.sim_ba = sim_ba_dev;
  if (c.max_page_rows > kPairSmemCols) {  // padded rows bound the true rows of every page
    if (int e = reserve(h, h->dup_cols, size_t(grid) * size_t(c.max_page_rows) * 4)) return e;
    a.col_scratch = h->dup_cols.p;
    a.col_stride = c.max_page_rows;
  }
  return launch_row_tiles(h, k, dim3(grid), a, s, "launch pair_maxsim");
}

B200MS_API int b200ms_duplicate_groups_device(b200ms_t* h, const int64_t* pair_a_dev, const int64_t* pair_b_dev,
                                              const float* sim_ab_dev, const float* sim_ba_dev, int64_t n_pairs,
                                              float threshold, const uint32_t* allow_mask_dev, int64_t* labels_dev,
                                              void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  if (n_pairs < 0 || (n_pairs > 0 && (!pair_a_dev || !pair_b_dev || !sim_ab_dev || !sim_ba_dev)) || !std::isfinite(threshold))
    return set_error(h, B200MS_EINVAL, "duplicate_groups_device: bad arguments (n_pairs >= 0, NULL arrays, finite threshold)");
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "duplicate_groups: no corpus attached (call b200ms_set_corpus first)");
  if (c.host) return set_error(h, B200MS_ESTATE, "duplicate_groups: a host-resident corpus is not supported (HBM corpora only)");
  if (c.n_pages == 0) return B200MS_OK;
  if (!labels_dev) return set_error(h, B200MS_EINVAL, "duplicate_groups_device: labels_dev is NULL");
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  labels_init_kernel<<<grid_stride_blocks(h, c.n_pages, kLabelThreads, 8), kLabelThreads, 0, s>>>(
      labels_dev, c.n_pages, allow_mask_dev);
  h->launches++;
  if (int e = check_cuda(h, cudaGetLastError(), "launch labels_init")) return e;
  if (n_pairs > 0) {
    hook_edges_kernel<<<grid_stride_blocks(h, n_pairs, kLabelThreads, 8), kLabelThreads, 0, s>>>(
        pair_a_dev, pair_b_dev, sim_ab_dev, sim_ba_dev, n_pairs, threshold, c.n_pages, allow_mask_dev, labels_dev);
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch hook_edges")) return e;
  }
  labels_finish_kernel<<<grid_stride_blocks(h, c.n_pages, kLabelThreads, 8), kLabelThreads, 0, s>>>(labels_dev, c.n_pages);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch labels_finish");
}
