// maxsim_mmr.cu -- diversified results by maximal marginal relevance (b200ms_mmr_device): a greedy pick over each query's
// candidate list that trades a page's relevance against how much of it the pages picked so far already cover.
//
// Coverage is page-to-page MaxSim, sim(j -> s) = sum over the true rows of j of the max over the true rows of s of the row
// dot product, per row of j.  Rows against rows of two pages is the scan's work, so it runs on the scan's instructions:
// the dense dtypes through row_tiles.cuh's row_block_maxsim (the tile loop b200ms_explain_device uses; A = a 64-row tile of
// candidate j, B = the page picked last, in 128-row tiles), 1-bit corpora through row_block_maxsim_b1 (128 - popc on the
// CUDA cores).  b200ms_pair_maxsim_device (duplicates.cu) runs the same routines, so its sims are these bit for bit.
//
// One call = a setup kernel (outputs, the live-slot table with the duplicate rule, pick 1 by relevance) and per further pick
// two kernels on the caller's stream, without a host synchronisation:
//   round  work item (query, slot j, 64-row tile of page j): per row of the tile the max against the last pick, the sum of
//          the tile's true rows in row order -> one partial per (slot, tile)
//   pick   one CTA per query: adds each live slot's partials in tile order (deterministic, no float atomics), folds the sim
//          into red, and picks the best value lambda * rel - (1 - lambda) * red for the next round.
// A slot that is picked, unused or a repeat of an earlier slot's page is never scored again.
#include <cstring>
#include <vector>

#include "common.cuh"
#include "mma_tile.cuh"
#include "ptx.cuh"
#include "row_tiles.cuh"
#include "topk_keys.cuh"

namespace bms {

constexpr int kMmrPickThreads = 256;  // setup / pick kernels: one CTA per query

struct MmrArgs {
  const int64_t* ids = nullptr;       // [n_q, n_cand] corpus page ids (-1 / out of range = unused slot)
  const float* scores = nullptr;      // [n_q, n_cand] the candidates' reported scores
  const int64_t* unit_ids = nullptr;  // the same slots as pages of the view (the ids themselves for an HBM corpus)
  const int32_t* q_lens = nullptr;    // [n_q] true query tokens (device copy)
  int n_q = 0, n_cand = 0, k = 0;
  int n_tiles = 0;                    // 64-row tiles of the corpus' longest page: partials per slot
  int64_t n_pages = 0;
  const int32_t* page_len = nullptr;  // [n_pages] TRUE row counts, by corpus id
  const void* rows = nullptr;         // the view's packed rows
  const int64_t* page_start = nullptr;  // the view's first padded row per page
  int64_t n_rows = 0;                 // rows the view holds (A-block reads past it are zero)
  float lambda = 0.5f, scale = 1.f;
  uint8_t* live = nullptr;            // [n_q, n_cand] valid, first slot of its page, not picked yet
  float* red = nullptr;               // [n_q, n_cand] fmaxf of the sims against the picks so far (NaN: none yet)
  int32_t* pick = nullptr;            // [n_q] slot of the last pick; -1: the list is exhausted
  void* partials = nullptr;           // [n_q, n_cand, n_tiles] float (BF16 / F8) or int64 (I8 / B1) tile sums
  int64_t* out_ids = nullptr;         // [n_q, k]
  float* out_scores = nullptr;        // [n_q, k]
  int32_t* out_counts = nullptr;      // [n_q]
  float* sims = nullptr;              // [n_q, k, n_cand] or NULL
};

__device__ __forceinline__ int slot_len(const MmrArgs& a, int64_t slot) {
  const int64_t pid = __ldg(a.ids + slot);
  return (pid >= 0 && pid < a.n_pages) ? __ldg(a.page_len + pid) : 0;
}

// rel = score / T_q (T_q = 0: the score), fp32
__device__ __forceinline__ float rel_of(const MmrArgs& a, int q, int64_t slot) {
  const float sc = __ldg(a.scores + slot);
  const int t = __ldg(a.q_lens + q);
  return t > 0 ? __fdiv_rn(sc, float(t)) : sc;
}

// the value of a later pick, every operation rounded to fp32 (no contraction)
__device__ __forceinline__ float mmr_value(float lambda, float rel, float red) {
  return __fsub_rn(__fmul_rn(lambda, rel), __fmul_rn(__fsub_rn(1.f, lambda), red));
}

// Pick i of query q among its live slots (all threads of the block): the highest value in b200ms_topk's total order, ties
// to the lower slot.  No live slot: the list is exhausted.
__device__ void choose(const MmrArgs& a, int q, int i) {
  __shared__ unsigned long long warp_best[kMmrPickThreads / 32];
  const int64_t base = int64_t(q) * a.n_cand;
  // pick 1, and every pick with lambda == 1, by rel alone: red is not read (0 * inf would make a NaN of it)
  const bool by_rel = i == 0 || a.lambda == 1.f;
  unsigned long long best = 0;  // (key << 32) | ~slot; 0 = nothing (every key of a real value is > 0)
  for (int j = threadIdx.x; j < a.n_cand; j += blockDim.x) {
    if (!a.live[base + j]) continue;
    const float rel = rel_of(a, q, base + j);
    const float v = by_rel ? rel : mmr_value(a.lambda, rel, a.red[base + j]);
    const unsigned long long c = (static_cast<unsigned long long>(key_of_canonical(v)) << 32) | (0xffffffffu - uint32_t(j));
    best = c > best ? c : best;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  if ((threadIdx.x & 31) == 0) warp_best[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < int(blockDim.x >> 5); ++w) best = warp_best[w] > best ? warp_best[w] : best;
    if (best) {
      const int j = int(0xffffffffu - uint32_t(best & 0xffffffffu));
      a.out_ids[int64_t(q) * a.k + i] = __ldg(a.ids + base + j);
      a.out_scores[int64_t(q) * a.k + i] = __ldg(a.scores + base + j);
      a.out_counts[q] = i + 1;
      a.live[base + j] = 0;
      a.pick[q] = j;
    } else {
      a.pick[q] = -1;
    }
  }
  __syncthreads();
}

// outputs, the live-slot table and pick 0; n_picks > 1 (lambda == 1 without sims): the following picks by rel alone too
__global__ void __launch_bounds__(kMmrPickThreads) mmr_setup_kernel(const __grid_constant__ MmrArgs a, int n_picks) {
  __shared__ int64_t sid[B200MS_MAX_K];
  const int q = blockIdx.x;
  const int64_t base = int64_t(q) * a.n_cand;
  const float ninf = -__int_as_float(0x7f800000), qnan = __int_as_float(0x7fffffff);
  for (int i = threadIdx.x; i < a.k; i += blockDim.x) {
    a.out_ids[int64_t(q) * a.k + i] = -1;
    a.out_scores[int64_t(q) * a.k + i] = ninf;
  }
  if (a.sims)
    for (int64_t e = threadIdx.x; e < int64_t(a.k) * a.n_cand; e += blockDim.x) a.sims[int64_t(q) * a.k * a.n_cand + e] = ninf;
  if (threadIdx.x == 0) a.out_counts[q] = 0;
  for (int j = threadIdx.x; j < a.n_cand; j += blockDim.x) sid[j] = __ldg(a.ids + base + j);
  __syncthreads();
  // a page listed in several slots counts once, at its earliest slot
  for (int j = threadIdx.x; j < a.n_cand; j += blockDim.x) {
    const int64_t id = sid[j];
    bool ok = id >= 0 && id < a.n_pages;
    for (int i = 0; ok && i < j; ++i) ok = sid[i] != id;
    a.live[base + j] = ok;
    a.red[base + j] = qnan;
  }
  __syncthreads();
  for (int i = 0; i < n_picks; ++i) {
    choose(a, q, i);
    if (a.pick[q] < 0) break;  // read after choose's barrier: uniform
  }
}

// sim(j -> s) from slot j's partials, added in tile order; 0 when either page has no rows
template <typename P>
__device__ __forceinline__ float finish_sim(const MmrArgs& a, int64_t slot, int len_j, int len_s) {
  if (len_j == 0 || len_s == 0) return 0.f;
  const P* p = static_cast<const P*>(a.partials) + slot * a.n_tiles;
  return page_sim<P>(ordered_sum<P>((len_j + kABlockRows - 1) / kABlockRows, [&](int t) { return p[t]; }), a.scale, len_j);
}

// sims against pick i - 1 into red (and row i - 1 of sims), then pick i; choose_next == 0: the sims row only
template <typename P>
__global__ void __launch_bounds__(kMmrPickThreads) mmr_pick_kernel(const __grid_constant__ MmrArgs a, int i, int choose_next) {
  const int q = blockIdx.x;
  const int ps = a.pick[q];
  if (ps < 0) return;  // exhausted (uniform)
  const int64_t base = int64_t(q) * a.n_cand;
  const int len_s = slot_len(a, base + ps);
  for (int j = threadIdx.x; j < a.n_cand; j += blockDim.x) {
    if (!a.live[base + j]) continue;
    const float sim = finish_sim<P>(a, base + j, slot_len(a, base + j), len_s);
    if (a.sims) a.sims[(int64_t(q) * a.k + (i - 1)) * a.n_cand + j] = sim;
    a.red[base + j] = fmaxf(a.red[base + j], sim);
  }
  if (choose_next) choose(a, q, i);
}

// What one round work item computes: rows [64 tt, 64 tt + rows) of slot j's page against the last pick s
struct MmrItem {
  int rows, len_s;
  int64_t a_row0, b_row0;
  bool compute;
};

__device__ __forceinline__ MmrItem mmr_item(const MmrArgs& a, int64_t slot, int tt) {
  MmrItem x;
  x.compute = false;
  x.rows = x.len_s = 0;
  x.a_row0 = x.b_row0 = 0;
  if (!a.live[slot]) return x;
  const int q = int(slot / a.n_cand);
  const int ps = a.pick[q];
  if (ps < 0) return x;
  x.rows = slot_len(a, slot) - tt * kABlockRows;
  if (x.rows <= 0) return x;
  if (x.rows > kABlockRows) x.rows = kABlockRows;
  const int64_t sslot = int64_t(q) * a.n_cand + ps;
  x.len_s = slot_len(a, sslot);
  if (x.len_s == 0) return x;
  x.a_row0 = __ldg(a.page_start + __ldg(a.unit_ids + slot)) + int64_t(tt) * kABlockRows;
  x.b_row0 = __ldg(a.page_start + __ldg(a.unit_ids + sslot));
  x.compute = true;
  return x;
}

// ------------------------------------------------------------------ dense dtypes on wgmma (row_tiles.cuh)
template <int KIND>
__global__ void __launch_bounds__(kRowTileThreads) mmr_round_wgmma(const __grid_constant__ MmrArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t b_addr = smem_u32(smem);                                  // [kPanels][128 rows x 128 B]
  const uint32_t a_addr = b_addr + Kind<KIND>::kPanels * kSubtileBytes;  // [kPanels][64 rows x 128 B]
  const uint4* prows = static_cast<const uint4*>(a.rows);
  const int64_t n_slots = int64_t(a.n_q) * a.n_cand;
  for (int tt = blockIdx.y; tt < a.n_tiles; tt += gridDim.y)
  for (int64_t slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
    const MmrItem x = mmr_item(a, slot, tt);
    if (!x.compute) continue;
    const RowSum<KIND> s = row_block_maxsim<KIND>(a_addr, b_addr, prows, x.a_row0, x.rows, a.n_rows, x.b_row0, x.len_s);
    if (threadIdx.x == 0) static_cast<RowSum<KIND>*>(a.partials)[slot * a.n_tiles + tt] = s;
  }
}

// ------------------------------------------------------------------ 1-bit corpora: 128 - popc(a ^ b), exact
__global__ void __launch_bounds__(kRowBlockB1Threads) mmr_round_b1(const __grid_constant__ MmrArgs a) {
  const uint4* prows = static_cast<const uint4*>(a.rows);
  const int64_t n_slots = int64_t(a.n_q) * a.n_cand;
  for (int tt = blockIdx.y; tt < a.n_tiles; tt += gridDim.y)
  for (int64_t slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
    const MmrItem x = mmr_item(a, slot, tt);
    if (!x.compute) continue;
    const long long s = row_block_maxsim_b1(prows, x.a_row0, x.rows, x.b_row0, x.len_s);
    if (threadIdx.x == 0) static_cast<long long*>(a.partials)[slot * a.n_tiles + tt] = s;
  }
}

// ------------------------------------------------------------------ host side
static int launch_round(b200ms_t* h, const MmrArgs& a, int dtype, cudaStream_t s) {
  // grid.y walks the 64-row tiles, grid.x the slots: about eight CTAs per SM in all (as b200ms_explain_device)
  const int64_t n_slots = int64_t(a.n_q) * a.n_cand;
  const int gy = a.n_tiles < 65535 ? a.n_tiles : 65535;
  int64_t gx = (int64_t(h->num_sms) * 8 + gy - 1) / gy;
  if (gx > n_slots) gx = n_slots;
  const dim3 grid{unsigned(gx), unsigned(gy)};
  RowTileKernel<MmrArgs> k;
  if (int e = row_tile_kernel(h, dtype, mmr_round_wgmma<0>, mmr_round_wgmma<1>, mmr_round_wgmma<2>, mmr_round_b1,
                              kRowBlockB1Threads, "mmr_round", &k))
    return e;
  return launch_row_tiles(h, k, grid, a, s, "launch mmr_round");
}

static int launch_pick(b200ms_t* h, const MmrArgs& a, int dtype, int i, int choose_next, cudaStream_t s) {
  if (dtype == B200MS_BF16 || dtype == B200MS_F8)
    mmr_pick_kernel<float><<<a.n_q, kMmrPickThreads, 0, s>>>(a, i, choose_next);
  else
    mmr_pick_kernel<long long><<<a.n_q, kMmrPickThreads, 0, s>>>(a, i, choose_next);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch mmr_pick");
}

static int run_mmr(b200ms_t* h, const MmrArgs& a, int dtype, bool with_sims, cudaStream_t s) {
  const int picks = a.k < a.n_cand ? a.k : a.n_cand;  // no list yields more picks than it has slots
  const bool rel_only = a.lambda == 1.f && !with_sims;
  mmr_setup_kernel<<<a.n_q, kMmrPickThreads, 0, s>>>(a, rel_only ? picks : 1);
  h->launches++;
  if (int e = check_cuda(h, cudaGetLastError(), "launch mmr_setup")) return e;
  if (rel_only) return B200MS_OK;
  for (int i = 1; i < picks; ++i) {
    if (int e = launch_round(h, a, dtype, s)) return e;
    if (int e = launch_pick(h, a, dtype, i, 1, s)) return e;
  }
  if (!with_sims) return B200MS_OK;
  // the sims against the last pick
  if (int e = launch_round(h, a, dtype, s)) return e;
  return launch_pick(h, a, dtype, picks, 0, s);
}

}  // namespace bms

using namespace bms;

#define B200MS_API extern "C" __attribute__((visibility("default")))

B200MS_API int b200ms_mmr_device(b200ms_t* h, const int64_t* cand_ids, const float* cand_scores, int n_cand,
                                 const int32_t* q_lens, int n_q, int k, float lambda_mult, float score_scale, int64_t* out_ids,
                                 float* out_scores, int32_t* out_counts, float* sims, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  if (!cand_ids || !cand_scores || !q_lens || !out_ids || !out_scores || !out_counts || n_q < 1 || k < 1 ||
      n_cand < 1 || n_cand > B200MS_MAX_K || int64_t(n_q) * n_cand >= (int64_t(1) << 30) ||
      !(lambda_mult >= 0.f && lambda_mult <= 1.f) || !(score_scale > 0.f && score_scale < INFINITY))
    return set_error(h, B200MS_EINVAL,
                     "mmr_device: bad arguments (NULL pointer, n_q >= 1, k >= 1, n_cand in [1, 4096], n_q*n_cand < 2^30, "
                     "lambda_mult in [0, 1], score_scale finite and > 0)");
  for (int i = 0; i < n_q; ++i)
    if (q_lens[i] < 0) return set_error(h, B200MS_EINVAL, "mmr_device: negative query length");
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "mmr: no corpus attached (call b200ms_set_corpus first)");
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  const int64_t n_slots = int64_t(n_q) * n_cand;
  if (c.host) {
    // every pair of candidate pages must be resident together: the call's unique pages must fit one gather round
    std::vector<int64_t> ids(static_cast<size_t>(n_slots));
    if (int e = check_cuda(h, cudaMemcpyAsync(ids.data(), cand_ids, size_t(n_slots) * 8, cudaMemcpyDeviceToHost, s),
                           "mmr: D2H candidate ids"))
      return e;
    if (int e = check_cuda(h, cudaStreamSynchronize(s), "mmr: stream sync")) return e;
    std::vector<uint8_t> seen(static_cast<size_t>(c.n_pages));
    int64_t rows = 0;
    for (int64_t id : ids)
      if (id >= 0 && id < c.n_pages && !seen[size_t(id)]) {
        seen[size_t(id)] = 1;
        rows += b200ms_padded_len(h->page_len_host[size_t(id)]);
      }
    if (host_tier_rounds(h, rows) > 1)
      return set_error(h, B200MS_EINVAL,
                       "mmr_device: the unique candidate pages of a host-resident corpus need more than one gather round "
                       "(option host_stage_bytes)");
  }
  // scratch: live [n_slots] | red [n_slots] | pick [n_q] | q_lens [n_q], and the partials
  const size_t off_red = (size_t(n_slots) + 15) & ~size_t(15);
  const size_t off_pick = off_red + size_t(n_slots) * 4;
  const size_t off_qlens = off_pick + ((size_t(n_q) * 4 + 15) & ~size_t(15));
  const size_t state_bytes = off_qlens + size_t(n_q) * 4;
  const int n_tiles = int((c.max_page_rows + kABlockRows - 1) / kABlockRows);
  if (int e = reserve(h, h->mmr_state, state_bytes)) return e;
  if (int e = reserve(h, h->mmr_partials, size_t(n_slots) * size_t(n_tiles > 0 ? n_tiles : 1) * 8)) return e;
  uint8_t* st = static_cast<uint8_t*>(h->mmr_state.p);
  if (int e = check_cuda(h, cudaMemcpyAsync(st + off_qlens, q_lens, size_t(n_q) * 4, cudaMemcpyHostToDevice, s),
                         "mmr: upload query lengths"))
    return e;
  MmrArgs a;
  a.ids = cand_ids;
  a.scores = cand_scores;
  a.unit_ids = cand_ids;
  a.q_lens = reinterpret_cast<const int32_t*>(st + off_qlens);
  a.n_q = n_q;
  a.n_cand = n_cand;
  a.k = k;
  a.n_tiles = n_tiles > 0 ? n_tiles : 1;
  a.n_pages = c.n_pages;
  a.page_len = static_cast<const int32_t*>(h->page_len.p);
  a.lambda = lambda_mult;
  a.scale = score_scale;
  a.live = st;
  a.red = reinterpret_cast<float*>(st + off_red);
  a.pick = reinterpret_cast<int32_t*>(st + off_pick);
  a.partials = h->mmr_partials.p;
  a.out_ids = out_ids;
  a.out_scores = out_scores;
  a.out_counts = out_counts;
  a.sims = sims;
  const CorpusView whole = corpus_view(h);
  a.rows = whole.rows;
  a.page_start = whole.page_start;
  a.n_rows = whole.n_rows;
  if (!c.host) return run_mmr(h, a, c.dtype, sims != nullptr, s);
  // host-resident corpus: the candidate pages are gathered once, in one round (checked above)
  struct Ctx {
    MmrArgs* a;
  } ctx{&a};
  auto round = [](b200ms_t* hh, const CorpusView& v, const int64_t* remap, int, int rounds, void* p) {
    if (rounds != 1) return set_error(hh, B200MS_EINVAL, "mmr_device: candidate pages need more than one gather round");
    MmrArgs& x = *static_cast<Ctx*>(p)->a;
    x.unit_ids = remap;
    x.rows = v.rows;
    x.page_start = v.page_start;
    x.n_rows = v.n_rows;
    return B200MS_OK;
  };
  if (int e = gather_host_tier(h, cand_ids, n_slots, s, round, &ctx)) return e;
  // no candidate page has a row: every sim is 0 and no round reads a row
  return run_mmr(h, a, c.dtype, sims != nullptr, s);
}
