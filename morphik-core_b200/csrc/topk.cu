// topk.cu -- exact top-k selection over per-page scores and the merge of per-shard candidate lists.
//
// Replaces  ORDER BY similarity DESC LIMIT k  (core/vector_store/multi_vector_store.py:759, with the
// WHERE document_id IN (...) filter :752-757 expressed as a page bitmask) and  torch.topk(scores, min(k, C))
// (core/vector_store/fast_multivector_store.py:556).  The reference leaves ties unspecified; this build orders by
// (score DESC, page id ASC), which is what the oracle's top-k does.
//
// topk_kernel: one 1024-thread CTA per query.  Scores are summed over the query's 32-token groups on the fly,
// mapped to order-preserving 32-bit keys, and the k-th key is found with a 4-pass 8-bit radix select; the
// collect pass takes every key above the threshold plus the lowest-id ties, and a shared-memory bitonic sort
// orders the (at most 4096) winners.  Traffic: n_pages * 4 B * groups * 5 passes per query -- negligible next to the
// corpus scan (128..256 B per patch vector, ~1000 patch vectors per page).
#include <math_constants.h>

#include "common.cuh"
#include "ptx.cuh"
#include "topk_keys.cuh"

namespace bms {

constexpr int kTopkThreads = 1024;

// block-wide bitonic sort (descending) of n2 (power of two) 64-bit keys in shared memory
__device__ void bitonic_desc_u64(uint64_t* a, int n2) {
  for (int size = 2; size <= n2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < n2 / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool desc = (lo & size) == 0;
        const uint64_t x = a[lo], y = a[hi];
        if (desc ? (x < y) : (x > y)) {
          a[lo] = y;
          a[hi] = x;
        }
      }
    }
  }
  __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(kTopkThreads)
topk_kernel(const T* __restrict__ gs, int64_t n_pages, int64_t ld, const int32_t* __restrict__ group_offsets,
            const uint32_t* __restrict__ allow_base, int k, float scale, int64_t id_base, const int64_t* __restrict__ id_map,
            float* __restrict__ top_scores, int64_t* __restrict__ top_ids, int32_t* __restrict__ top_counts,
            int64_t slice_pages, uint32_t* __restrict__ part_keys, int64_t* __restrict__ part_ids,
            const int32_t* __restrict__ mask_index, int64_t mask_stride, int64_t q_stride) {
  // grid = (n_q, n_slices): CTA (q, s) selects the exact top-k of pages [s*slice_pages, (s+1)*slice_pages).  With one slice
  // it writes the final result; otherwise (raw key, id) candidates for topk_merge_kernel (global top-k is a subset of the
  // union of the slices' top-k, and both levels order by (key DESC, id ASC), so the result is identical).
  extern __shared__ uint64_t win[];  // [n2] winners as (key << 32) | (0xffffffff - page)
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_prefix, s_need, s_total, s_gt, s_eq_base;
  __shared__ uint32_t warp_cnt[kTopkThreads / 32];

  const int q = blockIdx.x;
  // one allow-mask for every query (mask_index == NULL), or a row of a mask matrix per query (-1 = unfiltered)
  const uint32_t* allow = allow_base;
  if (mask_index && allow_base) {
    const int mi = __ldg(mask_index + q);
    allow = mi >= 0 ? allow_base + int64_t(mi) * mask_stride : nullptr;
  }
  const int g0 = group_offsets[q], g1 = group_offsets[q + 1];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // q_stride > 0 (batched rerank): query q ranks only its own slots [q*q_stride, q*q_stride + n_pages)
  const int64_t qbase = int64_t(q) * q_stride;
  const int64_t pbeg = qbase + int64_t(blockIdx.y) * slice_pages;
  const int64_t pend = (int64_t(blockIdx.y) + 1) * slice_pages < n_pages ? pbeg + slice_pages : qbase + n_pages;

  // ---- radix select of the k-th largest key (4 x 8 bits, most significant first)
  uint32_t prefix = 0, need = 0, total = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    if (tid < 256) hist[tid] = 0;
    __syncthreads();
    const uint32_t hi_mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    // Scores of one query usually share their leading bytes, so most pages fall into ONE bin: aggregate equal bins inside
    // the warp first (__match_any_sync) -- one shared-memory atomic per distinct bin per warp instead of one per page.
    // 4 pages per thread per trip, all loads issued before the first warp-synchronous step (a __match_any_sync between
    // two dependent loads would expose the full L2/HBM latency on every trip).
    for (int64_t base = pbeg; base < pend; base += 4 * kTopkThreads) {
      uint32_t key[4];
      bool in[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t p = base + u * kTopkThreads + tid;
        key[u] = 0;
        in[u] = p < pend && page_key(gs, ld, g0, g1, allow, p, &key[u]) && (key[u] & hi_mask) == prefix;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t bin = in[u] ? ((key[u] >> shift) & 0xffu) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(0xffffffffu, bin);
        if (in[u] && lane == __ffs(peers) - 1) atomicAdd(&hist[bin], uint32_t(__popc(peers)));
      }
    }
    __syncthreads();
    if (wid == 0) {
      // Which bin holds the need-th largest key?  Lane l owns bins [8l, 8l+8); a suffix scan over the lanes (high bins
      // first) replaces the serial 256-bin walk one thread used to do per pass (~4 us per pass: it dominated the latency of
      // small searches, configs[0]).
      uint32_t loc[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        loc[j] = hist[8 * lane + j];
        sum += loc[j];
      }
      uint32_t suf = sum;  // inclusive suffix sum: keys in bins >= 8*lane
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_down_sync(0xffffffffu, suf, o);
        if (lane + o < 32) suf += v;
      }
      const uint32_t tot = __shfl_sync(0xffffffffu, suf, 0);
      const uint32_t want = pass == 0 ? (tot < uint32_t(k) ? tot : uint32_t(k)) : s_need;
      const uint32_t above = suf - sum;  // keys in bins owned by higher lanes
      if (pass == 0 && lane == 0) s_total = tot;
      if (want == 0) {
        if (lane == 0) {
          s_prefix = prefix | (255u << shift);
          s_need = 0;
        }
      } else if (suf >= want && above < want) {  // exactly one lane
        uint32_t rem = want - above;
        int bsel = -1;
#pragma unroll
        for (int j = 7; j >= 0; --j) {
          if (bsel < 0) {
            if (loc[j] >= rem) bsel = j; else rem -= loc[j];
          }
        }
        s_prefix = prefix | (uint32_t(8 * lane + bsel) << shift);
        s_need = rem;  // how many keys inside that bin are still needed
      }
    }
    __syncthreads();
    prefix = s_prefix;
    need = s_need;
    total = s_total;
    __syncthreads();
  }
  const uint32_t kk = total < uint32_t(k) ? total : uint32_t(k);
  const uint32_t thr = prefix;    // exact k-th largest key
  const uint32_t need_eq = need;  // ties at thr to keep (lowest page ids first)
  int n2 = 1;
  while (n2 < int(kk)) n2 <<= 1;
  for (int i = tid; i < n2; i += kTopkThreads) win[i] = 0;
  if (tid == 0) {
    s_gt = 0;
    s_eq_base = 0;
  }
  __syncthreads();

  // ---- collect: keys > thr anywhere, keys == thr in ascending page order until need_eq are taken
  if (kk > 0) {
    const uint32_t n_gt = kk - need_eq;
    uint32_t nkey = 0;
    bool nvalid = pbeg + tid < pend && page_key(gs, ld, g0, g1, allow, pbeg + tid, &nkey);
    for (int64_t base = pbeg; base < pend; base += kTopkThreads) {
      const int64_t p = base + tid;
      const uint32_t key = nkey;
      const bool valid = nvalid;
      {  // software prefetch of the next chunk: its load overlaps the three block-wide barriers below
        const int64_t pn = p + kTopkThreads;
        nkey = 0;
        nvalid = pn < pend && page_key(gs, ld, g0, g1, allow, pn, &nkey);
      }
      const bool gt = valid && key > thr;
      const bool eq = valid && key == thr;
      if (gt) {
        const uint32_t pos = atomicAdd(&s_gt, 1u);
        win[pos] = (uint64_t(key) << 32) | uint64_t(0xffffffffu - uint32_t(p));
      }
      const uint32_t bal = __ballot_sync(0xffffffffu, eq);
      if (lane == 0) warp_cnt[wid] = __popc(bal);
      __syncthreads();
      uint32_t before = s_eq_base;
      for (int w = 0; w < wid; ++w) before += warp_cnt[w];
      const uint32_t rank = before + __popc(bal & ((1u << lane) - 1u));
      if (eq && rank < need_eq) win[n_gt + rank] = (uint64_t(key) << 32) | uint64_t(0xffffffffu - uint32_t(p));
      __syncthreads();
      if (tid == 0) {
        uint32_t t = 0;
        for (int w = 0; w < kTopkThreads / 32; ++w) t += warp_cnt[w];
        s_eq_base += t;
      }
      __syncthreads();
    }
    bitonic_desc_u64(win, n2);
  }
  for (int i = tid; i < k; i += kTopkThreads) {
    const bool live = uint32_t(i) < kk;
    const uint64_t w = live ? win[i] : 0;
    const int64_t slot = int64_t(0xffffffffu - uint32_t(w));
    const int64_t id = live ? (id_map ? __ldg(id_map + slot) : slot + id_base) : int64_t(-1);
    if (part_keys) {
      // candidate mode hands the merge SLOTS, not page ids: ties must come out in slot order, and the merge maps the winners'
      // slots to page ids itself
      const int64_t o = (int64_t(q) * gridDim.y + blockIdx.y) * k + i;
      part_keys[o] = uint32_t(w >> 32);
      part_ids[o] = (live && id_map) ? slot : id;
    } else {
      top_scores[int64_t(q) * k + i] = live ? score_of_key(uint32_t(w >> 32), T(0)) * scale : -CUDART_INF_F;
      top_ids[int64_t(q) * k + i] = id;
    }
  }
  if (tid == 0 && !part_keys) top_counts[q] = int32_t(kk);
}

// ------------------------------------------------------------------------------------------ small inputs: rank by counting
// n_pages <= 1024 (configs[0]'s 100 pages, every rerank of <= 1024 candidates): one key per thread, each thread counts the
// keys that precede its own -- (key DESC, page ASC), the same total order as the radix path -- and writes itself at that
// rank.  One pass, two barriers; the radix select's four histogram passes cost ~5 us on such inputs, this ~1 us.
template <typename T>
__global__ void __launch_bounds__(kTopkThreads)
topk_small_kernel(const T* __restrict__ gs, int64_t n_pages, int64_t ld, const int32_t* __restrict__ group_offsets,
                  const uint32_t* __restrict__ allow_base, int k, float scale, int64_t id_base, const int64_t* __restrict__ id_map,
                  float* __restrict__ top_scores, int64_t* __restrict__ top_ids, int32_t* __restrict__ top_counts,
                  const int32_t* __restrict__ mask_index, int64_t mask_stride, int64_t q_stride) {
  __shared__ uint32_t s_key[kTopkThreads];
  __shared__ uint8_t s_ok[kTopkThreads];
  __shared__ uint32_t s_total;
  const int q = blockIdx.x;
  const uint32_t* allow = allow_base;
  if (mask_index && allow_base) {
    const int mi = __ldg(mask_index + q);
    allow = mi >= 0 ? allow_base + int64_t(mi) * mask_stride : nullptr;
  }
  const int g0 = group_offsets[q], g1 = group_offsets[q + 1];
  const int tid = threadIdx.x;
  const int n = int(n_pages);
  const int64_t p = int64_t(q) * q_stride + tid;
  uint32_t key = 0;
  const bool valid = tid < n && page_key(gs, ld, g0, g1, allow, p, &key);
  s_key[tid] = key;
  s_ok[tid] = valid ? 1 : 0;
  if (tid == 0) s_total = 0;
  __syncthreads();
  uint32_t rank = 0;
  if (valid) {
    for (int j = 0; j < n; ++j) {
      const uint32_t kj = s_key[j];
      rank += (s_ok[j] && (kj > key || (kj == key && j < tid))) ? 1u : 0u;
    }
    atomicAdd(&s_total, 1u);
  }
  // unused output slots first, then the winners (disjoint slots: ranks are unique)
  for (int i = tid; i < k; i += kTopkThreads) {
    top_scores[int64_t(q) * k + i] = -CUDART_INF_F;
    top_ids[int64_t(q) * k + i] = -1;
  }
  __syncthreads();
  if (valid && rank < uint32_t(k)) {
    top_scores[int64_t(q) * k + rank] = score_of_key(key, T(0)) * scale;
    top_ids[int64_t(q) * k + rank] = id_map ? __ldg(id_map + p) : p + id_base;
  }
  if (tid == 0) top_counts[q] = int32_t(s_total < uint32_t(k) ? s_total : uint32_t(k));
}

// ------------------------------------------------------------------------------------------ merge of candidate lists
__device__ __forceinline__ bool cand_before(uint32_t ka, int64_t ia, uint32_t kb, int64_t ib) {
  return ka > kb || (ka == kb && ia < ib);  // score DESC, id ASC; invalid entries carry key 0 / id INT64_MAX
}

// cand_keys != NULL: candidates carry raw order-preserving keys of score type T (second level of topk_kernel; exact for int
// scores beyond 2^24 too); else float scores (merge of per-shard lists after the all-gather).
// gathered != NULL: candidates come straight from the all-gather buffer -- `world` blocks (one per rank) of
// [n_q*kx int64 ids | n_q*kx f32 scores] (the exchange layout the local top-k is written in, include/b200ms.h); candidate
// i of query q is entry q*kx + i%kx of rank i/kx.  No repacking kernels between the collective and the merge.
// id_map != NULL: the candidate ids are slots of a rerank (second level of topk_kernel in candidate mode); they are ordered
// as slots and reported as id_map[slot].
template <typename T>
__global__ void __launch_bounds__(1024)
merge_topk_kernel(const float* __restrict__ cand_scores, const uint32_t* __restrict__ cand_keys,
                  const int64_t* __restrict__ cand_ids, int m, int n2, int k, float scale, float* __restrict__ top_scores,
                  int64_t* __restrict__ top_ids, int32_t* __restrict__ top_counts, const uint8_t* __restrict__ gathered,
                  int kx, int64_t rank_stride, int64_t scores_off, const int64_t* __restrict__ id_map) {
  extern __shared__ uint8_t msm[];
  int64_t* ids = reinterpret_cast<int64_t*>(msm);
  uint32_t* keys = reinterpret_cast<uint32_t*>(ids + n2);
  __shared__ uint32_t s_valid;
  const int q = blockIdx.x;
  if (threadIdx.x == 0) s_valid = 0;
  __syncthreads();
  uint32_t mine = 0;
  for (int i = threadIdx.x; i < n2; i += blockDim.x) {
    int64_t id = -1;
    uint32_t kraw = 0;
    if (i < m) {
      if (gathered) {
        const uint8_t* blk = gathered + int64_t(i / kx) * rank_stride;
        const int64_t e = int64_t(q) * kx + (i % kx);
        id = reinterpret_cast<const int64_t*>(blk)[e];
        kraw = key_of_canonical(reinterpret_cast<const float*>(blk + scores_off)[e]);
      } else {
        id = cand_ids[int64_t(q) * m + i];
        kraw = cand_keys ? cand_keys[int64_t(q) * m + i] : key_of_canonical(cand_scores[int64_t(q) * m + i]);
      }
    }
    const bool ok = id >= 0;
    keys[i] = ok ? kraw : 0u;
    ids[i] = ok ? id : INT64_MAX;
    mine += ok;
  }
  atomicAdd(&s_valid, mine);
  for (int size = 2; size <= n2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < n2 / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool fwd = (lo & size) == 0;
        const uint32_t ka = keys[lo], kb = keys[hi];
        const int64_t ia = ids[lo], ib = ids[hi];
        const bool swap = fwd ? cand_before(kb, ib, ka, ia) : cand_before(ka, ia, kb, ib);
        if (swap) {
          keys[lo] = kb;
          keys[hi] = ka;
          ids[lo] = ib;
          ids[hi] = ia;
        }
      }
    }
  }
  __syncthreads();
  const uint32_t kk = s_valid < uint32_t(k) ? s_valid : uint32_t(k);
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    const bool live = uint32_t(i) < kk;
    top_scores[int64_t(q) * k + i] = live ? score_of_key(keys[i], T(0)) * scale : -CUDART_INF_F;
    top_ids[int64_t(q) * k + i] = live ? (id_map ? __ldg(id_map + ids[i]) : ids[i]) : int64_t(-1);
  }
  if (threadIdx.x == 0) top_counts[q] = int32_t(kk);
}

template <typename T>
static int launch_merge_impl(b200ms_t* h, const float* cand_scores, const uint32_t* cand_keys, const int64_t* cand_ids, int n_q,
                             int m, int k, float scale, float* top_scores, int64_t* top_ids, int32_t* top_counts,
                             cudaStream_t s, const uint8_t* gathered = nullptr, int kx = 1, int64_t rank_stride = 0,
                             int64_t scores_off = 0, const int64_t* id_map = nullptr) {
  int n2 = 2;
  while (n2 < m) n2 <<= 1;
  const size_t smem = size_t(n2) * (sizeof(int64_t) + sizeof(uint32_t));
  auto kern = merge_topk_kernel<T>;
  if (int e = ensure_smem(h, reinterpret_cast<const void*>(kern), int(smem), "cudaFuncSetAttribute(merge_topk)"))
    return e;
  kern<<<n_q, 1024, smem, s>>>(cand_scores, cand_keys, cand_ids, m, n2, k, scale, top_scores, top_ids, top_counts, gathered, kx,
                               rank_stride, scores_off, id_map);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch merge_topk");
}

int launch_topk(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                const int32_t* group_offsets_dev, int n_q, const uint32_t* allow_mask, int k, float scale,
                int64_t id_base, const int64_t* id_map, float* top_scores, int64_t* top_ids, int32_t* top_counts,
                cudaStream_t s, const int32_t* mask_index, int64_t mask_stride, int64_t q_stride) {
  if (n_q <= 0) return B200MS_OK;
  if (n_pages <= kTopkThreads) {  // small inputs (incl. every rerank of <= 1024 candidates): one counting pass
    if (score_dtype == B200MS_F32) {
      topk_small_kernel<float><<<n_q, kTopkThreads, 0, s>>>(static_cast<const float*>(group_scores), n_pages, ld, group_offsets_dev,
                                                           allow_mask, k, scale, id_base, id_map, top_scores, top_ids, top_counts,
                                                           mask_index, mask_stride, q_stride);
    } else {
      topk_small_kernel<int><<<n_q, kTopkThreads, 0, s>>>(static_cast<const int*>(group_scores), n_pages, ld, group_offsets_dev,
                                                         allow_mask, k, scale, id_base, id_map, top_scores, top_ids, top_counts,
                                                         mask_index, mask_stride, q_stride);
    }
    h->launches++;
    return check_cuda(h, cudaGetLastError(), "launch topk_small");
  }
  int n2 = 1;
  while (n2 < k) n2 <<= 1;
  const size_t smem = size_t(n2) * sizeof(uint64_t);
  // slices per query: enough CTAs to spread a big corpus over the SMs (one CTA sweeping 262144 pages took 0.87 ms),
  // bounded by the merge kernel's 8192-candidate capacity
  int64_t slices = n_pages / 8192;
  const int64_t cap = (2 * B200MS_MAX_K) / k;
  if (slices > cap) slices = cap;
  if (slices > 64) slices = 64;
  if (slices < 1) slices = 1;
  const int64_t slice_pages = (n_pages + slices - 1) / slices;
  uint32_t* part_keys = nullptr;
  int64_t* part_ids = nullptr;
  if (slices > 1) {
    if (int e = reserve(h, h->topk_keys, size_t(n_q) * slices * k * 4)) return e;
    if (int e = reserve(h, h->topk_ids, size_t(n_q) * slices * k * 8)) return e;
    part_keys = static_cast<uint32_t*>(h->topk_keys.p);
    part_ids = static_cast<int64_t*>(h->topk_ids.p);
  }
  const dim3 grid(n_q, unsigned(slices));
  if (score_dtype == B200MS_F32) {
    topk_kernel<float><<<grid, kTopkThreads, smem, s>>>(static_cast<const float*>(group_scores), n_pages, ld,
                                                       group_offsets_dev, allow_mask, k, scale, id_base, id_map, top_scores,
                                                       top_ids, top_counts, slice_pages, part_keys, part_ids, mask_index,
                                                       mask_stride, q_stride);
  } else {
    topk_kernel<int><<<grid, kTopkThreads, smem, s>>>(static_cast<const int*>(group_scores), n_pages, ld, group_offsets_dev,
                                                     allow_mask, k, scale, id_base, id_map, top_scores, top_ids, top_counts,
                                                     slice_pages, part_keys, part_ids, mask_index, mask_stride, q_stride);
  }
  h->launches++;
  if (int e = check_cuda(h, cudaGetLastError(), "launch topk")) return e;
  if (slices == 1) return B200MS_OK;
  const int m = int(slices) * k;
  return score_dtype == B200MS_F32
             ? launch_merge_impl<float>(h, nullptr, part_keys, part_ids, n_q, m, k, scale, top_scores, top_ids, top_counts, s,
                                        nullptr, 1, 0, 0, id_map)
             : launch_merge_impl<int>(h, nullptr, part_keys, part_ids, n_q, m, k, scale, top_scores, top_ids, top_counts, s,
                                      nullptr, 1, 0, 0, id_map);
}

int launch_merge_topk(b200ms_t* h, const float* cand_scores, const int64_t* cand_ids, int n_q, int m, int k,
                      float* top_scores, int64_t* top_ids, int32_t* top_counts, cudaStream_t s) {
  if (n_q <= 0) return B200MS_OK;
  return launch_merge_impl<float>(h, cand_scores, nullptr, cand_ids, n_q, m, k, 1.0f, top_scores, top_ids, top_counts, s);
}

int launch_merge_gathered(b200ms_t* h, const void* gathered, int world, int n_q, int k, float* top_scores, int64_t* top_ids,
                          int32_t* top_counts, cudaStream_t s) {
  if (n_q <= 0) return B200MS_OK;
  return launch_merge_impl<float>(h, nullptr, nullptr, nullptr, n_q, world * k, k, 1.0f, top_scores, top_ids, top_counts, s,
                                  static_cast<const uint8_t*>(gathered), k, int64_t(xchg_bytes(n_q, k)), int64_t(n_q) * k * 8);
}

}  // namespace bms
