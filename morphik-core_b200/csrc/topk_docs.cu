// topk_docs.cu -- the top k DOCUMENTS instead of the top k pages (b200ms_topk_docs, b200ms_search_docs_device,
// b200ms_rerank_docs_batch_device).  The result is a pure function of the flat ranking L of b200ms_topk: documents in the
// order of their first page in L, each with its first per_doc pages in L.
//
// Every item (a page of a full scan, a slot of a candidate list) gets the 64-bit key (page_key's 32-bit key << 32) |
// (0xffffffff - column); its order is L's order (score DESC, column ASC).  Then:
//   1. best[q, d]  = max key over q's eligible items of document d (warp-aggregated atomicMax);
//   2. a page mask with one bit per document, at its best item, and the flat top-k (launch_topk: radix select, slicing,
//      merge) over it -- the k winning documents in the order of their best pages, i.e. of their first page in L;
//   3. per_doc > 1: per_doc - 1 more passes, pass t taking for every winning document the largest key strictly below its
//      pick t-1 (a candidate slot whose page is already picked is skipped: a page counts once, at its earliest slot);
//   4. one kernel writes the outputs.
// Traffic per pass: one read of the query's group-score row and of page_doc, next to a scan of milliseconds.
#include <math_constants.h>

#include "common.cuh"
#include "topk_keys.cuh"

namespace bms {

constexpr int kDocThreads = 256;

// What the grouping kernels read.  Query q owns items j in [0, row), row a multiple of 32:
//   full scan (cand == NULL): item j < n_items is page j, score column j, eligible when its allow bit is set;
//   candidate mode: item j < n_items is slot j of q's list, score column q*row + j, page cand[q*row + j].
// An item is eligible when its page is in [0, n_pages) and page_doc[page] in [0, n_docs).
template <typename T>
struct DocView {
  const T* gs;
  int64_t ld;
  const int32_t* goff;
  const uint32_t* allow;
  const int32_t* mask_index;
  int64_t mask_stride;
  const int64_t* cand;
  int64_t n_items, row, n_pages;
  const int32_t* page_doc;
  int64_t n_docs;
};

template <typename T>
__device__ __forceinline__ bool doc_item(const DocView<T>& v, int q, int64_t j, int64_t* page, int64_t* doc, uint64_t* key) {
  if (j >= v.n_items) return false;
  const int64_t col = v.cand ? int64_t(q) * v.row + j : j;
  const int64_t pg = v.cand ? __ldg(v.cand + col) : j;
  if (pg < 0 || pg >= v.n_pages) return false;
  const uint32_t* allow = v.allow;
  if (allow && v.mask_index) {
    const int mi = __ldg(v.mask_index + q);
    allow = mi >= 0 ? allow + int64_t(mi) * v.mask_stride : nullptr;
  }
  if (allow && !((__ldg(allow + (pg >> 5)) >> (pg & 31)) & 1u)) return false;
  const int d = __ldg(v.page_doc + pg);
  if (d < 0 || d >= v.n_docs) return false;
  uint32_t k32;
  page_key(v.gs, v.ld, __ldg(v.goff + q), __ldg(v.goff + q + 1), nullptr, col, &k32);
  *page = pg;
  *doc = d;
  *key = (uint64_t(k32) << 32) | uint64_t(0xffffffffu - uint32_t(col));
  return true;
}

__device__ __forceinline__ int64_t col_of_key(uint64_t key) { return int64_t(0xffffffffu - uint32_t(key)); }

// atomicMax(dst, key) with one atomic per distinct dst in the warp (dst == NULL: no update; every lane calls).  Pages of
// one document are mostly contiguous, so a warp mostly holds one or two documents.  The plain read first skips the atomic
// once the word holds a larger key: in a one-document corpus every warp of a query targets the same word.
__device__ __forceinline__ void warp_max_u64(unsigned long long* dst, uint64_t key) {
  const unsigned peers = __match_any_sync(0xffffffffu, reinterpret_cast<unsigned long long>(dst));
  const uint32_t hi = __reduce_max_sync(peers, uint32_t(key >> 32));
  const uint32_t lo = __reduce_max_sync(peers, uint32_t(key >> 32) == hi ? uint32_t(key) : 0u);
  if (dst && int(threadIdx.x & 31) == __ffs(peers) - 1) {
    const unsigned long long m = (uint64_t(hi) << 32) | lo;
    if (m > *reinterpret_cast<volatile unsigned long long*>(dst)) atomicMax(dst, m);
  }
}

// grid = (chunks of the row, queries): whole warps walk whole 32-item words, so the warp-wide steps see all 32 lanes
#define DOC_ITEMS_LOOP(v, n_q)                                                                                      \
  for (int q = blockIdx.y; q < (n_q); q += gridDim.y)                                                               \
    for (int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < (v).row; j += int64_t(gridDim.x) * blockDim.x)

// 1. best[q, d] = max key over q's eligible items of document d (best zeroed by the caller)
template <typename T>
__global__ void __launch_bounds__(kDocThreads) docs_best_kernel(DocView<T> v, int n_q, unsigned long long* __restrict__ best) {
  DOC_ITEMS_LOOP(v, n_q) {
    int64_t page = 0, d = 0;
    uint64_t key = 0;
    const bool ok = doc_item(v, q, j, &page, &d, &key);
    warp_max_u64(ok ? best + int64_t(q) * v.n_docs + d : nullptr, key);
  }
}

// 2. bit j of mask row q = item j is its document's best; every word of the [n_q, row/32] mask is written.  mask_index
// (full scan): row q for query q, so that launch_topk reads the mask as a per-query allow mask.
template <typename T>
__global__ void __launch_bounds__(kDocThreads) docs_mark_kernel(DocView<T> v, int n_q, const unsigned long long* __restrict__ best,
                                                                uint32_t* __restrict__ mask, int32_t* __restrict__ mask_index) {
  DOC_ITEMS_LOOP(v, n_q) {
    int64_t page = 0, d = 0;
    uint64_t key = 0;
    const bool win = doc_item(v, q, j, &page, &d, &key) && best[int64_t(q) * v.n_docs + d] == key;
    const uint32_t bal = __ballot_sync(0xffffffffu, win);
    if ((threadIdx.x & 31) == 0) mask[int64_t(q) * (v.row / 32) + (j >> 5)] = bal;
    if (mask_index && j == 0) mask_index[q] = q;
  }
}

// 3a. the winners of query q, in rank order (top_ids: their columns): pick[q, i, 0] = the key of document i's best item;
// rank[q, d] = i (rank pre-filled with -1; NULL when per_doc == 1)
template <typename T>
__global__ void __launch_bounds__(kDocThreads) docs_rank_kernel(DocView<T> v, int k, int per_doc, const int64_t* __restrict__ top_ids,
                                                                const int32_t* __restrict__ top_counts, int32_t* __restrict__ rank,
                                                                unsigned long long* __restrict__ pick) {
  const int q = blockIdx.x;
  const int cnt = top_counts[q];
  const int g0 = __ldg(v.goff + q), g1 = __ldg(v.goff + q + 1);
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
    const int64_t col = top_ids[int64_t(q) * k + i];
    uint32_t k32;
    page_key(v.gs, v.ld, g0, g1, nullptr, col, &k32);
    pick[(int64_t(q) * k + i) * per_doc] = (uint64_t(k32) << 32) | uint64_t(0xffffffffu - uint32_t(col));
    if (rank) rank[int64_t(q) * v.n_docs + __ldg(v.page_doc + (v.cand ? __ldg(v.cand + col) : col))] = i;
  }
}

// 3b. pick[q, r, t] = the largest key of winning document r's items strictly below pick[q, r, t-1] (pick zeroed for t >= 1;
// 0 = none, as no item's key is 0)
template <typename T>
__global__ void __launch_bounds__(kDocThreads) docs_next_kernel(DocView<T> v, int n_q, int k, int per_doc, int t,
                                                                const int32_t* __restrict__ rank, unsigned long long* __restrict__ pick) {
  DOC_ITEMS_LOOP(v, n_q) {
    int64_t page = 0, d = 0;
    uint64_t key = 0;
    unsigned long long* dst = nullptr;
    if (doc_item(v, q, j, &page, &d, &key)) {
      const int r = rank[int64_t(q) * v.n_docs + d];
      if (r >= 0) {
        unsigned long long* mine = pick + (int64_t(q) * k + r) * per_doc;
        if (key < mine[t - 1]) {
          bool dup = false;
          if (v.cand)
            for (int u = 0; u < t; ++u) dup |= __ldg(v.cand + col_of_key(mine[u])) == page;
          if (!dup) dst = mine + t;
        }
      }
    }
    warp_max_u64(dst, key);
  }
}

// 4. outputs: [n_q, k, per_doc] scores / ids (unused: -inf / -1), [n_q, k] pages per document, [n_q] documents
template <typename T>
__global__ void __launch_bounds__(kDocThreads) docs_out_kernel(const int64_t* __restrict__ cand, const int32_t* __restrict__ top_counts,
                                                               const unsigned long long* __restrict__ pick, int k, int per_doc,
                                                               float scale, int64_t id_base, float* __restrict__ out_scores,
                                                               int64_t* __restrict__ out_ids, int32_t* __restrict__ page_counts,
                                                               int32_t* __restrict__ doc_counts) {
  const int q = blockIdx.x;
  const int cnt = top_counts ? top_counts[q] : 0;
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    int n = 0;
    for (int t = 0; t < per_doc; ++t) {
      const int64_t o = (int64_t(q) * k + i) * per_doc + t;
      const uint64_t w = i < cnt ? pick[o] : 0;
      const int64_t col = col_of_key(w);
      out_scores[o] = w ? score_of_key(uint32_t(w >> 32), T(0)) * scale : -CUDART_INF_F;
      out_ids[o] = w ? (cand ? __ldg(cand + col) : col + id_base) : int64_t(-1);
      n += w != 0;
    }
    page_counts[int64_t(q) * k + i] = n;
  }
  if (threadIdx.x == 0) doc_counts[q] = cnt;
}

template <typename T>
static int topk_docs_impl(b200ms_t* h, const T* gs, int sdt, int64_t n_items, int64_t ld, const int32_t* goff, int n_q,
                          const uint32_t* allow, const int32_t* mask_index, const int64_t* cand, int64_t q_stride,
                          int64_t n_pages, const DocSpec& d, int k, float scale, int64_t id_base, cudaStream_t s) {
  const int64_t row = cand ? q_stride : (n_items + 31) & ~int64_t(31);
  const DocView<T> v{gs, ld, goff, cand ? nullptr : allow, cand ? nullptr : mask_index, (n_pages + 31) / 32, cand, n_items, row,
                     n_pages, d.page_doc, d.n_docs};
  const int per_doc = d.per_doc;
  const int32_t* counts = nullptr;
  unsigned long long* pick = nullptr;
  if (n_items > 0 && d.n_docs > 0) {
    const size_t nk = size_t(n_q) * size_t(k);
    if (int e = reserve(h, h->docs_best, size_t(n_q) * size_t(d.n_docs) * 8)) return e;
    if (int e = reserve(h, h->docs_mask, size_t(n_q) * size_t(row / 32 + 1) * 4)) return e;
    if (int e = reserve(h, h->docs_top, nk * 12 + size_t(n_q) * 4)) return e;
    if (int e = reserve(h, h->docs_pick, nk * size_t(per_doc) * 8)) return e;
    auto* best = static_cast<unsigned long long*>(h->docs_best.p);
    auto* mask = static_cast<uint32_t*>(h->docs_mask.p);
    int32_t* iota = cand ? nullptr : reinterpret_cast<int32_t*>(mask + size_t(n_q) * size_t(row / 32));
    int64_t* top_ids = static_cast<int64_t*>(h->docs_top.p);
    float* top_scores = reinterpret_cast<float*>(top_ids + nk);
    int32_t* top_counts = reinterpret_cast<int32_t*>(top_scores + nk);
    pick = static_cast<unsigned long long*>(h->docs_pick.p);
    counts = top_counts;
    const int gy = n_q < 65535 ? n_q : 65535;
    int64_t gx = (row + kDocThreads - 1) / kDocThreads;
    const int64_t cap = (int64_t(h->num_sms) * 8 + gy - 1) / gy;
    if (gx > cap) gx = cap;
    const dim3 grid{unsigned(gx), unsigned(gy)};
    if (int e = check_cuda(h, cudaMemsetAsync(best, 0, size_t(n_q) * size_t(d.n_docs) * 8, s), "topk_docs: memset")) return e;
    docs_best_kernel<T><<<grid, kDocThreads, 0, s>>>(v, n_q, best);
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch docs_best")) return e;
    docs_mark_kernel<T><<<grid, kDocThreads, 0, s>>>(v, n_q, best, mask, iota);
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch docs_mark")) return e;
    if (int e = cand ? launch_topk(h, gs, sdt, n_items, ld, goff, n_q, mask, k, scale, 0, nullptr, top_scores, top_ids, top_counts,
                                   s, nullptr, 0, row)
                     : launch_topk(h, gs, sdt, n_items, ld, goff, n_q, mask, k, scale, 0, nullptr, top_scores, top_ids, top_counts,
                                   s, iota, row / 32))
      return e;
    int32_t* rank = nullptr;
    if (per_doc > 1) {  // best is done with: its words hold the rank table from here on
      rank = reinterpret_cast<int32_t*>(best);
      if (int e = check_cuda(h, cudaMemsetAsync(rank, 0xff, size_t(n_q) * size_t(d.n_docs) * 4, s), "topk_docs: memset")) return e;
      if (int e = check_cuda(h, cudaMemsetAsync(pick, 0, nk * size_t(per_doc) * 8, s), "topk_docs: memset")) return e;
    }
    docs_rank_kernel<T><<<n_q, kDocThreads, 0, s>>>(v, k, per_doc, top_ids, top_counts, rank, pick);
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch docs_rank")) return e;
    for (int t = 1; t < per_doc; ++t) {
      docs_next_kernel<T><<<grid, kDocThreads, 0, s>>>(v, n_q, k, per_doc, t, rank, pick);
      h->launches++;
      if (int e = check_cuda(h, cudaGetLastError(), "launch docs_next")) return e;
    }
  }
  docs_out_kernel<T><<<n_q, kDocThreads, 0, s>>>(cand, counts, pick, k, per_doc, scale, id_base, d.scores, d.ids, d.page_counts,
                                                 d.doc_counts);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch docs_out");
}

int launch_topk_docs(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_items, int64_t ld,
                     const int32_t* group_offsets_dev, int n_q, const uint32_t* allow, const int32_t* mask_index,
                     const int64_t* cand, int64_t q_stride, int64_t n_pages, const DocSpec& d, int k, float scale,
                     int64_t id_base, cudaStream_t s) {
  if (n_q <= 0) return B200MS_OK;
  return score_dtype == B200MS_F32
             ? topk_docs_impl(h, static_cast<const float*>(group_scores), score_dtype, n_items, ld, group_offsets_dev, n_q, allow,
                              mask_index, cand, q_stride, n_pages, d, k, scale, id_base, s)
             : topk_docs_impl(h, static_cast<const int*>(group_scores), score_dtype, n_items, ld, group_offsets_dev, n_q, allow,
                              mask_index, cand, q_stride, n_pages, d, k, scale, id_base, s);
}

}  // namespace bms
