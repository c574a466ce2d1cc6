// host_tier.cu -- candidate scoring of a corpus whose packed rows live in mapped pinned host memory (b200ms_set_corpus_host).
//
// Replaces the reference's storage model for multivectors: only the FDE vectors sit in the ANN index, and per query the store
// fetches the <= 75 candidate pages (load_multivector_from_storage, fast_multivector_store.py:545-548, :713-774).  Here the
// patch rows stay in host RAM and every rerank call copies only the pages its candidate lists name over PCIe:
//   1. dedup   the valid candidate ids of the whole call -> a page bitmap -> the unique pages in ascending id order
//              (prefix popcount over the bitmap words: deterministic, and no page crosses PCIe twice in one call)
//   2. plan    staging row offsets of the unique pages (their padded lengths, prefix-summed); ONE D2H of the unique count
//              and row total, the only synchronisation of the call
//   3. gather  per round, the pages whose staging offset falls in [r*W, (r+1)*W) are copied row-balanced with 16-byte loads
//              from the mapping into the HBM staging block, which then is a packed corpus of its own (page_start,
//              chunk_page and a TMA descriptor encoded once per (re)allocation of the block)
//   4. score   the unchanged scorers run on that block with the candidate slots remapped to it (slots of other rounds are
//              empty units); the top-k afterwards sees the original ids, so ids, ties and zero_pad_compat are those of HBM.
// A round holds at most host_stage_bytes of rows; W = budget - largest page + 32 rows, so a round's last page always fits.
#include "common.cuh"
#include "scan.cuh"

namespace bms {

constexpr int kGatherUnroll = 4;  // independent 16-byte PCIe reads in flight per thread

__device__ __forceinline__ int64_t lower_bound_i64(const int64_t* __restrict__ a, int64_t n, int64_t key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void ht_mark_kernel(const int64_t* __restrict__ ids, int64_t n_slots, int64_t n_pages, uint32_t* __restrict__ bitmap) {
  for (int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < n_slots; j += int64_t(gridDim.x) * blockDim.x) {
    const int64_t id = ids[j];
    if (id >= 0 && id < n_pages) atomicOr(bitmap + (id >> 5), 1u << (id & 31));
  }
}

__global__ void __launch_bounds__(kScanThreads)
ht_scan_words_kernel(const uint32_t* __restrict__ bitmap, int64_t n_words, int64_t* __restrict__ wpre) {
  block_scan([&](int64_t w) { return int64_t(__popc(bitmap[w])); }, n_words, wpre);
}

__global__ void ht_compact_kernel(const uint32_t* __restrict__ bitmap, int64_t n_words, const int64_t* __restrict__ wpre,
                                  int64_t* __restrict__ uniq) {
  for (int64_t w = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; w < n_words; w += int64_t(gridDim.x) * blockDim.x) {
    uint32_t b = bitmap[w];
    int64_t o = wpre[w];
    while (b) {
      uniq[o++] = w * 32 + (__ffs(b) - 1);
      b &= b - 1;
    }
  }
}

// staging offsets of the unique pages; hdr = {unique pages, staging rows}
__global__ void __launch_bounds__(kScanThreads)
ht_scan_rows_kernel(const int64_t* __restrict__ uniq, const int64_t* __restrict__ count, const int64_t* __restrict__ page_start,
                    int64_t* __restrict__ stage_off, int64_t* __restrict__ hdr) {
  const int64_t n = *count;
  block_scan([&](int64_t i) { const int64_t p = uniq[i]; return page_start[p + 1] - page_start[p]; }, n, stage_off);
  __syncthreads();
  if (threadIdx.x == 0) {
    hdr[0] = n;
    hdr[1] = stage_off[n];
  }
}

// Round r = unique pages [first, last) with stage_off in [r*W, (r+1)*W), local page li = i - first
struct Round {
  int64_t first, last, base;
};
__device__ __forceinline__ Round round_of(const int64_t* __restrict__ stage_off, int64_t n_uniq, int64_t W, int r) {
  Round x;
  x.first = lower_bound_i64(stage_off, n_uniq, int64_t(r) * W);
  x.last = lower_bound_i64(stage_off, n_uniq, int64_t(r + 1) * W);
  x.base = stage_off[x.first];
  return x;
}

// the staging block's page_start and chunk_page for round r
__global__ void ht_round_plan_kernel(const int64_t* __restrict__ stage_off, int64_t n_uniq, int64_t W, int r,
                                     int64_t* __restrict__ ps_local, int32_t* __restrict__ chunk_page_local) {
  const Round x = round_of(stage_off, n_uniq, W, r);
  for (int64_t li = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; li < x.last - x.first; li += int64_t(gridDim.x) * blockDim.x) {
    const int64_t i = x.first + li;
    const int64_t a = stage_off[i] - x.base, b = stage_off[i + 1] - x.base;
    ps_local[li] = a;
    if (i + 1 == x.last) ps_local[li + 1] = b;
    for (int64_t c = a / kGroup; c < b / kGroup; ++c) chunk_page_local[c] = int32_t(li);
  }
}

// slot j -> local page of round r, or -1 (invalid id, or a page of another round)
__global__ void ht_remap_kernel(const int64_t* __restrict__ ids, int64_t n_slots, int64_t n_pages, const uint32_t* __restrict__ bitmap,
                                const int64_t* __restrict__ wpre, const int64_t* __restrict__ stage_off, int64_t n_uniq, int64_t W,
                                int r, int64_t* __restrict__ remap) {
  const int64_t first = lower_bound_i64(stage_off, n_uniq, int64_t(r) * W);
  for (int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < n_slots; j += int64_t(gridDim.x) * blockDim.x) {
    const int64_t id = ids[j];
    int64_t out = -1;
    if (id >= 0 && id < n_pages) {
      const int64_t w = id >> 5;
      const int64_t i = wpre[w] + __popc(bitmap[w] & ((1u << (id & 31)) - 1u));
      if (stage_off[i] / W == r) out = i - first;
    }
    remap[j] = out;
  }
}

// Row-balanced copy of round r's pages from the mapped host rows into the staging block: 16-byte pieces (2^piece_shift per
// row), kGatherUnroll independent loads per thread before their stores.
__global__ void __launch_bounds__(256)
ht_gather_kernel(const uint4* __restrict__ src, int piece_shift, const int64_t* __restrict__ page_start,
                 const int64_t* __restrict__ uniq, const int64_t* __restrict__ stage_off, int64_t n_uniq, int64_t W, int r,
                 const int64_t* __restrict__ ps_local, const int32_t* __restrict__ chunk_page_local, uint4* __restrict__ dst) {
  const Round x = round_of(stage_off, n_uniq, W, r);
  const int64_t total = (x.last > x.first ? stage_off[x.last] - x.base : 0) << piece_shift;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  const int64_t mask = (int64_t(1) << piece_shift) - 1;
  for (int64_t p0 = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; p0 < total; p0 += stride * kGatherUnroll) {
    uint4 v[kGatherUnroll];
#pragma unroll
    for (int k = 0; k < kGatherUnroll; ++k) {
      const int64_t p = p0 + k * stride;
      if (p < total) {
        const int64_t row = p >> piece_shift;
        const int32_t li = chunk_page_local[row / kGroup];
        const int64_t srow = page_start[uniq[x.first + li]] + (row - ps_local[li]);
        v[k] = src[(srow << piece_shift) + (p & mask)];
      }
    }
#pragma unroll
    for (int k = 0; k < kGatherUnroll; ++k) {
      const int64_t p = p0 + k * stride;
      if (p < total) dst[p] = v[k];
    }
  }
}

// 1-bit rounds of a rerank: merge one round's own slots (score_host_tier)
__global__ void ht_merge_round_kernel(int32_t* __restrict__ dst, const int32_t* __restrict__ src, const int64_t* __restrict__ remap,
                                      int64_t n_slots, int64_t rows, int64_t ld) {
  for (int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; idx < rows * n_slots; idx += int64_t(gridDim.x) * blockDim.x) {
    const int64_t g = idx / n_slots, j = idx - g * n_slots;
    if (remap[j] >= 0) dst[g * ld + j] = src[g * ld + j];
  }
}

// round geometry: capacity cap rows (the budget, at least the largest page), pages starting in each W-row window
static void round_geometry(const b200ms_t* h, int64_t* cap, int64_t* W) {
  const Corpus& c = h->corpus;
  int64_t cp = (h->host_stage_bytes / b200ms_row_bytes(c.dtype)) & ~int64_t(kGroup - 1);
  if (cp < c.max_page_rows) cp = c.max_page_rows;
  *cap = cp;
  *W = cp - c.max_page_rows + kGroup;
}

int host_tier_rounds(const b200ms_t* h, int64_t rows) {
  int64_t cap = 0, W = 0;
  round_geometry(h, &cap, &W);
  return int((rows + W - 1) / W);
}

int gather_host_tier(b200ms_t* h, const int64_t* ids, int64_t n_slots, cudaStream_t s,
                     int (*round_fn)(b200ms_t*, const CorpusView&, const int64_t* remap, int r, int rounds, void* ctx),
                     void* ctx) {
  const Corpus& c = h->corpus;
  const int64_t rb = b200ms_row_bytes(c.dtype);
  const int64_t n_words = (c.n_pages + 31) / 32;
  h->ht_unique = h->ht_bytes = 0;
  h->ht_rounds = 0;
  if (int e = reserve(h, h->ht_bitmap, size_t(n_words > 0 ? n_words : 1) * 4)) return e;
  if (int e = reserve(h, h->ht_wpre, size_t(n_words + 1) * 8)) return e;
  if (int e = reserve(h, h->ht_uniq, size_t(n_slots > 0 ? n_slots : 1) * 8)) return e;
  if (int e = reserve(h, h->ht_stage_off, size_t(n_slots + 1) * 8)) return e;
  if (int e = reserve(h, h->ht_hdr, 16)) return e;
  if (int e = reserve(h, h->ht_remap, size_t(n_slots > 0 ? n_slots : 1) * 8)) return e;
  uint32_t* bitmap = static_cast<uint32_t*>(h->ht_bitmap.p);
  int64_t* wpre = static_cast<int64_t*>(h->ht_wpre.p);
  int64_t* uniq = static_cast<int64_t*>(h->ht_uniq.p);
  int64_t* stage_off = static_cast<int64_t*>(h->ht_stage_off.p);
  int64_t* remap = static_cast<int64_t*>(h->ht_remap.p);
  const int64_t* ps = static_cast<const int64_t*>(h->page_start.p);
  // 1-2: dedup + plan
  if (int e = check_cuda(h, cudaMemsetAsync(bitmap, 0, size_t(n_words > 0 ? n_words : 1) * 4, s), "host tier: memset")) return e;
  ht_mark_kernel<<<grid_stride_blocks(h, n_slots, 256, 8), 256, 0, s>>>(ids, n_slots, c.n_pages, bitmap);
  ht_scan_words_kernel<<<1, kScanThreads, 0, s>>>(bitmap, n_words, wpre);
  ht_compact_kernel<<<grid_stride_blocks(h, n_words, 256, 8), 256, 0, s>>>(bitmap, n_words, wpre, uniq);
  ht_scan_rows_kernel<<<1, kScanThreads, 0, s>>>(uniq, wpre + n_words, ps, stage_off, static_cast<int64_t*>(h->ht_hdr.p));
  h->launches += 4;
  if (int e = check_cuda(h, cudaGetLastError(), "launch host-tier dedup")) return e;
  int64_t hdr[2] = {0, 0};
  if (int e = check_cuda(h, cudaMemcpyAsync(hdr, h->ht_hdr.p, 16, cudaMemcpyDeviceToHost, s), "host tier: D2H plan")) return e;
  if (int e = check_cuda(h, cudaStreamSynchronize(s), "host tier: stream sync")) return e;
  const int64_t n_uniq = hdr[0], rows = hdr[1];
  h->ht_unique = n_uniq;
  h->ht_bytes = rows * rb;
  if (rows == 0) return B200MS_OK;  // no valid candidate, or only empty pages: nothing to gather
  int64_t cap = 0, W = 0;
  round_geometry(h, &cap, &W);
  const int rounds = int((rows + W - 1) / W);
  const int64_t stage_rows = rounds == 1 ? rows : cap;
  if (int e = reserve(h, h->ht_stage, size_t(stage_rows) * size_t(rb) + 1024)) return e;
  const uintptr_t raw = reinterpret_cast<uintptr_t>(h->ht_stage.p);
  void* stage = reinterpret_cast<void*>((raw + 1023) & ~uintptr_t(1023));
  const int64_t rows_cap = int64_t(h->ht_stage.cap - (reinterpret_cast<uintptr_t>(stage) - raw)) / rb;
  const bool b1 = c.dtype == B200MS_B1;
  if (!b1 && (h->ht_tmap_base != stage || h->ht_tmap_dtype != c.dtype || h->ht_tmap_rows != rows_cap)) {
    if (int e = make_tmap_rows(h, &h->ht_tmap, stage, c.dtype, rows_cap, kTileN)) return e;
    h->ht_tmap_base = stage;
    h->ht_tmap_dtype = c.dtype;
    h->ht_tmap_rows = rows_cap;
  }
  if (int e = reserve(h, h->ht_ps, size_t(n_uniq + 1) * 8)) return e;
  if (int e = reserve(h, h->ht_chunk_page, size_t(stage_rows / kGroup > 0 ? stage_rows / kGroup : 1) * 4)) return e;
  while (h->ht_ev.size() < size_t(2 * rounds)) {
    cudaEvent_t ev = nullptr;
    if (int e = check_cuda(h, cudaEventCreate(&ev), "host tier: cudaEventCreate")) return e;
    h->ht_ev.push_back(ev);
  }
  CorpusView v;
  v.rows = stage;
  v.dtype = c.dtype;
  v.n_pages = n_uniq;
  v.n_rows = rows_cap;
  v.tmap = b1 ? nullptr : &h->ht_tmap;
  v.chunk_page = static_cast<const int32_t*>(h->ht_chunk_page.p);
  v.page_start = static_cast<const int64_t*>(h->ht_ps.p);
  const int piece_shift = rb == 256 ? 4 : rb == 128 ? 3 : 0;
  for (int r = 0; r < rounds; ++r) {
    ht_round_plan_kernel<<<grid_stride_blocks(h, n_uniq, 256, 8), 256, 0, s>>>(
        stage_off, n_uniq, W, r, static_cast<int64_t*>(h->ht_ps.p), static_cast<int32_t*>(h->ht_chunk_page.p));
    ht_remap_kernel<<<grid_stride_blocks(h, n_slots, 256, 8), 256, 0, s>>>(
        ids, n_slots, c.n_pages, bitmap, wpre, stage_off, n_uniq, W, r, remap);
    if (int e = check_cuda(h, cudaEventRecord(h->ht_ev[2 * r], s), "host tier: event record")) return e;
    ht_gather_kernel<<<h->num_sms * 8, 256, 0, s>>>(static_cast<const uint4*>(c.rows), piece_shift, ps, uniq, stage_off, n_uniq,
                                                   W, r, v.page_start, v.chunk_page, static_cast<uint4*>(stage));
    if (int e = check_cuda(h, cudaEventRecord(h->ht_ev[2 * r + 1], s), "host tier: event record")) return e;
    h->launches += 3;
    if (int e = check_cuda(h, cudaGetLastError(), "launch host-tier gather")) return e;
    h->ht_rounds = r + 1;
    if (int e = round_fn(h, v, remap, r, rounds, ctx)) return e;
  }
  return B200MS_OK;
}

int score_host_tier(b200ms_t* h, const CandSpec& cs, int n_q, int64_t gp, int64_t ld, void* group_scores, cudaStream_t s,
                    int (*score_round)(b200ms_t*, const CorpusView&, const int64_t* unit_ids, void* scores, bool fill,
                                       void* ctx),
                    void* ctx) {
  const int64_t n_slots = cs.n_slots(n_q);
  struct Ctx {
    int64_t n_slots, gp, ld;
    void* group_scores;
    cudaStream_t s;
    int (*score_round)(b200ms_t*, const CorpusView&, const int64_t*, void*, bool, void*);
    void* ctx;
  } x{n_slots, gp, ld, group_scores, s, score_round, ctx};
  auto round = [](b200ms_t* hh, const CorpusView& v, const int64_t* remap, int r, int rounds, void* p) {
    const Ctx& x = *static_cast<const Ctx*>(p);
    if (v.dtype != B200MS_B1 || rounds == 1) return x.score_round(hh, v, remap, x.group_scores, r == 0, x.ctx);
    // 1-bit rounds: the POPC rerank kernel writes 0 for every slot outside its round, so each round scores into scratch and
    // only its own slots are copied over
    if (r == 0) {
      if (int e = reserve(hh, hh->ht_scores, size_t(x.gp) * size_t(x.ld) * 4)) return e;
      if (int e = check_cuda(hh, cudaMemsetAsync(x.group_scores, 0, size_t(x.gp) * size_t(x.ld) * 4, x.s), "host tier: memset scores"))
        return e;
    }
    if (int e = x.score_round(hh, v, remap, hh->ht_scores.p, true, x.ctx)) return e;
    ht_merge_round_kernel<<<grid_stride_blocks(hh, x.gp * x.n_slots, 256, 8), 256, 0, x.s>>>(
        static_cast<int32_t*>(x.group_scores), static_cast<const int32_t*>(hh->ht_scores.p), remap, x.n_slots, x.gp, x.ld);
    hh->launches++;
    return check_cuda(hh, cudaGetLastError(), "launch host-tier merge");
  };
  if (int e = gather_host_tier(h, cs.ids, n_slots, s, round, &x)) return e;
  if (h->ht_rounds == 0)  // no valid candidate, or only empty pages: every score is 0, what the scorers leave for them
    return check_cuda(h, cudaMemsetAsync(group_scores, 0, size_t(gp) * size_t(ld) * 4, s), "host tier: memset scores");
  return B200MS_OK;
}

}  // namespace bms
