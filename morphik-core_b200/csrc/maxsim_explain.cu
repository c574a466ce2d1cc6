// maxsim_explain.cu -- per-token MaxSim breakdown of chosen pages (b200ms_explain_device): for every query token the best
// patch row of the page, its similarity (the token's share of the page score) and, when asked, the whole token x row map.
//
// The search keeps only sum_t max_r sim(q_t, d_r); this recomputes the same products for the pages a caller names (normally
// the top-k just returned) and keeps what the search discards.  So that the explanation adds up to the score the caller was
// shown, the dense dtypes run on the scan's own tensor-core instructions with the same operand kinds and the same K order
// (mma_tile.cuh): bf16 k16 / fp32, s8 k32 / int32, e4m3 widened to f16 k16 / fp32.  One token x row product is therefore the
// value the scan took its max over, bit for bit; only the sum over tokens is done by the caller.
//
// Work item = (query q, candidate slot j, 64-token tile of q).  Dense dtypes: one warpgroup per item loads the 64 query rows
// (the packed rows of b200ms_search_device) as the wgmma A block, then walks the page in 128-row tiles (B, plain 16-byte
// loads of the next tile in flight while the current one is on the tensor pipe), and per tile runs one m64n128 chain.  The
// epilogue writes the map tile and keeps a running (max, lowest row) per token; the four lanes of a quad are combined once at
// the end.  1-bit corpora: one warp per token, 128 - popc(q ^ d) per row, exact.
#include <cstring>

#include "common.cuh"
#include "mma_tile.cuh"
#include "ptx.cuh"
#include "row_tiles.cuh"

namespace bms {

constexpr int kExplainTokens = kABlockRows;       // query tokens per work item (one wgmma M block)
constexpr int kExplainThreads = kRowTileThreads;  // one warpgroup
constexpr int kExplainB1Threads = 256;            // 1-bit kernel: 8 warps, one token each at a time

struct ExplainArgs {
  const void* q = nullptr;            // packed query rows of the corpus dtype (b200ms_pack_queries layout)
  int64_t q_rows = 0;                 // rows the packed block holds (reads past it are zero)
  const int64_t* ss = nullptr;        // [n_q + 1] true-row offsets of the queries (lengths)
  const int32_t* goff = nullptr;      // [n_q + 1] 32-row group offsets into the packed block
  int n_q = 0, n_cand = 0, t_max = 0, n_ttiles = 0;
  const int64_t* ids = nullptr;       // [n_q, n_cand] corpus page ids (-1 / out of range = unused slot)
  const int64_t* unit_ids = nullptr;  // the same slots as pages of the view's rows; -1 = not in this view (host-tier round)
  int64_t n_pages = 0;                // corpus pages
  const int32_t* page_len = nullptr;  // [n_pages] TRUE row counts, by corpus id
  const void* rows = nullptr;         // the view's packed rows
  const int64_t* page_start = nullptr;  // the view's first padded row per page
  float scale = 1.f;
  float* token_scores = nullptr;      // [n_q, n_cand, t_max]
  int32_t* best_rows = nullptr;       // [n_q, n_cand, t_max]
  float* sim_map = nullptr;           // [n_q, n_cand, t_max, map_rows] or NULL
  int64_t map_rows = 0;
};

// What one work item does: fill (unused slot, empty page, tokens past the query), skip (page gathered in another host-tier
// round: that round writes it) or compute rows [row0, row0 + len) of the view.
struct ExplainItem {
  int64_t slot;
  int q, t0, t1, qlen, len;  // tokens [t0, t1) of the output, t1 <= t_max
  int64_t row0;
  bool compute, skip;
};

__device__ __forceinline__ ExplainItem explain_item(const ExplainArgs& a, int slot, int tt) {
  ExplainItem x;
  x.slot = slot;
  x.q = slot / a.n_cand;
  x.t0 = tt * kExplainTokens;
  x.t1 = min(x.t0 + kExplainTokens, a.t_max);
  x.qlen = int(__ldg(a.ss + x.q + 1) - __ldg(a.ss + x.q));
  const int64_t pid = __ldg(a.ids + x.slot);
  x.len = (pid >= 0 && pid < a.n_pages) ? __ldg(a.page_len + pid) : 0;
  x.compute = x.len > 0 && x.t0 < x.qlen;
  x.skip = false;
  x.row0 = 0;
  if (x.compute) {
    const int64_t vid = __ldg(a.unit_ids + x.slot);
    if (vid < 0) {
      x.skip = true;
      x.compute = false;
    } else {
      x.row0 = __ldg(a.page_start + vid);
    }
  }
  return x;
}

__device__ __forceinline__ int64_t map_index(const ExplainArgs& a, int64_t slot, int t, int64_t r) {
  return (slot * a.t_max + t) * a.map_rows + r;
}

// tokens [t0, t1) of a slot: score 0, best row -1, map rows [r0, map_rows) -inf (all threads of the block)
__device__ __forceinline__ void explain_fill(const ExplainArgs& a, int64_t slot, int t0, int t1, int64_t r0, bool scores) {
  if (scores)
    for (int t = t0 + int(threadIdx.x); t < t1; t += blockDim.x) {
      a.token_scores[slot * a.t_max + t] = 0.f;
      a.best_rows[slot * a.t_max + t] = -1;
    }
  if (!a.sim_map) return;
  for (int t = t0; t < t1; ++t)
    for (int64_t r = r0 + threadIdx.x; r < a.map_rows; r += blockDim.x)
      a.sim_map[map_index(a, slot, t, r)] = -__int_as_float(0x7f800000);
}

// (v, i) beats (bv, bi): higher value, or the same value (or both NaN) at a lower row; a NaN loses to any number -- the max
// is the fmaxf reduction the scan does, the row the lowest one holding it.  i < 0: nothing.
template <typename Acc>
__device__ __forceinline__ bool beats(Acc v, int i, Acc bv, int bi) {
  if (i < 0) return false;
  if (bi < 0) return true;
  if constexpr (std::is_same<Acc, float>::value) {
    const bool vn = v != v, bn = bv != bv;
    if (vn != bn) return bn;
    if (!vn && v != bv) return v > bv;
  } else {
    if (v != bv) return v > bv;
  }
  return i < bi;
}

template <typename Acc>
__device__ __forceinline__ void shfl_best(Acc& bv, int& bi, int lane_mask) {
  const Acc ov = __shfl_xor_sync(0xffffffffu, bv, lane_mask);
  const int oi = __shfl_xor_sync(0xffffffffu, bi, lane_mask);
  if (beats(ov, oi, bv, bi)) {
    bv = ov;
    bi = oi;
  }
}

__device__ __forceinline__ void write_token(const ExplainArgs& a, const ExplainItem& x, int t, float v, int bi) {
  const bool ok = t < x.qlen && bi >= 0;
  a.token_scores[x.slot * a.t_max + t] = ok ? v : 0.f;
  a.best_rows[x.slot * a.t_max + t] = ok ? bi : -1;
}

// ------------------------------------------------------------------ dense dtypes on wgmma
// KIND 0 bf16, 1 int8, 2 fp8 e4m3 (widened to f16 in shared memory on both operands); the tile loop is row_tiles.cuh's
template <int KIND>
__global__ void __launch_bounds__(kExplainThreads)
maxsim_explain_wgmma(const __grid_constant__ ExplainArgs a) {
  using K = Kind<KIND>;
  using Acc = typename K::Acc;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t b_addr = smem_u32(smem);                   // [kPanels][128 rows x 128 B]
  const uint32_t a_addr = b_addr + K::kPanels * kSubtileBytes;  // [kPanels][64 rows x 128 B]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint4* qrows = static_cast<const uint4*>(a.q);
  const uint4* prows = static_cast<const uint4*>(a.rows);

  const int n_slots = a.n_q * a.n_cand;
  for (int tt = blockIdx.y; tt < a.n_ttiles; tt += gridDim.y)
  for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
    const ExplainItem x = explain_item(a, slot, tt);
    if (x.skip) continue;
    if (!x.compute) {
      explain_fill(a, x.slot, x.t0, x.t1, 0, true);
      continue;
    }
    const int padded = (x.len + kGroup - 1) & ~(kGroup - 1);
    const int n_tiles = (padded + kTileN - 1) / kTileN;
    // per token (accumulator rows m0 = 16 warp + lane/4 and m0 + 8): this lane's running max and lowest row
    Acc bv0 = Acc(0), bv1 = Acc(0);
    int bi0 = -1, bi1 = -1;
    const int m0 = 16 * warp + (lane >> 2);
    const int tok0 = x.t0 + m0, tok1 = tok0 + 8;
    const int64_t qrow0 = int64_t(__ldg(a.goff + x.q)) * kGroup + x.t0;
    rows_vs_page_tiles<KIND>(
        a_addr, b_addr, prows, x.row0, padded, [&] { load_a_block<KIND>(a_addr, qrows, qrow0, a.q_rows); },
        [&](const Acc(&d)[64], int n) {
          const int rbase = n * kTileN + 2 * (lane & 3);
#pragma unroll
          for (int jb = 0; jb < 16; ++jb) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int row = rbase + 8 * jb + e;
              if (row < x.len) {
                if (beats(d[4 * jb + e], row, bv0, bi0)) {
                  bv0 = d[4 * jb + e];
                  bi0 = row;
                }
                if (beats(d[4 * jb + 2 + e], row, bv1, bi1)) {
                  bv1 = d[4 * jb + 2 + e];
                  bi1 = row;
                }
              }
            }
          }
          if (a.sim_map) {
            const float ninf = -__int_as_float(0x7f800000);
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2) {
              const int t = h2 ? tok1 : tok0;
              if (t >= x.t1) continue;
              const bool live = t < x.qlen;
#pragma unroll
              for (int jb = 0; jb < 16; ++jb) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int row = rbase + 8 * jb + e;
                  if (row < a.map_rows)
                    a.sim_map[map_index(a, x.slot, t, row)] =
                        (live && row < x.len) ? float(d[4 * jb + 2 * h2 + e]) * a.scale : ninf;
                }
              }
            }
          }
        });
    shfl_best(bv0, bi0, 1);
    shfl_best(bv0, bi0, 2);
    shfl_best(bv1, bi1, 1);
    shfl_best(bv1, bi1, 2);
    if ((lane & 3) == 0) {
      if (tok0 < x.t1) write_token(a, x, tok0, float(bv0) * a.scale, bi0);
      if (tok1 < x.t1) write_token(a, x, tok1, float(bv1) * a.scale, bi1);
    }
    explain_fill(a, x.slot, x.t0, x.t1, int64_t(n_tiles) * kTileN, false);  // map rows past the last tile
  }
}

// ------------------------------------------------------------------ 1-bit corpora: 128 - popc(q ^ d), exact
__global__ void __launch_bounds__(kExplainB1Threads)
maxsim_explain_b1(const __grid_constant__ ExplainArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint4* qrows = static_cast<const uint4*>(a.q);
  const uint4* prows = static_cast<const uint4*>(a.rows);
  const float ninf = -__int_as_float(0x7f800000);
  const int n_slots = a.n_q * a.n_cand;
  for (int tt = blockIdx.y; tt < a.n_ttiles; tt += gridDim.y)
  for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
    const ExplainItem x = explain_item(a, slot, tt);
    if (x.skip) continue;
    if (!x.compute) {
      explain_fill(a, x.slot, x.t0, x.t1, 0, true);
      continue;
    }
    const int64_t qrow0 = int64_t(__ldg(a.goff + x.q)) * kGroup;
    for (int t = x.t0 + warp; t < x.t1; t += kExplainB1Threads / 32) {
      if (t >= x.qlen) {  // warp-uniform
        if (lane == 0) write_token(a, x, t, 0.f, -1);
        if (a.sim_map)
          for (int64_t row = lane; row < a.map_rows; row += 32) a.sim_map[map_index(a, x.slot, t, row)] = ninf;
        continue;
      }
      const uint4 qv = __ldg(qrows + qrow0 + t);
      int bv = 0, bi = -1;
      for (int row = lane; row < x.len; row += 32) {
        const uint4 dv = __ldg(prows + x.row0 + row);
        const int v = 128 - (__popc(qv.x ^ dv.x) + __popc(qv.y ^ dv.y) + __popc(qv.z ^ dv.z) + __popc(qv.w ^ dv.w));
        if (beats(v, row, bv, bi)) {
          bv = v;
          bi = row;
        }
        if (a.sim_map && row < a.map_rows) a.sim_map[map_index(a, x.slot, t, row)] = float(v) * a.scale;
      }
      if (a.sim_map)
        for (int64_t row = x.len + lane; row < a.map_rows; row += 32) a.sim_map[map_index(a, x.slot, t, row)] = ninf;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) shfl_best(bv, bi, o);
      if (lane == 0) write_token(a, x, t, float(bv) * a.scale, bi);
    }
  }
}

// ------------------------------------------------------------------ host side
static int launch_explain(b200ms_t* h, const ExplainArgs& a, int dtype, cudaStream_t s) {
  // grid.y walks the token tiles, grid.x the slots: about eight CTAs per SM in all
  const int n_slots = a.n_q * a.n_cand;
  if (n_slots == 0 || a.n_ttiles == 0) return B200MS_OK;
  const int gy = a.n_ttiles < 65535 ? a.n_ttiles : 65535;
  int gx = (h->num_sms * 8 + gy - 1) / gy;
  if (gx > n_slots) gx = n_slots;
  const dim3 grid{unsigned(gx), unsigned(gy)};
  RowTileKernel<ExplainArgs> k;
  if (int e = row_tile_kernel(h, dtype, maxsim_explain_wgmma<0>, maxsim_explain_wgmma<1>, maxsim_explain_wgmma<2>,
                              maxsim_explain_b1, kExplainB1Threads, "maxsim_explain", &k))
    return e;
  return launch_row_tiles(h, k, grid, a, s, "launch maxsim_explain");
}

}  // namespace bms

using namespace bms;

#define B200MS_API extern "C" __attribute__((visibility("default")))

B200MS_API int b200ms_explain_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                     const int64_t* page_ids_dev, int n_cand, float i8_q_scale, float score_scale,
                                     float* token_scores, int32_t* best_rows, float* sim_map, int64_t map_rows, void* stream) {
  if (!h) return B200MS_EINVAL;
  if ((src_dtype != B200MS_F32 && src_dtype != B200MS_BF16) || !q_dev || !q_lens || n_q < 1 || !page_ids_dev || n_cand < 1 ||
      int64_t(n_q) * n_cand >= (int64_t(1) << 30) || map_rows < 0 || !token_scores || !best_rows)
    return set_error(h, B200MS_EINVAL,
                     "explain_device: bad arguments (F32/BF16 queries, n_q >= 1, n_cand >= 1, n_q*n_cand < 2^30, map_rows >= 0)");
  int t_max = 0;
  for (int i = 0; i < n_q; ++i) {
    if (q_lens[i] < 0) return set_error(h, B200MS_EINVAL, "explain_device: negative query length");
    t_max = q_lens[i] > t_max ? q_lens[i] : t_max;
  }
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "explain: no corpus attached (call b200ms_set_corpus first)");
  if (t_max == 0) return B200MS_OK;  // every output is empty
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  // the queries, packed as b200ms_search_device packs them
  const SearchMeta m = build_search_meta(q_lens, n_q);
  const int64_t q_rows = m.groups_padded * kGroup;
  if (int e = reserve(h, h->q_packed, size_t(q_rows) * size_t(b200ms_row_bytes(c.dtype)))) return e;
  if (int e = upload(h, h->meta, m.host.data(), m.host.size(), s)) return e;
  const uint8_t* md = static_cast<const uint8_t*>(h->meta.p);
  const int64_t* ss_dev = reinterpret_cast<const int64_t*>(md);
  if (int e = launch_pack_rows(h, q_dev, src_dtype, ss_dev, reinterpret_cast<const int64_t*>(md + m.off_ds), n_q, q_rows, 1,
                               h->q_packed.p, c.dtype, i8_q_scale, s))
    return e;
  ExplainArgs a;
  a.q = h->q_packed.p;
  a.q_rows = q_rows;
  a.ss = ss_dev;
  a.goff = reinterpret_cast<const int32_t*>(md + m.off_goff);
  a.n_q = n_q;
  a.n_cand = n_cand;
  a.t_max = t_max;
  a.n_ttiles = (t_max + kExplainTokens - 1) / kExplainTokens;
  a.ids = page_ids_dev;
  a.unit_ids = page_ids_dev;
  a.n_pages = c.n_pages;
  a.page_len = static_cast<const int32_t*>(h->page_len.p);
  a.scale = score_scale;
  a.token_scores = token_scores;
  a.best_rows = best_rows;
  a.sim_map = map_rows > 0 ? sim_map : nullptr;
  a.map_rows = map_rows;
  const CorpusView whole = corpus_view(h);
  a.rows = whole.rows;
  a.page_start = whole.page_start;
  if (!c.host) return launch_explain(h, a, c.dtype, s);
  // host-resident corpus: the requested pages are gathered into the staging block round by round, exactly as for a rerank;
  // every round writes the slots whose page it holds (and the fill of unused slots, which is the same in every round)
  struct Ctx {
    ExplainArgs a;
    cudaStream_t s;
  } ctx{a, s};
  auto round = [](b200ms_t* hh, const CorpusView& v, const int64_t* remap, int, int, void* p) {
    Ctx& x = *static_cast<Ctx*>(p);
    ExplainArgs ar = x.a;
    ar.unit_ids = remap;
    ar.rows = v.rows;
    ar.page_start = v.page_start;
    return launch_explain(hh, ar, v.dtype, x.s);
  };
  if (int e = gather_host_tier(h, page_ids_dev, int64_t(n_q) * n_cand, s, round, &ctx)) return e;
  // no requested page has a row: nothing was gathered and every slot is a fill, which reads no rows
  if (h->ht_rounds == 0) return launch_explain(h, a, c.dtype, s);
  return B200MS_OK;
}
