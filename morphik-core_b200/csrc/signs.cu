// signs.cu -- asymmetric 1-bit MaxSim: full-precision queries against an HBM copy of the corpus' sign bits, the first stage
// of a two-stage search (no reference counterpart: the reference's first stages are the Turbopuffer ANN over FDEs,
// fast_multivector_store.py:521-532, and the symmetric SQL max_sim over sign bits, multi_vector_store.py:287-311).
//
// A sign row costs 16 B per patch vector (1/16 of bf16), so HBM holds the signs of corpora far larger than itself -- a
// host-resident one included -- and every page of them is scanned exhaustively; only the rerank candidates cross PCIe.
//
// Score:  S[q, p] = sum over the query's true tokens t of max over the page's true rows r of sum_i q8[t,i] * (+1 | -1)
// with q8 = clamp(rint(x * scale), -63, 63).  It runs on the 1-bit wgmma scan unchanged: the A operand is 2 q8 (|2 q8| <= 126
// fits int8), the patch bits are expanded to d' in {0, 1}, and the per-token constant is c_t = -sum_i q8[t,i], so
//   <2 q8, d'> + c_t = sum_i q8_i (2 d'_i - 1)  exactly.
#include <cmath>

#include "common.cuh"
#include "ptx.cuh"

namespace bms {

// Sign bits of packed rows [r0, r0 + n_rows): one thread per output byte (elements 8b .. 8b+7, MSB first).  The rule reads
// the packed value, so a corpus loaded from a shard file gets the signs of the live one: bit = value > 0, i.e.
//   BF16 0x0001 .. 0x7f80 (positive, +inf included; +-0 and NaN give 0), I8 1 .. 127, F8 e4m3 0x01 .. 0x7e (0x7f is NaN).
__global__ void __launch_bounds__(256)
sign_rows_kernel(const uint8_t* __restrict__ rows, int dtype, int64_t r0, int64_t n_rows, uint8_t* __restrict__ out) {
  const int64_t n = n_rows * 16;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t row = r0 + (i >> 4);
    const int b = int(i & 15);
    uint32_t byte = 0;
    if (dtype == B200MS_BF16) {
      const uint4 v = *reinterpret_cast<const uint4*>(rows + row * 256 + b * 16);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t x = (w[e >> 1] >> (16 * (e & 1))) & 0xffffu;
        byte |= uint32_t(x >= 1u && x <= 0x7f80u) << (7 - e);
      }
    } else {
      const uint2 v = *reinterpret_cast<const uint2*>(rows + row * 128 + b * 8);
      const uint32_t hi = dtype == B200MS_I8 ? 0x7fu : 0x7eu;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const uint32_t x = ((e < 4 ? v.x : v.y) >> (8 * (e & 3))) & 0xffu;
        byte |= uint32_t(x >= 1u && x <= hi) << (7 - e);
      }
    }
    out[i] = uint8_t(byte);
  }
}

// The A operand of the asymmetric scan: one warp per padded query row (lane l owns elements 4l .. 4l+3).  A row of query q
// at offset k < len(q) holds 2 q8 of token k and tok_const = -sum q8; padding rows and rows past the queries hold 0 and 0.
// ss / ds: [n_q + 1] true / padded row offsets (SearchMeta).
__global__ void __launch_bounds__(256)
sign_query_kernel(const void* __restrict__ src, int src_dtype, const int64_t* __restrict__ ss, const int64_t* __restrict__ ds,
                  int n_q, int64_t n_rows, float scale, uint32_t* __restrict__ q_i8, int32_t* __restrict__ tok_const) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t warp_stride = (int64_t(gridDim.x) * blockDim.x) >> 5;
  const int64_t used = n_q > 0 ? __ldg(ds + n_q) : 0;
  for (int64_t r = warp_global; r < n_rows; r += warp_stride) {
    int q8[4] = {0, 0, 0, 0};
    if (r < used) {
      int lo = 0, hi = n_q - 1;  // last query with ds[q] <= r
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(ds + mid) <= r) lo = mid; else hi = mid - 1;
      }
      const int64_t k = r - __ldg(ds + lo), s0 = __ldg(ss + lo);
      if (k < __ldg(ss + lo + 1) - s0) {
        const float4 v = load_row4(src, src_dtype, s0 + k, lane);
        const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float t = rintf(x[e] * scale);  // ties to even; +-inf clamp to +-63, NaN -> 0
          q8[e] = isnan(t) ? 0 : int(fminf(fmaxf(t, -63.f), 63.f));
        }
      }
    }
    q_i8[r * 32 + lane] = (uint32_t(2 * q8[0]) & 0xffu) | ((uint32_t(2 * q8[1]) & 0xffu) << 8) |
                          ((uint32_t(2 * q8[2]) & 0xffu) << 16) | ((uint32_t(2 * q8[3]) & 0xffu) << 24);
    const int sum = warp_sum(q8[0] + q8[1] + q8[2] + q8[3]);
    if (lane == 0) tok_const[r] = -sum;
  }
}

}  // namespace bms

using namespace bms;

#define B200MS_API extern "C" __attribute__((visibility("default")))

B200MS_API int b200ms_sign_rows(b200ms_t* h, int64_t first_page, int64_t n_pages, uint8_t* out, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "sign_rows: no corpus attached");
  if (c.dtype == B200MS_B1)
    return set_error(h, B200MS_ESTATE, "sign_rows: a 1-bit corpus has no more precise rows to rerank its signs with");
  if (first_page < 0 || n_pages < 0 || first_page + n_pages > c.n_pages || (n_pages > 0 && !out))
    return set_error(h, B200MS_EINVAL, "sign_rows: bad page range or NULL output");
  int64_t r0 = 0, r1 = 0;
  for (int64_t p = 0; p < first_page + n_pages; ++p) {
    const int64_t len = b200ms_padded_len(h->page_len_host[size_t(p)]);
    if (p < first_page) r0 += len;
    r1 += len;
  }
  if (r1 == r0) return B200MS_OK;
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  const int64_t n = (r1 - r0) * 16;
  const int64_t want = (n + 255) / 256, cap = int64_t(h->num_sms) * 16;
  sign_rows_kernel<<<int(want < cap ? want : cap), 256, 0, s>>>(static_cast<const uint8_t*>(c.rows), c.dtype, r0, r1 - r0, out);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch sign_rows");
}

B200MS_API int b200ms_set_sign_rows(b200ms_t* h, const void* sign_rows, int64_t n_rows, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "set_sign_rows: no corpus attached");
  if (c.dtype == B200MS_B1) return set_error(h, B200MS_ESTATE, "set_sign_rows: the corpus is 1-bit already");
  if (n_rows != c.n_rows || (n_rows > 0 && !sign_rows) || (reinterpret_cast<uintptr_t>(sign_rows) & 15))
    return set_error(h, B200MS_EINVAL, "set_sign_rows: need 16-byte aligned rows, exactly b200ms_corpus_rows of them");
  if (!c.scan_tables) {  // a host-resident corpus: the scan of its signs needs the tables an HBM corpus has from set_corpus
    DeviceGuard g(h->device);
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    StreamOrder order(h, s);  // a call still in flight may read the scratch the tables replace
    if (int e = order.error()) return e;
    std::vector<int64_t> ps(size_t(c.n_pages) + 1, 0);
    for (int64_t i = 0; i < c.n_pages; ++i) ps[size_t(i) + 1] = ps[size_t(i)] + b200ms_padded_len(h->page_len_host[size_t(i)]);
    if (int e = build_scan_tables(h, c, ps.data(), s)) return e;
    h->generation++;
  }
  c.sign_rows = sign_rows;
  c.signs = true;
  return B200MS_OK;
}

B200MS_API int b200ms_sign_candidates_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                             int n_cand, const uint32_t* allow_masks_dev, int n_masks,
                                             const int32_t* mask_index_dev, float i8_q_scale, float score_scale,
                                             float* cand_scores, int64_t* cand_ids, int32_t* cand_counts, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "sign_candidates: no corpus attached");
  if (!c.signs)
    return set_error(h, B200MS_ESTATE, "sign_candidates: no sign rows attached (b200ms_set_sign_rows after every set_corpus)");
  if ((src_dtype != B200MS_F32 && src_dtype != B200MS_BF16) || n_q < 1 || !q_lens || !q_dev || n_cand < 1 ||
      n_cand > B200MS_MAX_K || !cand_scores || !cand_ids || !cand_counts || !(i8_q_scale > 0.f) || !std::isfinite(i8_q_scale) ||
      n_masks < 0 || (n_masks > 0 && (!allow_masks_dev || !mask_index_dev)))
    return set_error(h, B200MS_EINVAL,
                     "sign_candidates: bad arguments (F32/BF16 queries, n_q >= 1, 1 <= n_cand <= 4096, finite i8_q_scale > 0, "
                     "n_masks > 0 needs the mask matrix and one index per query)");
  for (int i = 0; i < n_q; ++i)
    if (q_lens[i] < 0) return set_error(h, B200MS_EINVAL, "sign_candidates: negative query length");
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  const SearchMeta m = build_search_meta(q_lens, n_q);
  const int ng = int(m.groups);
  const auto [gp, ld] = score_layout(m, c.n_pages);
  if (int e = reserve(h, h->scores, size_t(gp) * size_t(ld) * 4)) return e;
  if (int e = upload(h, h->meta, m.host.data(), m.host.size(), s)) return e;
  const uint8_t* md = static_cast<const uint8_t*>(h->meta.p);
  const int32_t* goff_dev = reinterpret_cast<const int32_t*>(md + m.off_goff);
  const uint32_t* allow = n_masks > 0 ? allow_masks_dev : nullptr;
  const int32_t* mask_index = n_masks > 0 ? mask_index_dev : nullptr;
  if (ng > 0 && c.n_pages > 0) {
    const int64_t n_rows = gp * kGroup;
    int8_t* q_i8 = nullptr;
    int32_t* tok_const = nullptr;
    if (int e = reserve_b1_query(h, n_rows, &q_i8, &tok_const)) return e;
    const int64_t want = (n_rows + 7) / 8, cap = int64_t(h->num_sms) * 16;
    sign_query_kernel<<<int(want < cap ? want : cap), 256, 0, s>>>(
        q_dev, src_dtype, reinterpret_cast<const int64_t*>(md), reinterpret_cast<const int64_t*>(md + m.off_ds), n_q, n_rows,
        i8_q_scale, reinterpret_cast<uint32_t*>(q_i8), tok_const);
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch sign_query")) return e;
    if (c.has_empty)
      if (int e = zero_scores(h, h->scores.p, gp, ld, s, "sign_candidates: memset")) return e;
    UnitPlan plan;
    if (int e = plan_full_scan(h, allow, mask_index, n_q, s, &plan)) return e;
    CorpusView v = corpus_view(h);
    v.rows = c.sign_rows;
    v.dtype = B200MS_B1;
    v.tmap = nullptr;
    if (int e = launch_b1_tiles(h, v, plan, q_i8, tok_const, ng, h->scores.p, ld, s)) return e;
  } else if (int e = zero_scores(h, h->scores.p, gp, ld, s, "sign_candidates: memset")) {
    return e;
  }
  return launch_topk(h, h->scores.p, B200MS_I32, c.n_pages, ld, goff_dev, n_q, allow, n_cand, score_scale, 0, nullptr,
                     cand_scores, cand_ids, cand_counts, s, mask_index, (c.n_pages + 31) / 32);
}
