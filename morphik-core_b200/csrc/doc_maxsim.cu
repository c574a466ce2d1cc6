// doc_maxsim.cu -- documents ranked by document-level MaxSim (b200ms_search_doc_maxsim_device,
// b200ms_rerank_doc_maxsim_batch_device):  S(q, D) = sum over q's tokens t of max over D's pages p and rows r of <q_t, d_r>.
//
//   1. the wgmma scan in document mode (maxsim_wgmma.cu, DocScan) leaves table[t, D] = the best (token max, page) of every
//      true token row t of the pass and every document, as a packed 64-bit key (0 = no page of D counted);
//   2. doc_sum_kernel adds every (query, document)'s token maxima in the order a page's score is added -- group_sum's tree
//      inside a 32-token group, then the groups in order as page_key adds them (SumOf / finish_sum for int scores) -- into
//      a [n_q, n_docs] score matrix with one "group" per query, and a mask of the documents that have a counted page;
//   3. launch_topk selects the k best documents of every query from that matrix (key_of's order, ties to the lower
//      document);
//   4. doc_evidence_kernel decodes the arg-max pages of each selected document, adds each distinct page's share in token
//      order and keeps the per_doc largest.
// The two-stage form first turns every query's candidate pages into an allow-mask row over the pages of their documents.
// A batch whose table would pass kDocTableBytes runs as several passes of whole queries.
#include <math_constants.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "topk_keys.cuh"

namespace bms {

constexpr int kDocSumThreads = 256;
constexpr int kEvidenceThreads = 256;

// evidence order of a share: float shares as key_of_canonical orders them (NaN first, -0 = +0), int shares by value
__device__ __forceinline__ uint64_t share_key(float s) { return key_of_canonical(s); }
__device__ __forceinline__ uint64_t share_key(int64_t s) { return uint64_t(s) ^ (uint64_t(1) << 63); }

// token max of a table entry: the key doc_token_key wrote (1 = NaN)
__device__ __forceinline__ float token_of_key(uint32_t k, float) { return k == 1u ? __int_as_float(0x7fffffff) : score_of_key(k, 0.f); }
__device__ __forceinline__ int token_of_key(uint32_t k, int) { return int(k ^ 0x80000000u); }
// M[t, D] of a table entry of token row `row`: its token max, plus the 1-bit token constant c_t (tok_const != NULL), which
// the document-mode scan leaves out
template <typename T>
__device__ __forceinline__ T token_max(unsigned long long e, const int32_t* tok_const, int64_t row) {
  T m = token_of_key(uint32_t(e >> 32), T(0));
  if (tok_const) m += T(__ldg(tok_const + row));
  return m;
}

// score[q, d] (row stride ld) and bit d of found row q (ld / 32 words): one thread per (query, document).  The 32 token
// maxima of a group are added as group_sum adds them: lane quad j holds tokens j, j+8, j+16, j+24 and sums them as
// (t_j + t_j+8) + (t_j+16 + t_j+24), then the quads pair up by xor 1, 2 and 4 -- float addition is commutative, so the
// butterfly's result is this tree's.
template <typename T>
__global__ void __launch_bounds__(kDocSumThreads)
doc_sum_kernel(const unsigned long long* __restrict__ table, int64_t n_docs, const int32_t* __restrict__ goff,
               const int32_t* __restrict__ ntok, const int32_t* __restrict__ tok_const, T* __restrict__ score, int64_t ld,
               uint32_t* __restrict__ found) {
  const int q = blockIdx.y;
  const int64_t d = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int g0 = __ldg(goff + q), g1 = __ldg(goff + q + 1);
  bool ok = d < n_docs && g1 > g0 && table[int64_t(g0) * kGroup * n_docs + d] != 0ull;
  if (ok) {
    typename SumOf<T>::type acc = 0;
    for (int g = g0; g < g1; ++g) {
      const int nt = __ldg(ntok + g);
      const unsigned long long* col = table + int64_t(g) * kGroup * n_docs + d;
      T s[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        T v[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int t = j + 8 * c;
          v[c] = t < nt ? token_max<T>(col[int64_t(t) * n_docs], tok_const, int64_t(g) * kGroup + t) : T(0);
        }
        s[j] = (v[0] + v[1]) + (v[2] + v[3]);
      }
      acc += ((s[0] + s[1]) + (s[2] + s[3])) + ((s[4] + s[5]) + (s[6] + s[7]));
    }
    score[int64_t(q) * ld + d] = finish_sum(acc);
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, ok);
  if ((threadIdx.x & 31) == 0 && d < ld) found[int64_t(q) * (ld / 32) + (d >> 5)] = bal;
}

// Evidence of selected document i of query q (one block each): the distinct arg-max pages of its tokens, each with its
// share (the token maxima it holds, added in token order), the per_doc largest shares first (ties: lower page).
template <typename T>
__global__ void __launch_bounds__(kEvidenceThreads)
doc_evidence_kernel(const unsigned long long* __restrict__ table, int64_t n_docs, const int32_t* __restrict__ goff,
                    const int32_t* __restrict__ ntok, const int32_t* __restrict__ tok_const, const int64_t* __restrict__ top_ids,
                    const int32_t* __restrict__ top_counts, int k, int per_doc, float scale, int64_t id_base,
                    float* __restrict__ ev_scores, int64_t* __restrict__ ev_ids, int32_t* __restrict__ ev_counts) {
  using S = typename SumOf<T>::type;
  extern __shared__ uint8_t smem_raw[];
  __shared__ int n_dist;
  const int q = blockIdx.y, i = blockIdx.x;
  const int64_t o = (int64_t(q) * k + i) * per_doc;
  const int cnt = top_counts[q];
  const int g0 = __ldg(goff + q), g1 = __ldg(goff + q + 1);
  const int n_tok = i < cnt && g1 > g0 ? (g1 - g0 - 1) * kGroup + __ldg(ntok + g1 - 1) : 0;
  S* share = reinterpret_cast<S*>(smem_raw);                      // [n_tok]
  T* val = reinterpret_cast<T*>(share + n_tok);                  // [n_tok]
  uint32_t* page = reinterpret_cast<uint32_t*>(val + n_tok);     // [n_tok]
  uint32_t* dpage = page + n_tok;                                // [n_tok]
  if (threadIdx.x == 0) n_dist = 0;
  if (n_tok > 0) {
    const int64_t d = top_ids[int64_t(q) * k + i];
    const unsigned long long* col = table + int64_t(g0) * kGroup * n_docs + d;
    for (int t = threadIdx.x; t < n_tok; t += blockDim.x) {
      const unsigned long long key = col[int64_t(t) * n_docs];
      page[t] = ~uint32_t(key);
      val[t] = token_max<T>(key, tok_const, int64_t(g0) * kGroup + t);
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < n_tok; t += blockDim.x) {
    const uint32_t p = page[t];
    bool first = true;
    for (int u = 0; u < t && first; ++u) first = page[u] != p;
    if (first) {
      S acc = 0;
      for (int u = t; u < n_tok; ++u)
        if (page[u] == p) acc += val[u];
      const int e = atomicAdd(&n_dist, 1);
      dpage[e] = p;
      share[e] = acc;
    }
  }
  __syncthreads();
  const int n = n_dist;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const uint64_t ke = share_key(share[e]);
    int rank = 0;
    for (int f = 0; f < n && rank < per_doc; ++f) {
      const uint64_t kf = share_key(share[f]);
      rank += kf > ke || (kf == ke && dpage[f] < dpage[e]);
    }
    if (rank < per_doc) {
      ev_scores[o + rank] = float(finish_sum(share[e])) * scale;
      ev_ids[o + rank] = int64_t(dpage[e]) + id_base;
    }
  }
  const int used = n < per_doc ? n : per_doc;
  for (int t = used + threadIdx.x; t < per_doc; t += blockDim.x) {
    ev_scores[o + t] = -CUDART_INF_F;
    ev_ids[o + t] = -1;
  }
  if (threadIdx.x == 0) ev_counts[int64_t(q) * k + i] = used;
}

// bit d of docs row q = some valid slot of q's candidate list is a page of document d (rows zeroed by the caller)
__global__ void doc_mark_kernel(const int64_t* __restrict__ cand, int n_cand, int n_q, int64_t n_pages,
                                const int32_t* __restrict__ page_doc, int64_t n_docs, uint32_t* __restrict__ docs,
                                int64_t doc_words) {
  const int64_t n = int64_t(n_q) * n_cand;
  for (int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < n; j += int64_t(gridDim.x) * blockDim.x) {
    const int64_t p = __ldg(cand + j);
    if (p < 0 || p >= n_pages) continue;
    const int d = __ldg(page_doc + p);
    if (d < 0 || d >= n_docs) continue;
    atomicOr(docs + (j / n_cand) * doc_words + (d >> 5), 1u << (d & 31));
  }
}

// allow row q over the pages = (q's row of the caller's masks, as SearchRequest) AND (the page's document is marked in q's
// docs row); one thread per (query, page word)
__global__ void doc_allow_kernel(const uint32_t* __restrict__ docs, int64_t doc_words, int n_q, int64_t n_pages,
                                 const int32_t* __restrict__ page_doc, int64_t n_docs, const uint32_t* __restrict__ allow,
                                 const int32_t* __restrict__ mask_index, uint32_t* __restrict__ out) {
  const int64_t words = (n_pages + 31) / 32;
  const int64_t n = int64_t(n_q) * words;
  for (int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < n; j += int64_t(gridDim.x) * blockDim.x) {
    const int q = int(j / words);
    const int64_t w = j - int64_t(q) * words;
    uint32_t a = 0xffffffffu;
    if (allow) {
      const int mi = mask_index ? __ldg(mask_index + q) : 0;
      if (mi >= 0) a = __ldg(allow + int64_t(mi) * words + w);
    }
    uint32_t b = 0;
    for (int l = 0; l < 32 && (a >> l); ++l) {
      const int64_t p = w * 32 + l;
      if (!((a >> l) & 1u) || p >= n_pages) continue;
      const int d = __ldg(page_doc + p);
      if (d >= 0 && d < n_docs && ((__ldg(docs + q * doc_words + (d >> 5)) >> (d & 31)) & 1u)) b |= 1u << l;
    }
    out[j] = b;
  }
}

// outputs of queries that find no document
__global__ void doc_empty_kernel(int n, int k, int per_doc, float* doc_scores, int64_t* doc_ids, float* ev_scores,
                                 int64_t* ev_ids, int32_t* ev_counts, int32_t* doc_counts) {
  const int64_t nk = int64_t(n) * k;
  for (int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < nk * per_doc; j += int64_t(gridDim.x) * blockDim.x) {
    ev_scores[j] = -CUDART_INF_F;
    ev_ids[j] = -1;
    if (j < nk) {
      doc_scores[j] = -CUDART_INF_F;
      doc_ids[j] = -1;
      ev_counts[j] = 0;
    }
    if (j < n) doc_counts[j] = 0;
  }
}

int64_t doc_table_bytes(int64_t groups, int64_t n_docs) { return groups * kGroup * n_docs * 8; }

// One pass: queries [q0, q0 + n) of the call.  allow / mask_index as DocScan (mask_index already offset to the pass);
// row_per_query: allow holds one row per query of the pass.
template <typename T>
static int doc_pass(b200ms_t* h, const DocMaxSimCall& x, int q0, int n, const uint32_t* allow, const int32_t* mask_index,
                    bool row_per_query, cudaStream_t s) {
  const Corpus& c = h->corpus;
  const int32_t* lens = x.q_lens + q0;
  int64_t row0 = 0;
  for (int q = 0; q < q0; ++q) row0 += x.q_lens[q];
  const void* q = static_cast<const uint8_t*>(x.q) + row0 * kDim * (x.q_dtype == B200MS_F32 ? 4 : 2);
  const SearchMeta m = build_search_meta(lens, n);
  const int ng = int(m.groups);
  // device block: [meta | group_query int32 [groups] | iota int32 [n + 1]]
  std::vector<uint8_t> blk(m.host);
  blk.resize((blk.size() + 15) & ~size_t(15));
  const size_t off_gq = blk.size(), off_iota = off_gq + size_t(ng) * 4;
  blk.resize(off_iota + size_t(n + 1) * 4);
  int32_t* gq = reinterpret_cast<int32_t*>(blk.data() + off_gq);
  for (int i = 0; i < n; ++i)
    for (int g = m.goff()[i]; g < m.goff()[i + 1]; ++g) gq[g] = i;
  int32_t* iota = reinterpret_cast<int32_t*>(blk.data() + off_iota);
  for (int i = 0; i <= n; ++i) iota[i] = i;
  if (int e = upload(h, h->meta, blk.data(), blk.size(), s)) return e;
  const uint8_t* md = static_cast<const uint8_t*>(h->meta.p);
  const int32_t* ntok_dev = reinterpret_cast<const int32_t*>(md + m.off_ntok);
  const int32_t* goff_dev = reinterpret_cast<const int32_t*>(md + m.off_goff);
  const int32_t* iota_dev = reinterpret_cast<const int32_t*>(md + off_iota);
  float* doc_scores = x.doc_scores + int64_t(q0) * x.k;
  int64_t* doc_ids = x.doc_ids + int64_t(q0) * x.k;
  int32_t* doc_counts = x.doc_counts + q0;
  float* ev_scores = x.ev_scores + int64_t(q0) * x.k * x.per_doc;
  int64_t* ev_ids = x.ev_ids + int64_t(q0) * x.k * x.per_doc;
  int32_t* ev_counts = x.ev_counts + int64_t(q0) * x.k;
  if (ng == 0 || x.n_docs == 0 || c.n_pages == 0) {
    doc_empty_kernel<<<grid_stride_blocks(h, int64_t(n) * x.k * x.per_doc, 256, 8), 256, 0, s>>>(
        n, x.k, x.per_doc, doc_scores, doc_ids, ev_scores, ev_ids, ev_counts, doc_counts);
    h->launches++;
    return check_cuda(h, cudaGetLastError(), "launch doc_empty");
  }
  // pack -> filtered plan -> table -> document-mode scan
  const int64_t gp = m.groups_padded;
  if (int e = reserve(h, h->q_packed, size_t(gp) * kGroup * size_t(b200ms_row_bytes(c.dtype)))) return e;
  const int64_t* ss_dev = reinterpret_cast<const int64_t*>(md);
  const int64_t* ds_dev = reinterpret_cast<const int64_t*>(md + m.off_ds);
  if (int e = launch_pack_rows(h, q, x.q_dtype, ss_dev, ds_dev, n, gp * kGroup, 1, h->q_packed.p, c.dtype, x.i8_q_scale, s))
    return e;
  if (row_per_query) mask_index = iota_dev;
  UnitPlan plan;
  if (int e = plan_full_scan(h, allow, mask_index, n, s, &plan)) return e;
  const int64_t tb = doc_table_bytes(ng, x.n_docs);
  if (int e = reserve(h, h->dm_table, size_t(tb))) return e;
  auto* table = static_cast<unsigned long long*>(h->dm_table.p);
  if (int e = check_cuda(h, cudaMemsetAsync(table, 0, size_t(tb), s), "doc_maxsim: memset")) return e;
  DocScan ds;
  ds.table = table;
  ds.n_docs = x.n_docs;
  ds.page_doc = x.page_doc;
  ds.group_query = reinterpret_cast<const int32_t*>(md + off_gq);
  ds.allow = allow;
  ds.mask_index = mask_index;
  ds.mask_stride = (c.n_pages + 31) / 32;
  if (int e = c.dtype == B200MS_B1 ? launch_score_b1_wgmma(h, plan, h->q_packed.p, ntok_dev, ng, nullptr, 0, s, &ds)
                                   : launch_score_wgmma(h, corpus_view(h), plan, h->q_packed.p, ng, ntok_dev, nullptr, 0, s, 0,
                                                        -1, &ds))
    return e;
  const int32_t* tok_const = c.dtype == B200MS_B1 ? static_cast<const int32_t*>(h->b1_tok_const.p) : nullptr;
  // document scores and the found mask, then the selection over documents
  const int64_t ld = (x.n_docs + 31) & ~int64_t(31);
  if (int e = reserve(h, h->dm_scores, size_t(n) * size_t(ld) * 4 + size_t(n) * size_t(ld / 32) * 4)) return e;
  T* score = static_cast<T*>(h->dm_scores.p);
  uint32_t* found = reinterpret_cast<uint32_t*>(score + int64_t(n) * ld);
  doc_sum_kernel<T><<<dim3(unsigned(ld / kDocSumThreads + (ld % kDocSumThreads != 0)), unsigned(n)), kDocSumThreads, 0, s>>>(
      table, x.n_docs, goff_dev, ntok_dev, tok_const, score, ld, found);
  h->launches++;
  if (int e = check_cuda(h, cudaGetLastError(), "launch doc_sum")) return e;
  const int sdt = std::is_same<T, float>::value ? B200MS_F32 : B200MS_I32;
  if (int e = launch_topk(h, score, sdt, x.n_docs, ld, iota_dev, n, found, x.k, x.score_scale, 0, nullptr, doc_scores, doc_ids,
                          doc_counts, s, iota_dev, ld / 32))
    return e;
  // evidence
  int max_tok = 0;
  for (int i = 0; i < n; ++i) max_tok = std::max(max_tok, lens[i]);
  const int smem = max_tok * int(sizeof(typename SumOf<T>::type) + sizeof(T) + 8);
  auto kern = doc_evidence_kernel<T>;
  if (int e = ensure_smem(h, reinterpret_cast<const void*>(kern), smem, "cudaFuncSetAttribute(doc_evidence)")) return e;
  kern<<<dim3(unsigned(x.k), unsigned(n)), kEvidenceThreads, smem, s>>>(table, x.n_docs, goff_dev, ntok_dev, tok_const, doc_ids, doc_counts,
                                                                          x.k, x.per_doc, x.score_scale, x.id_base, ev_scores,
                                                                          ev_ids, ev_counts);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch doc_evidence");
}

int doc_maxsim(b200ms_t* h, const DocMaxSimCall& x, cudaStream_t s) {
  const Corpus& c = h->corpus;
  const char* what = x.cand ? "rerank_doc_maxsim_batch_device" : "search_doc_maxsim_device";
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, std::string(what) + ": no corpus attached");
  if (c.host)
    return set_error(h, B200MS_ESTATE, std::string(what) + ": the corpus is host-resident (document-level MaxSim reads "
                                                            "every page of a document; attach the corpus to HBM)");
  if (x.n_q < 1 || !x.q || !x.q_lens || x.k < 1 || x.k > B200MS_MAX_K || x.per_doc < 1 || x.per_doc > B200MS_MAX_PER_DOC ||
      !x.page_doc || x.n_docs < 0 || (c.n_pages > 0 && x.n_docs < 1) || x.n_docs > c.n_pages || x.n_masks < 0 ||
      (x.n_masks > 0 && (!x.allow || !x.mask_index)) || !x.doc_scores || !x.doc_ids || !x.ev_scores || !x.ev_ids ||
      !x.ev_counts || !x.doc_counts || (x.cand && x.n_cand < 1))
    return set_error(h, B200MS_EINVAL, std::string(what) + ": bad arguments (n_q >= 1, 1 <= k <= 4096, 1 <= per_doc <= 64, "
                                                            "1 <= n_docs <= n_pages, n_masks > 0 needs masks and indices)");
  for (int q = 0; q < x.n_q; ++q)
    if (x.q_lens[q] < 0 || x.q_lens[q] > kDocMaxTokens)
      return set_error(h, B200MS_EINVAL, std::string(what) + ": query " + std::to_string(q) + " has " +
                                             std::to_string(x.q_lens[q]) + " tokens (0 .. " +
                                             std::to_string(kDocMaxTokens) + ")");
  // passes of whole queries, each table within kDocTableBytes
  std::vector<int> cut{0};
  int64_t groups = 0;
  for (int q = 0; q < x.n_q; ++q) {
    const int64_t g = (x.q_lens[q] + kGroup - 1) / kGroup;
    if (doc_table_bytes(g, x.n_docs) > kDocTableBytes)
      return set_error(h, B200MS_EINVAL, std::string(what) + ": query " + std::to_string(q) + " (" +
                                             std::to_string(x.q_lens[q]) + " tokens, " + std::to_string(g * kGroup) +
                                             " padded) over " + std::to_string(x.n_docs) + " documents needs a " +
                                             std::to_string(doc_table_bytes(g, x.n_docs)) +
                                             "-byte token table; the bound is " + std::to_string(kDocTableBytes));
    if (doc_table_bytes(groups + g, x.n_docs) > kDocTableBytes) {
      cut.push_back(q);
      groups = 0;
    }
    groups += g;
  }
  cut.push_back(x.n_q);
  const int64_t words = (c.n_pages + 31) / 32;
  const uint32_t* allow = x.n_masks > 0 ? x.allow : nullptr;
  if (x.cand) {  // candidate documents -> one allow row per query
    const int64_t doc_words = (x.n_docs + 31) / 32 + 1;
    if (int e = reserve(h, h->dm_allow, size_t(x.n_q) * size_t(doc_words + words) * 4)) return e;
    uint32_t* docs = static_cast<uint32_t*>(h->dm_allow.p);
    uint32_t* rows = docs + int64_t(x.n_q) * doc_words;
    if (int e = check_cuda(h, cudaMemsetAsync(docs, 0, size_t(x.n_q) * size_t(doc_words) * 4, s), "doc_maxsim: memset"))
      return e;
    doc_mark_kernel<<<grid_stride_blocks(h, int64_t(x.n_q) * x.n_cand, 256, 8), 256, 0, s>>>(
        x.cand, x.n_cand, x.n_q, c.n_pages, x.page_doc, x.n_docs, docs, doc_words);
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch doc_mark")) return e;
    doc_allow_kernel<<<grid_stride_blocks(h, int64_t(x.n_q) * words, 256, 8), 256, 0, s>>>(
        docs, doc_words, x.n_q, c.n_pages, x.page_doc, x.n_docs, allow, x.n_masks > 0 ? x.mask_index : nullptr, rows);
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch doc_allow")) return e;
    allow = rows;
  }
  for (size_t i = 0; i + 1 < cut.size(); ++i) {
    const int q0 = cut[i], n = cut[i + 1] - cut[i];
    // a candidate call has one allow row per query (mask_index: the pass's own iota); else the caller's masks
    const uint32_t* a = x.cand ? allow + int64_t(q0) * words : allow;
    const int32_t* mask_index = !x.cand && x.n_masks > 0 ? x.mask_index + q0 : nullptr;
    const bool fl = c.dtype == B200MS_BF16 || c.dtype == B200MS_F8;
    const int e = fl ? doc_pass<float>(h, x, q0, n, a, mask_index, x.cand != nullptr, s)
                     : doc_pass<int>(h, x, q0, n, a, mask_index, x.cand != nullptr, s);
    if (e) return e;
  }
  return B200MS_OK;
}

}  // namespace bms
