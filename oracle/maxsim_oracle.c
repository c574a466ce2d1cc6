/*
 * oracle/maxsim_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C) of the reference's ColPali late-interaction path.  Nothing in the
 * product (morphik-core_b200/) may link, import or call this file; it is the checker used by
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
 *
 * Every function cites the reference lines it restates (paths relative to the morphik-core repository root):
 *   - sign quantise + MSB-first pack : core/utils/fast_ops.py:191-227 (authoritative pure-Python
 *                                      fallback), morphik_rust/src/binary_ops.rs:147-222
 *   - Hamming distance               : core/utils/fast_ops.py:230-248, binary_ops.rs:237-292
 *   - binary MaxSim (SQL max_sim)    : core/vector_store/multi_vector_store.py:287-311
 *   - float MaxSim                   : core/vector_store/fast_multivector_store.py:553-557 calling
 *                                      colpali_engine v0.3.13 score_multi_vector (third party, pinned
 *                                      pyproject.toml:72; identical port in transformers
 *                                      models/colpali/processing_colpali.py:350-362)
 *   - top-k                          : multi_vector_store.py:759 (ORDER BY similarity DESC LIMIT k),
 *                                      fast_multivector_store.py:556 (torch.topk)
 *
 * Pinning (see tests/test_oracle_golden.py): the quantiser and Hamming functions are checked against
 * outputs of the reference's own fast_ops.py executed in the build container plus the Rust unit-test
 * vectors (binary_ops.rs:299-333); float MaxSim against outputs of the transformers port of
 * score_multi_vector; binary MaxSim against the known answers implied by
 * core/tests/unit/test_multivector.py:94-109,166-177,222-256 (Postgres itself is not runnable here).
 * The int8 scorer has no reference counterpart (SURVEY F5) -- it is defined here.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define ORACLE_API __attribute__((visibility("default")))

ORACLE_API int oracle_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* ------------------------------------------------------------------------------------------------
 * fast_ops.py:191-227 / binary_ops.rs:96-118: bit_i = (float32(x_i) > 0) (strict: 0.0, -0.0, NaN -> 0),
 * element i goes to bit (7 - i%8) of byte i/8 (MSB first).  dim need not be a multiple of 8
 * (the fallback pads the last byte with zero bits: num_bytes = (len+7)//8).
 * ---------------------------------------------------------------------------------------------- */
ORACLE_API void oracle_sign_pack(const float* x, int64_t n_rows, int dim, uint8_t* out) {
  const int nb = (dim + 7) / 8;
  for (int64_t r = 0; r < n_rows; ++r) {
    uint8_t* o = out + r * nb;
    memset(o, 0, (size_t)nb);
    for (int i = 0; i < dim; ++i) {
      if (x[r * dim + i] > 0.0f) o[i / 8] |= (uint8_t)(1u << (7 - (i % 8)));
    }
  }
}

/* fast_ops.py:230-239 / binary_ops.rs:237-251: popcount(a XOR b) summed byte-wise. */
ORACLE_API uint32_t oracle_hamming(const uint8_t* a, const uint8_t* b, int64_t len) {
  uint32_t s = 0;
  for (int64_t i = 0; i < len; ++i) s += (uint32_t)__builtin_popcount((unsigned)(a[i] ^ b[i]));
  return s;
}

/* ------------------------------------------------------------------------------------------------
 * SQL public.max_sim(document bit[], query bit[]) -- multi_vector_store.py:287-311.
 *   similarity(q,d) = 1.0 - bit_count(d # q) / greatest(bit_length(q), 1)
 *   per query element (row_number => duplicates count separately): MAX over document elements
 *   result = COALESCE(SUM(max), 0.0)      (empty document or empty query -> 0.0)
 * Corpus rows are nbytes-wide packed bit strings; page p owns rows [page_off[p], page_off[p+1]).
 * scores_out[p] is a double like Postgres' float8; sim_int_out (optional) is the exact integer
 * form  sum_t max_p (nbits - ham)  that the GPU kernel is compared with bit-for-bit.
 * ---------------------------------------------------------------------------------------------- */
ORACLE_API void oracle_binary_maxsim(const uint8_t* q_bits, int n_tok, const uint8_t* d_bits,
                                     const int64_t* page_off, int64_t n_pages, int nbytes,
                                     double* scores_out, int64_t* sim_int_out) {
  const int nbits = nbytes * 8;
  const double denom = (double)(nbits > 1 ? nbits : 1);
#pragma omp parallel for schedule(dynamic, 16)
  for (int64_t p = 0; p < n_pages; ++p) {
    const int64_t r0 = page_off[p], r1 = page_off[p + 1];
    double total = 0.0;
    int64_t total_int = 0;
    if (r1 > r0) {
      for (int t = 0; t < n_tok; ++t) {
        const uint8_t* q = q_bits + (int64_t)t * nbytes;
        uint32_t best = 0xffffffffu; /* min Hamming == max similarity */
        for (int64_t r = r0; r < r1; ++r) {
          const uint32_t h = oracle_hamming(q, d_bits + r * nbytes, nbytes);
          if (h < best) best = h;
        }
        total += 1.0 - (double)best / denom;
        total_int += (int64_t)nbits - (int64_t)best;
      }
    }
    scores_out[p] = total;
    if (sim_int_out) sim_int_out[p] = total_int;
  }
}

/* ------------------------------------------------------------------------------------------------
 * Float MaxSim -- restates score_multi_vector (A.2 of SURVEY.md):
 *   for passage batches of `batch` pages: zero-pad pages to the batch's longest page,
 *   S[q,c] = sum_n max_s dot(Q[q,n,:], P[c,s,:])        (max INCLUDES the zero rows when
 *   zero_pad_compat != 0 and the page is shorter than its batch max => max(true_max, 0)).
 * With zero_pad_compat == 0 this is the clean MaxSim (explicit page lengths, empty page -> 0).
 * One query at a time: q is [n_tok, dim].  Dot products accumulate in double, output is float32
 * (the reference returns .to(float32)).
 * ---------------------------------------------------------------------------------------------- */
ORACLE_API void oracle_float_maxsim(const float* q, int n_tok, const float* rows, const int64_t* page_off,
                                    int64_t n_pages, int dim, int zero_pad_compat, int batch,
                                    float* scores_out) {
  if (batch <= 0) batch = 128;
#pragma omp parallel for schedule(dynamic, 4)
  for (int64_t p = 0; p < n_pages; ++p) {
    const int64_t r0 = page_off[p], r1 = page_off[p + 1];
    int padded = 0;
    if (zero_pad_compat) {
      const int64_t b0 = (p / batch) * batch;
      const int64_t b1 = (b0 + batch < n_pages) ? b0 + batch : n_pages;
      int64_t longest = 0;
      for (int64_t j = b0; j < b1; ++j) {
        const int64_t len = page_off[j + 1] - page_off[j];
        if (len > longest) longest = len;
      }
      padded = (r1 - r0) < longest;
    }
    double total = 0.0;
    if (r1 > r0 || padded) {
      for (int t = 0; t < n_tok; ++t) {
        const float* qt = q + (int64_t)t * dim;
        double best = padded ? 0.0 : -INFINITY;
        for (int64_t r = r0; r < r1; ++r) {
          const float* pr = rows + r * dim;
          double acc = 0.0;
          for (int d = 0; d < dim; ++d) acc += (double)qt[d] * (double)pr[d];
          if (acc > best) best = acc;
        }
        total += best;
      }
    }
    scores_out[p] = (float)total;
  }
}

/* ------------------------------------------------------------------------------------------------
 * int8 MaxSim (no reference counterpart, SURVEY F5 / 8d "bit-exact mode"): pure integer
 *   S[p] = sum_t max_s sum_d q_i8[t,d] * p_i8[s,d]      (int32 dot, int64 sum; empty page -> 0)
 * zero_pad_compat / batch: the same switch as oracle_float_maxsim -- a page shorter than the longest page of its
 * batch of `batch` pages (page-id order) scores sum_t max(max_s dot, 0).
 * ---------------------------------------------------------------------------------------------- */
ORACLE_API void oracle_int8_maxsim(const int8_t* q, int n_tok, const int8_t* rows, const int64_t* page_off,
                                   int64_t n_pages, int dim, int zero_pad_compat, int batch, int64_t* scores_out) {
  if (batch <= 0) batch = 128;
#pragma omp parallel for schedule(dynamic, 4)
  for (int64_t p = 0; p < n_pages; ++p) {
    const int64_t r0 = page_off[p], r1 = page_off[p + 1];
    int padded = 0;
    if (zero_pad_compat) {
      const int64_t b0 = (p / batch) * batch;
      const int64_t b1 = (b0 + batch < n_pages) ? b0 + batch : n_pages;
      int64_t longest = 0;
      for (int64_t j = b0; j < b1; ++j) {
        const int64_t len = page_off[j + 1] - page_off[j];
        if (len > longest) longest = len;
      }
      padded = (r1 - r0) < longest;
    }
    int64_t total = 0;
    if (r1 > r0 || padded) {
      for (int t = 0; t < n_tok; ++t) {
        const int8_t* qt = q + (int64_t)t * dim;
        int32_t best = padded ? 0 : INT32_MIN;
        for (int64_t r = r0; r < r1; ++r) {
          const int8_t* pr = rows + r * dim;
          int32_t acc = 0;
          for (int d = 0; d < dim; ++d) acc += (int32_t)qt[d] * (int32_t)pr[d];
          if (acc > best) best = acc;
        }
        total += best;
      }
    }
    scores_out[p] = total;
  }
}

/* ------------------------------------------------------------------------------------------------
 * Top-k: ORDER BY similarity DESC LIMIT k (multi_vector_store.py:759) / torch.topk
 * (fast_multivector_store.py:556).  Ties are unspecified in the reference; the build's rule is
 * "lower page index first".  allow (optional) is a bitmask, bit (p & 31) of word p >> 5.
 * Returns the number of results written (<= k).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
  double s;
  int64_t id;
} oracle_pair_t;

static int oracle_pair_cmp(const void* a, const void* b) {
  const oracle_pair_t* x = (const oracle_pair_t*)a;
  const oracle_pair_t* y = (const oracle_pair_t*)b;
  if (x->s > y->s) return -1;
  if (x->s < y->s) return 1;
  return (x->id > y->id) - (x->id < y->id);
}

ORACLE_API int64_t oracle_topk(const double* scores, int64_t n, const uint32_t* allow, int64_t k,
                               double* top_scores, int64_t* top_ids) {
  oracle_pair_t* v = (oracle_pair_t*)malloc(sizeof(oracle_pair_t) * (size_t)(n > 0 ? n : 1));
  int64_t m = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (allow && !((allow[i >> 5] >> (i & 31)) & 1u)) continue;
    v[m].s = scores[i];
    v[m].id = i;
    ++m;
  }
  qsort(v, (size_t)m, sizeof(oracle_pair_t), oracle_pair_cmp);
  const int64_t out = m < k ? m : k;
  for (int64_t i = 0; i < out; ++i) {
    top_scores[i] = v[i].s;
    top_ids[i] = v[i].id;
  }
  free(v);
  return out;
}
