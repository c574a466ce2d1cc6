// maxsim_b1.cu -- the 1-bit (sign / Hamming) MaxSim scorer.
//
// Replaces SQL public.max_sim(document bit[], query bit[]) evaluated by Postgres over every row of
// multi_vector_embeddings (core/vector_store/multi_vector_store.py:287-311, scan at :746-763):
//     score = sum_t max_r (1 - popcount(d_r XOR q_t) / 128)
// The kernel produces the exact integer form  S[g,p] = sum_{t in group g} max_r (128 - popcount(d_r ^ q_t));
// score = S / 128 is exact in fp32 (SURVEY Appendix A.1), so parity with the oracle is bit-for-bit.
//
// Layout: corpus rows are 16-byte MSB-first packed sign bits (core/utils/fast_ops.py:191-227), pages padded to
// 32-row chunks by repeating the last row (min-Hamming invariant).  One warp owns one page; lane t owns query
// token t of up to G resident 32-token groups (bits in registers).  Each 32-row chunk is fetched with ONE
// coalesced 512-byte request (lane i loads row i as a uint4), parked in a per-warp shared-memory slab, and
// replayed row by row as 128-bit broadcast reads; per (row, token) the work is 6 LOP3 + 3 POPC (carry-save trick, see
// the kernel) + 2 ADD + 1 MIN.
// Bound: the integer POPC pipe, not HBM (16 B per patch vector; SURVEY 8d).
#include "common.cuh"
#include "ptx.cuh"

namespace bms {

constexpr int kB1Warps = 8;

template <int G>
__global__ void __launch_bounds__(kB1Warps * 32)
maxsim_b1_kernel(const uint4* __restrict__ rows, const int64_t* __restrict__ page_start, int64_t n_pages,
                 const int64_t* __restrict__ cand_ids /* NULL: every page; else n_pages candidates, output slot = index */,
                 const int32_t* __restrict__ n_cand_dev /* != NULL: the candidate count, a device word (n_pages bounds it) */,
                 int by_page /* candidates write their page's column, not their slot's (a filtered full scan) */,
                 int64_t corpus_pages /* candidate ids outside [0, corpus_pages) are unused slots */,
                 const uint4* __restrict__ q_bits /*[n_groups*32]*/, const int32_t* __restrict__ group_ntok, int g_base,
                 int n_groups, int32_t* __restrict__ group_scores, int64_t ld) {
  __shared__ uint4 slab[kB1Warps][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Hamming of 128 bits with 3 POPC instead of 4 (the POPC pipe, 16 lanes/clk/SM, is the measured limiter):
  // a carry-save adder compresses x0,x1,x2 (x_i = q_i ^ d_i) into sum s = x0^x1^x2 and carry c = maj(x0,x1,x2), so
  //   ham = popc(x0)+popc(x1)+popc(x2)+popc(x3) = popc(s) + 2*popc(c) + popc(x3).
  // s = (q0^q1^q2) ^ (d0^d1^d2): the query half is hoisted per token, the row half per row.
  uint4 q[G];
  uint32_t qs[G];
  int ntok[G];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int gg = g_base + g;
    const bool live = gg < n_groups;
    q[g] = live ? __ldg(q_bits + int64_t(gg) * 32 + lane) : make_uint4(0, 0, 0, 0);
    qs[g] = q[g].x ^ q[g].y ^ q[g].z;
    ntok[g] = live ? __ldg(group_ntok + gg) : 0;
  }
  if (n_cand_dev) n_pages = __ldg(n_cand_dev);
  const int64_t warp_global = int64_t(blockIdx.x) * kB1Warps + warp;
  const int64_t warp_stride = int64_t(gridDim.x) * kB1Warps;
  for (int64_t p = warp_global; p < n_pages; p += warp_stride) {
    const int64_t pg = cand_ids ? __ldg(cand_ids + p) : p;
    const bool live_page = pg >= 0 && pg < corpus_pages;
    const int64_t r0 = live_page ? __ldg(page_start + pg) : 0, r1 = live_page ? __ldg(page_start + pg + 1) : 0;
    int best[G];
#pragma unroll
    for (int g = 0; g < G; ++g) best[g] = 129;  // min Hamming so far (129 = none)
    for (int64_t r = r0; r < r1; r += 32) {
      const uint4 mine = __ldg(rows + r + lane);
      __syncwarp();
      slab[warp][lane] = mine;
      __syncwarp();
#pragma unroll 8
      for (int i = 0; i < 32; ++i) {
        const uint4 d = slab[warp][i];
        const uint32_t ds = d.x ^ d.y ^ d.z;
#pragma unroll
        for (int g = 0; g < G; ++g) {
          const uint32_t x0 = d.x ^ q[g].x, x1 = d.y ^ q[g].y, x2 = d.z ^ q[g].z;
          const uint32_t c = (x0 & x1) | (x2 & (x0 | x1));  // majority: one LOP3
          const int ham = __popc(ds ^ qs[g]) + 2 * __popc(c) + __popc(d.w ^ q[g].w);
          best[g] = min(best[g], ham);
        }
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int gg = g_base + g;
      if (gg >= n_groups) break;
      int v = (r1 > r0 && lane < ntok[g]) ? (128 - best[g]) : 0;  // empty page -> 0 (COALESCE)
      v = warp_sum(v);
      if (lane == 0 && (live_page || !by_page)) group_scores[int64_t(gg) * ld + (by_page ? pg : p)] = v;
    }
  }
}

int launch_score_b1(b200ms_t* h, const CorpusView& c, const int64_t* cand_ids, int64_t n_cand, const void* q_packed,
                    int n_groups, const int32_t* group_ntok_dev, void* group_scores, int64_t ld, cudaStream_t s, int g_lo,
                    int g_hi, const UnitPlan* scan) {
  const int32_t* n_dev = nullptr;
  if (scan && !cand_ids) {
    cand_ids = scan->pages;
    n_dev = scan->n_pages_dev;
  }
  const int by_page = n_dev != nullptr;
  const int64_t n_items = cand_ids && !by_page ? n_cand : c.n_pages;
  if (n_items == 0 || n_groups == 0) return B200MS_OK;
  int64_t want = (n_items + kB1Warps - 1) / kB1Warps;
  const int64_t cap = int64_t(h->num_sms) * 8;
  const int grid = int(want < cap ? want : cap);
  const uint4* rows = static_cast<const uint4*>(c.rows);
  const int64_t* ps = c.page_start;
  const uint4* qb = static_cast<const uint4*>(q_packed);
  int32_t* out = static_cast<int32_t*>(group_scores);
  // groups [g_lo, g_hi) only (the batched rerank scores each query against its own candidate list)
  if (g_hi > n_groups) g_hi = n_groups;
  n_groups = g_hi;  // the kernels treat groups >= n_groups as absent
  for (int base = g_lo; base < g_hi;) {
    const int rem = g_hi - base;
    if (rem >= 8) {
      maxsim_b1_kernel<8><<<grid, kB1Warps * 32, 0, s>>>(rows, ps, n_items, cand_ids, n_dev, by_page, c.n_pages, qb, group_ntok_dev, base, n_groups, out, ld);
      base += 8;
    } else if (rem >= 4) {
      maxsim_b1_kernel<4><<<grid, kB1Warps * 32, 0, s>>>(rows, ps, n_items, cand_ids, n_dev, by_page, c.n_pages, qb, group_ntok_dev, base, n_groups, out, ld);
      base += 4;
    } else if (rem >= 2) {
      maxsim_b1_kernel<2><<<grid, kB1Warps * 32, 0, s>>>(rows, ps, n_items, cand_ids, n_dev, by_page, c.n_pages, qb, group_ntok_dev, base, n_groups, out, ld);
      base += 2;
    } else {
      maxsim_b1_kernel<1><<<grid, kB1Warps * 32, 0, s>>>(rows, ps, n_items, cand_ids, n_dev, by_page, c.n_pages, qb, group_ntok_dev, base, n_groups, out, ld);
      base += 1;
    }
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch maxsim_b1")) return e;
  }
  return B200MS_OK;
}

}  // namespace bms
