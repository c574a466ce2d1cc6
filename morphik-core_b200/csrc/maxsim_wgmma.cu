// maxsim_wgmma.cu -- the bf16, int8, fp8 and 1-bit MaxSim scorers on Hopper (sm_90a) warpgroup MMA.
//
// Replaces the reference's float scorer  einsum("bnd,csd->bcns").max(3).sum(2)  (colpali_engine score_multi_vector,
// called at core/vector_store/fast_multivector_store.py:553-555) and the SQL public.max_sim of the 1-bit path
// (core/vector_store/multi_vector_store.py:287-311).  The [B_q, C, T, P] similarity tensor is never materialised: each
// 64 x 128 (query tokens x patch rows) product lives only in the registers of one warpgroup.
//
// Data layout in HBM
//   corpus rows   [n_rows, 128] bf16|s8|e4m3 (or [n_rows, 16 B] sign bits), row-major, every page padded to a multiple of
//                 32 rows ("chunks") by repeating its last row; chunk_page[c] = page index of chunk c
//   work units    unit_start[u] .. unit_end[u] = chunk range of unit u, always whole pages (so no page is ever split across
//                 CTAs and the per-token running max never crosses a CTA boundary)
//   queries       [n_groups*32, 128] same dtype, each query padded with zero rows to 32-row groups; a query tile is 4 groups
//                 = 128 query tokens
//   scores        group_scores[g, p] (f32 | s32), g = 32-token group, p = page (slot_mode: candidate slot)
//
// Kernel (persistent, one CTA per SM, 384 threads, warp-specialised):
//   warpgroup 0     producer.  Dense dtypes: one thread streams 128-row patch tiles (SWIZZLE_128B TMA boxes) through an
//                   S-stage mbarrier ring.  1-bit corpora: all 128 threads fetch 16 B of sign bits per row and expand them
//                   to {0,1} bytes in the same swizzled K-major layout (thread r owns row r of the tile); e4m3 corpora: the
//                   same, 128 B of e4m3 per row widened to f16 (mma_tile.cuh says why).
//   warpgroups 1-2  MMA + epilogue.  Warpgroup e owns the resident query tiles m with m % 2 == e.  A query tile is loaded as
//                   two 64-row wgmma A blocks: block h holds tokens 16h .. 16h+15 of each of the four groups, so warp w of the
//                   warpgroup ends up holding all 32 tokens of group w (rows l/4 and l/4+8 of both blocks) and sums its
//                   group with warp shuffles only.  Per patch tile and query tile: two m64n128 wgmma chains (8 x k16 for
//                   bf16 / f16, 4 x k32 for int8), each issued before the previous one is reduced (two accumulator sets,
//                   also across query-tile and patch-tile boundaries), per-lane running maxima over the 8 columns of every
//                   chunk a lane holds, and at a page end a quad shuffle for the other 24 columns and the group's sum.
// Registers: setmaxnreg moves the producer warpgroup's share to the consumers (RegPlan).
// 1-bit:  128 - ham(q, d) = (128 - popc(q)) + <q', d'>  with q' = +1 / -1 per query bit and d' = 1 / 0 per document bit, so
//         max_r (128 - ham) = c_t + max_r <q'_t, d'_r> runs as the int8 kernel plus a per-token constant c_t (0 for padding).
#include "common.cuh"
#include "mma_tile.cuh"
#include "ptx.cuh"
#include "topk_keys.cuh"

namespace bms {

constexpr int kThreads = 384;
constexpr uint32_t kQBlockBytes = 64 * 128;  // one 64-row A block of one 128-byte panel

// Registers per thread of each warpgroup role.  __launch_bounds__(kThreads, 1) gives every thread kLaunchRegs registers;
// setmaxnreg moves them from the producer warpgroup to the two consumer warpgroups, which hold two 64-register accumulator
// sets each.  setmaxnreg.inc blocks until the CTA's pool has the registers, so budgets that overdraw the pool would hang
// the kernel: the static_assert rules that out.  One TMA thread needs 40; the fp8 widener (16 uint4 of loads per thread)
// and the 1-bit expander (a ring of 8 uint4) spill below about 90.  The budgets are the splits ptxas compiled with the
// fewest spills (none, except the consumers of the 1-bit kernel with NM = 8).
constexpr int kLaunchRegs = (65536 / kThreads) & ~7;  // 168
template <int KIND, bool BITS>
struct RegPlan {
  static constexpr int kProducer = BITS ? 104 : KIND == 2 ? 120 : 40;
  static constexpr int kConsumer = BITS ? 200 : KIND == 2 ? 192 : 232;
  static_assert(kProducer + 2 * kConsumer <= 3 * kLaunchRegs, "register budgets overdraw the CTA's pool");
};

// ------------------------------------------------------------------ 1-bit query side: bits -> +-1 int8 rows + token constants
__global__ void __launch_bounds__(256)
b1_query_expand_kernel(const uint8_t* __restrict__ q_bits /*[rows,16]*/, const int32_t* __restrict__ group_ntok, int n_rows,
                       int8_t* __restrict__ out /*[rows,128]*/, int32_t* __restrict__ tok_const /*[rows]*/) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;  // one thread per (row, byte of bits)
  const int row = idx >> 4, b = idx & 15;
  if (row >= n_rows) return;
  const bool real = (row & 31) < __ldg(group_ntok + (row >> 5));
  const uint32_t bits = q_bits[row * 16 + b];
  uint32_t lo = 0, hi = 0;  // elements 8b..8b+3 and 8b+4..8b+7 as int8 (MSB of the byte = first element)
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    lo |= (real ? (((bits >> (7 - e)) & 1u) ? 0x01u : 0xffu) : 0u) << (8 * e);
    hi |= (real ? (((bits >> (3 - e)) & 1u) ? 0x01u : 0xffu) : 0u) << (8 * e);
  }
  reinterpret_cast<uint2*>(out)[row * 16 + b] = make_uint2(lo, hi);
  if (b == 0) {
    const uint4 w = *reinterpret_cast<const uint4*>(q_bits + row * 16);
    tok_const[row] = real ? 128 - (__popc(w.x) + __popc(w.y) + __popc(w.z) + __popc(w.w)) : 0;
  }
}

// ------------------------------------------------------------------ tile iterator shared by all warp roles
// units u, u + step, u + 2 step, ... (start: the CTA's first unit and the stride of the launch, see maxsim_wgmma_kernel)
struct TileIter {
  int u, step, t, n_tiles, c0, c1;
  __device__ __forceinline__ void start(int splits, const int32_t* us, const int32_t* ue, int n_units) {
    u = blockIdx.x / splits;
    step = gridDim.x / splits;
    load(us, ue, n_units);
  }
  __device__ __forceinline__ void load(const int32_t* us, const int32_t* ue, int n_units) {
    n_tiles = 0;
    while (u < n_units) {
      c0 = __ldg(us + u);
      c1 = __ldg(ue + u);
      n_tiles = (c1 - c0 + 3) >> 2;
      if (n_tiles > 0) break;
      u += step;
    }
    t = 0;
  }
  __device__ __forceinline__ bool valid(int n_units) const { return u < n_units; }
  __device__ __forceinline__ void next(const int32_t* us, const int32_t* ue, int n_units) {
    if (++t == n_tiles) {
      u += step;
      load(us, ue, n_units);
    }
  }
  __device__ __forceinline__ int64_t row0() const { return int64_t(c0 + 4 * t) * kGroup; }
};

template <int KIND>
__device__ __forceinline__ void mma_chain(typename Kind<KIND>::Acc (&d)[64], uint32_t a_addr, uint32_t b_addr) {
  const uint64_t ad = wgmma_desc_kmajor_sw128(a_addr);
  const uint64_t bd = wgmma_desc_kmajor_sw128(b_addr);
#pragma unroll
  for (int ks = 0; ks < Kind<KIND>::kKSteps; ++ks) {  // 32 B of K per step; 4 steps per 128 B panel
    const uint32_t off = ((ks >> 2) * kSubtileBytes + (ks & 3) * 32) >> 4;
    if constexpr (KIND == 0) {
      wgmma_m64n128k16_bf16(d, ad + off, bd + off, ks != 0);
    } else if constexpr (KIND == 1) {
      wgmma_m64n128k32_s8(d, ad + off, bd + off, ks != 0);
    } else {
      wgmma_m64n128k16_f16(d, ad + off, bd + off, ks != 0);
    }
  }
  wgmma_commit();
}

// group sum of one warp: 4 token values per thread (the quad's four lanes hold the same ones), 8 quads
template <typename Acc>
__device__ __forceinline__ Acc group_sum(const Acc (&v)[4]) {
  Acc s = (v[0] + v[1]) + (v[2] + v[3]);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  s += __shfl_xor_sync(0xffffffffu, s, 8);
  s += __shfl_xor_sync(0xffffffffu, s, 16);
  return s;
}

// e4m3 query rows -> f16 rows (the A operand of the KIND 2 kernel)
__global__ void __launch_bounds__(256)
f8_query_widen_kernel(const uint2* __restrict__ q, int64_t n_words, uint4* __restrict__ out) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n_words; i += int64_t(gridDim.x) * blockDim.x) {
    const uint2 v = __ldg(q + i);
    out[i] = e4m3x8_to_f16x8(v.x, v.y);
  }
}

// Document mode (DOC): a page's per-token maxima m go to the document table instead of a group score.  Each true token t
// of the group takes atomicMax(table[32 * group + t, doc], doc_token_key(m) << 32 | ~page) when the page's document is in
// [0, n_docs) and the group's query may see the page; the key orders numbers like key_of and puts NaN between "unset" (0)
// and every number, as fmaxf lets any number beat NaN, and a tie goes to the lower page.  The atomics commute, so the table
// does not depend on the order the CTAs reach the pages.
__device__ __forceinline__ uint32_t doc_token_key(float m) { return m != m ? 1u : key_of(m); }
__device__ __forceinline__ uint32_t doc_token_key(int m) { return key_of(m); }  // m > INT32_MIN: the key is never 0

// KIND 0 bf16, 1 int8 (BITS: 1-bit corpus expanded to int8), 2 fp8 e4m3 (widened to f16 by the producer warpgroup);
// NM = resident query tiles (1, 2, 4 or 8).  The body of maxsim_wgmma_kernel (DOC = false) and maxsim_wgmma_doc_kernel.
template <int KIND, int NM, bool BITS, bool DOC>
__device__ __forceinline__ void
maxsim_wgmma_body(const CUtensorMap& tmap_rows, const CUtensorMap& tmap_q,
                  const uint4* __restrict__ bit_rows, int64_t n_rows, const int32_t* __restrict__ tok_const,
                  const int32_t* __restrict__ chunk_page, const int32_t* __restrict__ unit_start,
                  const int32_t* __restrict__ unit_end, int slot_mode, int n_units,
                  const int32_t* __restrict__ n_units_dev, int m_tile_base, int n_groups_real,
                  const int32_t* __restrict__ group_ntok, const uint32_t* __restrict__ clamp_bits, typename Kind<KIND>::Acc* __restrict__ group_scores, int64_t ld,
                  int num_stages, int splits, const DocScan& doc) {
  using K = Kind<KIND>;
  using Acc = typename K::Acc;
  static_assert(!BITS || KIND == 1, "1-bit corpora run on the int8 MMA");
  // a filtered scan's units are counted on the device (scan_plan.cu); a CTA past the count finds no tile and falls through
  if (n_units_dev) n_units = __ldg(n_units_dev);
  // splits = 2: CTAs 2k and 2k + 1 walk the same units, CTA 2k + 1 with the NM query tiles after CTA 2k's (see launch_one)
  m_tile_base += NM * int(blockIdx.x % splits);
  constexpr int NWG = NM >= 2 ? 2 : 1;   // consumer warpgroups with work
  constexpr int MPW = (NM + 1) / 2;      // query tiles per consumer warpgroup

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_q = smem;                                            // NM query tiles
  uint8_t* smem_st = smem + NM * K::kTileBytes;                      // num_stages patch tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_st + size_t(num_stages) * K::kTileBytes);
  uint64_t* full = bars;                     // [num_stages] producer -> MMA
  uint64_t* empty = bars + 16;               // [num_stages] MMA -> producer
  uint64_t* qfull = bars + 32;               // query tiles landed

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  constexpr bool kExpand = BITS || KIND == 2;  // the producer warpgroup writes the patch tiles itself
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_q);
    if constexpr (!kExpand) prefetch_tmap(&tmap_rows);
    for (int i = 0; i < num_stages; ++i) {
      mbar_init(&full[i], kExpand ? 4 : 1);  // expanding producers: one arrival per warp
      mbar_init(&empty[i], 4 * NWG);      // one arrival per consumer warp
    }
    mbar_init(qfull, 1);
    fence_mbar_init();
  }
  __syncthreads();

  using Regs = RegPlan<KIND, BITS>;
  if (warp < 4) {
    // ================================================================ producer warpgroup
    if constexpr (Regs::kProducer > 0) setmaxnreg_dec<Regs::kProducer>();
    if (threadIdx.x == 0) {
      // query tile m, block h, group g: rows 32g + 16h .. +16 of the tile -> rows 16g .. 16g+15 of A block h
      const uint64_t pol_q = policy_evict_last();
      mbar_expect_tx(qfull, NM * K::kTileBytes);
      for (int m = 0; m < NM; ++m)
        for (int p = 0; p < K::kPanels; ++p)
          for (int hb = 0; hb < 2; ++hb)
            for (int g = 0; g < 4; ++g)
              tma_load_2d(&tmap_q, qfull, smem_q + m * K::kTileBytes + p * kSubtileBytes + hb * kQBlockBytes + g * 2048,
                          p * K::kPanelElems, (m_tile_base + m) * kTileM + 32 * g + 16 * hb, pol_q);
    }
    if constexpr (!kExpand) {
      if (threadIdx.x == 0) {
        // a patch tile read by both CTAs of a split pair stays in L2 for the second read
        const uint64_t pol_rows = splits > 1 ? policy_evict_normal() : policy_evict_first();
        int stage = 0;
        uint32_t phase = 0;
        TileIter it;
        it.start(splits, unit_start, unit_end, n_units);
        for (; it.valid(n_units); it.next(unit_start, unit_end, n_units)) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], K::kTileBytes);
          uint8_t* dst = smem_st + size_t(stage) * K::kTileBytes;
#pragma unroll
          for (int p = 0; p < K::kPanels; ++p)
            tma_load_2d(&tmap_rows, &full[stage], dst + p * kSubtileBytes, p * K::kPanelElems, int32_t(it.row0()), pol_rows);
          if (++stage == num_stages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    } else if constexpr (KIND == 2) {
      // widening: e4m3 rows -> f16, swizzled K-major, two 64-element panels; thread r owns row r of the tile and keeps the
      // loads of the next tile in flight while it converts the current one
      const int r = threadIdx.x;
      const uint32_t row_off = uint32_t(r >> 3) * 1024u + uint32_t(r & 7) * 128u;
      const uint32_t sw = uint32_t(r & 7);
      const uint4* rows16 = reinterpret_cast<const uint4*>(bit_rows);  // [n_rows, 8] x 16 B
      TileIter cur, pf;
      cur.start(splits, unit_start, unit_end, n_units);
      pf = cur;
      uint4 nxt[8];
      auto fetch = [&](uint4 (&v)[8]) {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = make_uint4(0, 0, 0, 0);
        if (pf.valid(n_units)) {
          const int64_t row = pf.row0() + r;
          if (row < n_rows) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = __ldg(rows16 + row * 8 + i);
          }
          pf.next(unit_start, unit_end, n_units);
        }
      };
      fetch(nxt);
      int stage = 0;
      uint32_t phase = 0;
      while (cur.valid(n_units)) {
        uint4 mine[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) mine[i] = nxt[i];
        fetch(nxt);
        mbar_wait(&empty[stage], phase ^ 1);
        const uint32_t tile = smem_u32(smem_st) + uint32_t(stage) * K::kTileBytes + row_off;
#pragma unroll
        for (int i = 0; i < 8; ++i) {  // elements 16i .. 16i+15 -> f16 chunks 2i, 2i+1 (panel 2i / 8)
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const uint32_t c = uint32_t(2 * i + hh);
            const uint4 o = hh == 0 ? e4m3x8_to_f16x8(mine[i].x, mine[i].y) : e4m3x8_to_f16x8(mine[i].z, mine[i].w);
            st_shared_v4(tile + (c >> 3) * kSubtileBytes + (((c & 7) ^ sw) << 4), o);
          }
        }
        fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core's async-proxy reads
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[stage]);
        if (++stage == num_stages) {
          stage = 0;
          phase ^= 1;
        }
        cur.next(unit_start, unit_end, n_units);
      }
    } else {
      // expanders: packed bits -> {0,1} int8, swizzled K-major; loads of the next 8 tiles stay in flight meanwhile
      const int r = threadIdx.x;  // row of the tile this thread owns
      const uint32_t row_off = uint32_t(r >> 3) * 1024u + uint32_t(r & 7) * 128u;
      const uint32_t sw = uint32_t(r & 7);
      TileIter cur, pf;
      cur.start(splits, unit_start, unit_end, n_units);
      pf = cur;
      constexpr int kRing = 8;
      uint4 ring[kRing];
#pragma unroll
      for (int i = 0; i < kRing; ++i) {
        ring[i] = make_uint4(0, 0, 0, 0);
        if (pf.valid(n_units)) {
          const int64_t row = pf.row0() + r;
          if (row < n_rows) ring[i] = __ldg(bit_rows + row);
          pf.next(unit_start, unit_end, n_units);
        }
      }
      int stage = 0;
      uint32_t phase = 0;
      while (cur.valid(n_units)) {
#pragma unroll
        for (int i = 0; i < kRing; ++i) {
          if (!cur.valid(n_units)) break;
          const uint4 mine = ring[i];
          ring[i] = make_uint4(0, 0, 0, 0);
          if (pf.valid(n_units)) {
            const int64_t row = pf.row0() + r;
            if (row < n_rows) ring[i] = __ldg(bit_rows + row);
            pf.next(unit_start, unit_end, n_units);
          }
          mbar_wait(&empty[stage], phase ^ 1);
          const uint32_t tile = smem_u32(smem_st) + uint32_t(stage) * K::kTileBytes + row_off;
          const uint32_t words[4] = {mine.x, mine.y, mine.z, mine.w};
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            // __brev: bit e%8 of (reversed) byte 3-b now holds element 8b + e%8 of this word's 32 elements
            const uint32_t rev = __brev(words[w]);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {  // 16-byte chunk c = 2w + hh  <-  source bytes 2hh, 2hh+1 of the word
              // nibble n (bit e = element e) * 0x204081 puts bit k at k, k+7, k+14, k+21; masked with 0x01010101 that is
              // one element per byte.  (Only valid for 4-bit inputs: with 8 bits the shifted copies overlap and carry.)
              const uint32_t b0 = (rev >> (8 * (3 - 2 * hh))) & 0xffu, b1 = (rev >> (8 * (2 - 2 * hh))) & 0xffu;
              uint4 o;
              o.x = ((b0 & 0xfu) * 0x00204081u) & 0x01010101u;
              o.y = ((b0 >> 4) * 0x00204081u) & 0x01010101u;
              o.z = ((b1 & 0xfu) * 0x00204081u) & 0x01010101u;
              o.w = ((b1 >> 4) * 0x00204081u) & 0x01010101u;
              const uint32_t c = uint32_t(2 * w + hh);
              st_shared_v4(tile + ((c ^ sw) << 4), o);
            }
          }
          fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core's async-proxy reads
          __syncwarp();
          if (lane == 0) mbar_arrive(&full[stage]);
          if (++stage == num_stages) {
            stage = 0;
            phase ^= 1;
          }
          cur.next(unit_start, unit_end, n_units);
        }
      }
    }
    return;
  }

  // ================================================================ consumer warpgroups: MMA + epilogue
  const int wg = (warp >> 2) - 1;
  const int w = warp & 3;  // group w of every query tile this warpgroup owns
  if (wg >= NWG) return;
  if constexpr (Regs::kConsumer > 0) setmaxnreg_inc<Regs::kConsumer>();
  mbar_wait(qfull, 0);
  const uint32_t q_addr = smem_u32(smem_q);
  const uint32_t st_addr = smem_u32(smem_st);
  // A block of query tile i of this warpgroup (tile m = wg + 2i < NM for every i < MPW)
  auto a_block = [&](int i) { return q_addr + uint32_t(wg + 2 * i) * K::kTileBytes; };

  // runmax: this lane's running max of its 8 columns per chunk, per (query tile, token); the quad's four lanes together
  // hold the token's max, combined at flush.
  Acc runmax[MPW][4];
#pragma unroll
  for (int i = 0; i < MPW; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) runmax[i][k] = Acc(0);

  // score of page `page` (unit u in slot_mode) for the group of query tile i; page < 0: nothing accumulated yet.  Only the
  // group's true tokens count (group_ntok; NULL: all 32): a zero padding row's max is NaN on a page whose rows all hold an
  // infinity (0 * inf), not 0.
  auto flush = [&](int i, int u, int page) {
    const int mt = m_tile_base + wg + 2 * i;
    const int group = mt * 4 + w;
    if (group < n_groups_real && page >= 0) {
      const int o = slot_mode ? u : page;
      const int ntok = group_ntok ? __ldg(group_ntok + group) : kGroup;
      if constexpr (DOC) {
        // the page's document and whether the group's query may see the page; then one atomic per true token, from the
        // quad's first lane.  A 1-bit token's constant c_t is left out: it moves neither the max nor the arg-max, and
        // doc_maxsim.cu adds it when it reads the table.
        const int d = __ldg(doc.page_doc + page);
        bool ok = d >= 0 && d < doc.n_docs;
        if (ok && doc.allow) {
          const int mi = doc.mask_index ? __ldg(doc.mask_index + __ldg(doc.group_query + group)) : 0;
          ok = mi < 0 || ((__ldg(doc.allow + int64_t(mi) * doc.mask_stride + (page >> 5)) >> (page & 31)) & 1u);
        }
        // 32-bit entry index: a table holds at most kDocTableBytes / 8 = 2^27 entries
        const uint32_t nd = uint32_t(doc.n_docs);
        const uint32_t row = uint32_t(group * kGroup + (lane >> 2)) * nd + uint32_t(d);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int tok = 16 * (k >> 1) + 8 * (k & 1) + (lane >> 2);
          const Acc m = quad_max(runmax[i][k]);
          if (ok && (lane & 3) == 0 && tok < ntok)
            atomicMax(doc.table + (row + uint32_t(tok - (lane >> 2)) * nd),
                      (uint64_t(doc_token_key(m)) << 32) | uint64_t(~uint32_t(page)));
        }
      } else {
        Acc v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          Acc cnst = Acc(0);
          // token k of this thread: 16 * (k >> 1) + 8 * (k & 1) + lane / 4 of group w; read here, not held in registers
          const int tok = 16 * (k >> 1) + 8 * (k & 1) + (lane >> 2);
          if constexpr (BITS) cnst = __ldg(tok_const + int64_t(mt) * kTileM + 32 * w + tok);
          const Acc m = clamp_token_max(clamp_bits, o, quad_max(runmax[i][k])) + cnst;
          v[k] = tok < ntok ? m : Acc(0);
        }
        const Acc s = group_sum(v);
        if (lane == 0) group_scores[int64_t(group) * ld + o] = s;
      }
    }
  };

  // The warpgroup's wgmma blocks form one stream: per patch tile, per query tile i, the A blocks h = 0 and h = 1.  Every
  // tile holds an even number of blocks, so block h always accumulates in acc0 (h = 0) or acc1 (h = 1).  The next block's
  // chain is issued before the current block is reduced, also across query-tile and patch-tile boundaries, so the
  // warpgroup keeps a chain on the tensor pipe while it runs its epilogue.  The next tile's first chain is retired at the end of the iteration, after the
  // last block's epilogue and the next tile's bookkeeping: ptxas serialises every wgmma of a loop that carries a pending
  // wgmma group across its back-edge.
  Acc acc0[64], acc1[64];
  int stage = 0;
  uint32_t phase = 0;
  int last_u = -1;
  int cur_page = -1;  // page of the running maxima (the same for every query tile: all walk the same chunks)
  int pg[4];          // page of each chunk of the tile; -1: past the end of the unit
  bool same = false;  // all four chunks continue cur_page (the common case)
  TileIter it;
  it.start(splits, unit_start, unit_end, n_units);
  auto begin_tile = [&]() {
    if (it.u != last_u) {  // new unit: units end on page boundaries
#pragma unroll
      for (int i = 0; i < MPW; ++i) flush(i, last_u, cur_page);
      cur_page = -1;
      last_u = it.u;
    }
    const int cb = it.c0 + 4 * it.t;
#pragma unroll
    for (int j = 0; j < 4; ++j) pg[j] = (cb + j < it.c1) ? __ldg(chunk_page + cb + j) : -1;
    same = pg[0] == cur_page && pg[1] == cur_page && pg[2] == cur_page && pg[3] == cur_page;
  };
  // Every chain is issued unconditionally, the ones past the last tile included (their results are dropped and no producer
  // writes a stage any more by then): a chain on a data-dependent path also makes ptxas serialise the wgmmas.
  if (it.valid(n_units)) {
    begin_tile();
    mbar_wait(&full[0], 0);
  }
  wgmma_fence();
  mma_chain<KIND>(acc0, a_block(0), st_addr);
  wgmma_wait<0>();
  while (it.valid(n_units)) {
    TileIter nx = it;
    nx.next(unit_start, unit_end, n_units);
    int nstage = stage + 1;
    uint32_t nphase = phase;
    if (nstage == num_stages) {
      nstage = 0;
      nphase ^= 1;
    }
    const uint32_t b_addr = st_addr + uint32_t(stage) * K::kTileBytes;
#pragma unroll
    for (int i = 0; i < MPW; ++i) {
      Acc cm[4][4];  // [token k][chunk]: this lane's partial maxima
      wgmma_fence();
      mma_chain<KIND>(acc1, a_block(i) + kQBlockBytes, b_addr);
      wgmma_wait<1>();
      reg_fence_all(acc0);
      chunk_maxima(acc0, cm[0], cm[1]);
      if (i + 1 < MPW) {
        wgmma_fence();
        mma_chain<KIND>(acc0, a_block(i + 1), b_addr);
      } else {  // the next tile's first block
        if (nx.valid(n_units)) mbar_wait(&full[nstage], nphase);
        wgmma_fence();
        mma_chain<KIND>(acc0, a_block(0), st_addr + uint32_t(nstage) * K::kTileBytes);
      }
      wgmma_wait<1>();
      reg_fence_all(acc1);
      if (i == MPW - 1) {  // every read of this stage has completed
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
      }
      chunk_maxima(acc1, cm[2], cm[3]);
      if (same) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          runmax[i][k] = acc_max(acc_max(runmax[i][k], acc_max(cm[k][0], cm[k][1])), acc_max(cm[k][2], cm[k][3]));
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (pg[j] < 0) continue;  // chunk belongs to the next unit
          const int prev = j == 0 ? cur_page : pg[j - 1];
          if (pg[j] != prev) {
            flush(i, it.u, prev);
#pragma unroll
            for (int k = 0; k < 4; ++k) runmax[i][k] = cm[k][j];
          } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) runmax[i][k] = acc_max(runmax[i][k], cm[k][j]);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (pg[j] >= 0) cur_page = pg[j];
    it = nx;
    stage = nstage;
    phase = nphase;
    if (it.valid(n_units)) begin_tile();
    wgmma_wait<0>();
  }
#pragma unroll
  for (int i = 0; i < MPW; ++i) flush(i, last_u, cur_page);
}

#define MAXSIM_WGMMA_PARAMS                                                                                                  \
  const __grid_constant__ CUtensorMap tmap_rows, const __grid_constant__ CUtensorMap tmap_q,                              \
      const uint4* __restrict__ bit_rows, int64_t n_rows, const int32_t* __restrict__ tok_const,                             \
      const int32_t* __restrict__ chunk_page, const int32_t* __restrict__ unit_start, const int32_t* __restrict__ unit_end, \
      int slot_mode, int n_units, const int32_t* __restrict__ n_units_dev, int m_tile_base, int n_groups_real,              \
      const int32_t* __restrict__ group_ntok, const uint32_t* __restrict__ clamp_bits,                                     \
      typename Kind<KIND>::Acc* __restrict__ group_scores, int64_t ld, int num_stages, int splits
#define MAXSIM_WGMMA_ARGS                                                                                                   \
  tmap_rows, tmap_q, bit_rows, n_rows, tok_const, chunk_page, unit_start, unit_end, slot_mode, n_units, n_units_dev,      \
      m_tile_base, n_groups_real, group_ntok, clamp_bits, group_scores, ld, num_stages, splits

template <int KIND, int NM, bool BITS>
__global__ void __launch_bounds__(kThreads, 1) maxsim_wgmma_kernel(MAXSIM_WGMMA_PARAMS) {
  maxsim_wgmma_body<KIND, NM, BITS, false>(MAXSIM_WGMMA_ARGS, DocScan{});
}

// document mode: no group_scores (NULL), no clamp (clamp_bits NULL), full-scan units (slot_mode 0)
template <int KIND, int NM, bool BITS>
__global__ void __launch_bounds__(kThreads, 1) maxsim_wgmma_doc_kernel(MAXSIM_WGMMA_PARAMS, const DocScan doc) {
  maxsim_wgmma_body<KIND, NM, BITS, true>(MAXSIM_WGMMA_ARGS, doc);
}

// ---------------------------------------------------------------------------------------------- host side
// Query tiles [m_tile_base, m_tile_base + splits * NM) in one launch.  splits = 2: CTAs 2k and 2k + 1 walk the same units,
// CTA 2k with the first NM tiles and CTA 2k + 1 with the next NM, so the pair reads every patch tile from HBM once and
// the second read hits L2 -- two back-to-back passes over the corpus would read it from HBM twice.
template <int KIND, int NM, bool BITS>
static int launch_one(b200ms_t* h, const CorpusView& c, const UnitPlan& up, const CUtensorMap& tq, const int32_t* tok_const,
                      const int32_t* group_ntok, int m_tile_base, int n_groups_real, void* scores, int64_t ld, cudaStream_t s,
                      const DocScan* doc, int splits = 1) {
  using K = Kind<KIND>;
  const uint32_t avail = kSmemLimit - 1024 /*align*/ - kBarrierBytes - NM * K::kTileBytes;
  int stages = int(avail / K::kTileBytes);
  if (stages > 8) stages = 8;
  if (stages < 2) return set_error(h, B200MS_EINVAL, "maxsim_wgmma: not enough shared memory for 2 stages");
  const uint32_t smem = 1024 + NM * K::kTileBytes + uint32_t(stages) * K::kTileBytes + kBarrierBytes;
  const void* fn = doc ? reinterpret_cast<const void*>(maxsim_wgmma_doc_kernel<KIND, NM, BITS>)
                       : reinterpret_cast<const void*>(maxsim_wgmma_kernel<KIND, NM, BITS>);
  if (int e = ensure_smem(h, fn, int(smem), "cudaFuncSetAttribute(maxsim_wgmma)")) return e;
  int grid = h->max_ctas > 0 ? h->max_ctas : h->num_sms;
  if (grid > splits * up.n_units) grid = splits * up.n_units;  // with n_units_dev an upper bound: the count is not known here
  grid -= grid % splits;
  if (grid < 1) return B200MS_OK;
  static const CUtensorMap kNoTmap{};  // 1-bit rows: the producer expands bits and never issues TMA loads for them
  if (doc)
    maxsim_wgmma_doc_kernel<KIND, NM, BITS><<<grid, kThreads, smem, s>>>(
        c.tmap ? *c.tmap : kNoTmap, tq, static_cast<const uint4*>(c.rows), c.n_rows, tok_const, c.chunk_page, up.start, up.end,
        0, up.n_units, up.n_units_dev, m_tile_base, n_groups_real, group_ntok, nullptr, nullptr, 0, stages, splits, *doc);
  else
    maxsim_wgmma_kernel<KIND, NM, BITS><<<grid, kThreads, smem, s>>>(
        c.tmap ? *c.tmap : kNoTmap, tq, static_cast<const uint4*>(c.rows), c.n_rows, tok_const, c.chunk_page, up.start, up.end,
        up.slot_mode, up.n_units, up.n_units_dev, m_tile_base, n_groups_real, group_ntok, up.clamp_bits,
        static_cast<typename K::Acc*>(scores), ld, stages, splits);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch maxsim_wgmma");
}

// Query tiles [base, base + nm) in one pass over the corpus.  nm is rounded up to a power of two: a phantom (all-zero) tile
// costs less than a second pass over the corpus.  Two full passes' worth of tiles run as one split launch (launch_one) when
// the grid holds a pair of CTAs.
template <int KIND, bool BITS>
static int launch_tiles(b200ms_t* h, const CorpusView& c, const UnitPlan& up, const CUtensorMap& tq, const int32_t* tok_const,
                        const int32_t* group_ntok, int n_groups_real, int m_lo, int m_hi, void* scores, int64_t ld, cudaStream_t s,
                        const DocScan* doc = nullptr) {
  constexpr int kMaxNM = Kind<KIND>::kMaxNM;
  const bool pairs = (h->max_ctas > 0 ? h->max_ctas : h->num_sms) >= 2;
  for (int base = m_lo; base < m_hi;) {
    const int rem = m_hi - base;
    if (pairs && rem >= 2 * kMaxNM) {
      if (int e = launch_one<KIND, kMaxNM, BITS>(h, c, up, tq, tok_const, group_ntok, base, n_groups_real, scores, ld, s, doc, 2)) return e;
      base += 2 * kMaxNM;
      continue;
    }
    int nm = 1;
    while (nm < rem && nm < kMaxNM) nm <<= 1;
    int e;
    switch (nm) {
      case 1: e = launch_one<KIND, 1, BITS>(h, c, up, tq, tok_const, group_ntok, base, n_groups_real, scores, ld, s, doc); break;
      case 2: e = launch_one<KIND, 2, BITS>(h, c, up, tq, tok_const, group_ntok, base, n_groups_real, scores, ld, s, doc); break;
      case 4: e = launch_one<KIND, 4, BITS>(h, c, up, tq, tok_const, group_ntok, base, n_groups_real, scores, ld, s, doc); break;
      default:
        if constexpr (kMaxNM >= 8) {
          e = launch_one<KIND, 8, BITS>(h, c, up, tq, tok_const, group_ntok, base, n_groups_real, scores, ld, s, doc);
        } else {
          e = set_error(h, B200MS_EINVAL, "maxsim_wgmma: bad NM");
        }
    }
    if (e) return e;
    base += nm;
  }
  return B200MS_OK;
}

// query rows as 16-row TMA boxes (two per group and A block, see the kernel); re-encoded only when (pointer, dtype, rows) change
static int query_tmap(b200ms_t* h, const void* q, int dtype, int n_q_rows) {
  if (h->tmap_q_base == q && h->tmap_q_dtype == dtype && h->tmap_q_rows == n_q_rows) return B200MS_OK;
  if (int e = make_tmap_rows(h, &h->tmap_q, q, dtype, int64_t(n_q_rows), 16)) return e;
  h->tmap_q_base = q;
  h->tmap_q_dtype = dtype;
  h->tmap_q_rows = n_q_rows;
  return B200MS_OK;
}

// m_tile_lo / m_tile_hi: score only query tiles [m_tile_lo, m_tile_hi) (hi < 0: all) -- the batched rerank walks the query
// tiles one launch at a time, each against its own candidate units.
int launch_score_wgmma(b200ms_t* h, const CorpusView& c, const UnitPlan& up, const void* q_packed, int n_groups_real,
                       const int32_t* group_ntok, void* group_scores, int64_t ld, cudaStream_t s, int m_tile_lo, int m_tile_hi,
                       const DocScan* doc) {
  if (!c.tmap) return set_error(h, B200MS_ESTATE, "score: corpus has no TMA descriptor");
  const int n_groups_padded = int(groups_padded(n_groups_real));
  const int n_mtiles = n_groups_padded / 4;
  const int n_q_rows = n_groups_padded * kGroup;
  if (c.dtype == B200MS_F8) {  // the A operand of the f16 MMA: the e4m3 query rows widened to f16
    if (int e = reserve(h, h->f8_q_f16, size_t(n_q_rows) * 256 + 1024)) return e;
    void* wide = reinterpret_cast<void*>((reinterpret_cast<uintptr_t>(h->f8_q_f16.p) + 1023) & ~uintptr_t(1023));
    const int64_t n_words = int64_t(n_q_rows) * 16;
    f8_query_widen_kernel<<<int((n_words + 255) / 256 < 4 * h->num_sms ? (n_words + 255) / 256 : 4 * h->num_sms), 256, 0, s>>>(
        static_cast<const uint2*>(q_packed), n_words, static_cast<uint4*>(wide));
    h->launches++;
    if (int e = check_cuda(h, cudaGetLastError(), "launch f8_query_widen")) return e;
    if (int e = query_tmap(h, wide, B200MS_BF16, n_q_rows)) return e;  // any 2-byte element type: TMA only copies
  } else if (int e = query_tmap(h, q_packed, c.dtype, n_q_rows)) {
    return e;
  }
  int lo = 0, hi = n_mtiles;
  if (m_tile_hi >= 0) {
    lo = m_tile_lo;
    hi = m_tile_hi < n_mtiles ? m_tile_hi : n_mtiles;
  }
  switch (kind_of_dtype(c.dtype)) {
    case 0: return launch_tiles<0, false>(h, c, up, h->tmap_q, nullptr, group_ntok, n_groups_real, lo, hi, group_scores, ld, s, doc);
    case 1: return launch_tiles<1, false>(h, c, up, h->tmap_q, nullptr, group_ntok, n_groups_real, lo, hi, group_scores, ld, s, doc);
    case 2: return launch_tiles<2, false>(h, c, up, h->tmap_q, nullptr, group_ntok, n_groups_real, lo, hi, group_scores, ld, s, doc);
    default: return set_error(h, B200MS_ESTATE, "score: corpus dtype has no wgmma scorer");
  }
}

int reserve_b1_query(b200ms_t* h, int64_t n_rows, int8_t** q_i8, int32_t** tok_const) {
  if (int e = reserve(h, h->b1_q_i8, size_t(n_rows) * 128 + 1024)) return e;
  if (int e = reserve(h, h->b1_tok_const, size_t(n_rows) * 4)) return e;
  *q_i8 = reinterpret_cast<int8_t*>((reinterpret_cast<uintptr_t>(h->b1_q_i8.p) + 1023) & ~uintptr_t(1023));
  *tok_const = static_cast<int32_t*>(h->b1_tok_const.p);
  return B200MS_OK;
}

int launch_b1_tiles(b200ms_t* h, const CorpusView& v, const UnitPlan& plan, const int8_t* q_i8, const int32_t* tok_const,
                    int n_groups_real, void* group_scores, int64_t ld, cudaStream_t s, const int32_t* group_ntok,
                    const DocScan* doc) {
  const int n_groups_padded = int(groups_padded(n_groups_real));
  if (int e = query_tmap(h, q_i8, B200MS_I8, n_groups_padded * kGroup)) return e;
  return launch_tiles<1, true>(h, v, plan, h->tmap_q, tok_const, group_ntok, n_groups_real, 0, n_groups_padded / 4, group_scores,
                               ld, s, doc);
}

// 1-bit full scan: the query bits become +-1 int8 rows (b1_q_i8) and per-token constants, then the int8 kernel with the
// expanding producer.
int launch_score_b1_wgmma(b200ms_t* h, const UnitPlan& plan, const void* q_bits, const int32_t* group_ntok_dev,
                          int n_groups_real, void* group_scores, int64_t ld, cudaStream_t s, const DocScan* doc) {
  const int n_rows = int(groups_padded(n_groups_real)) * kGroup;
  int8_t* q_i8 = nullptr;
  int32_t* tok_const = nullptr;
  if (int e = reserve_b1_query(h, n_rows, &q_i8, &tok_const)) return e;
  b1_query_expand_kernel<<<(n_rows * 16 + 255) / 256, 256, 0, s>>>(static_cast<const uint8_t*>(q_bits), group_ntok_dev, n_rows,
                                                                  q_i8, tok_const);
  h->launches++;
  if (int e = check_cuda(h, cudaGetLastError(), "launch b1_query_expand")) return e;
  return launch_b1_tiles(h, corpus_view(h), plan, q_i8, tok_const, n_groups_real, group_scores, ld, s,
                         doc ? group_ntok_dev : nullptr, doc);
}

}  // namespace bms
