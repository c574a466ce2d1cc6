// row_tiles.cuh -- one 64-row block of packed rows (the wgmma A operand) against every 128-row tile of a page (B), on the
// scan's own tensor-core instructions (mma_tile.cuh): bf16 k16 / fp32, s8 k32 / int32, e4m3 widened to f16 k16 / fp32, in
// the scan's K order, so every row x row product is the value the scan takes its max over, bit for bit.
//
// Used by b200ms_explain_device (A = 64 query tokens, maxsim_explain.cu) and b200ms_mmr_device (A = 64 rows of a candidate
// page, B = the page picked last, maxsim_mmr.cu).  One warpgroup (128 threads) runs it; thread r stages row r of every B tile
// with plain 16-byte loads, the next tile in flight while the current one is on the tensor pipe.  Shared memory: the B tile
// ([kPanels][128 rows x 128 B]) at b_addr, the A block ([kPanels][64 rows x 128 B]) right behind it, both 1024-byte aligned.
#pragma once
#include "common.cuh"
#include "mma_tile.cuh"
#include "ptx.cuh"

namespace bms {

constexpr int kRowTileThreads = 128;         // one warpgroup
constexpr int kABlockRows = 64;              // rows of the A block (one wgmma M block)
constexpr uint32_t kABlockPanel = 64 * 128;  // one 128-byte K panel of the 64-row A block

// dynamic shared memory a kernel that runs rows_vs_page_tiles<KIND> asks for (B tile + A block + alignment slack)
template <int KIND>
constexpr int row_tiles_smem() {
  return 1024 + 3 * Kind<KIND>::kPanels * int(kABlockPanel);
}

// one 128-byte-row K-major SWIZZLE_128B atom: row r, 16-byte chunk c (0..7) of a panel
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return uint32_t(r >> 3) * 1024u + uint32_t(r & 7) * 128u + ((uint32_t(c) ^ uint32_t(r & 7)) << 4);
}

// 16-byte piece c of a stored row -> shared memory (e4m3: two f16 pieces)
template <int KIND>
__device__ __forceinline__ void put_piece(uint32_t base, uint32_t panel_bytes, int row, int c, const uint4& v) {
  if constexpr (KIND == 2) {
    const uint4 lo = e4m3x8_to_f16x8(v.x, v.y), hi = e4m3x8_to_f16x8(v.z, v.w);
    st_shared_v4(base + uint32_t((2 * c) >> 3) * panel_bytes + sw128_off(row, (2 * c) & 7), lo);
    st_shared_v4(base + uint32_t((2 * c + 1) >> 3) * panel_bytes + sw128_off(row, (2 * c + 1) & 7), hi);
  } else {
    st_shared_v4(base + uint32_t(c >> 3) * panel_bytes + sw128_off(row, c & 7), v);
  }
}

// 16-byte pieces of one stored row
template <int KIND>
constexpr int row_chunks() {
  return KIND == 0 ? 16 : 8;
}

// rows [row0, row0 + 64) of `rows` -> the A block; a row at or past `limit` (the end of what `rows` holds) is zero
template <int KIND>
__device__ __forceinline__ void load_a_block(uint32_t a_addr, const uint4* rows, int64_t row0, int64_t limit) {
  constexpr int kSrcChunks = row_chunks<KIND>();
  constexpr int kPieces = kABlockRows * kSrcChunks / kRowTileThreads;
#pragma unroll
  for (int k = 0; k < kPieces; ++k) {
    const int p = int(threadIdx.x) + k * kRowTileThreads;
    const int row = p / kSrcChunks, c = p % kSrcChunks;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row0 + row < limit) v = __ldg(rows + (row0 + row) * kSrcChunks + c);
    put_piece<KIND>(a_addr, kABlockPanel, row, c, v);
  }
}

// The tile loop.  B = rows [row0, row0 + padded) of `prows` (padded: the page's rows rounded up to 32; rows past it are
// zero), in tiles of 128.  Fetches tile 0, waits until the previous work item's wgmmas have read shared memory, runs
// load_a() (which fills the A block), then per tile n: one m64n128 chain over the 128-d rows and epi(d, n) with the
// accumulators d (ptx.cuh fragment layout: d[4 jb + 2 h + e] is A row 16 warp + lane/4 + 8 h, B row 128 n + 8 jb +
// 2 (lane & 3) + e).  Every thread of the warpgroup calls it with the same arguments.
template <int KIND, class LoadA, class Epi>
__device__ __forceinline__ void rows_vs_page_tiles(uint32_t a_addr, uint32_t b_addr, const uint4* prows, int64_t row0,
                                                   int padded, LoadA&& load_a, Epi&& epi) {
  using K = Kind<KIND>;
  using Acc = typename K::Acc;
  constexpr int kSrcChunks = row_chunks<KIND>();
  const int r = threadIdx.x;  // B: row r of every page tile
  const int n_tiles = (padded + kTileN - 1) / kTileN;
  uint4 nxt[kSrcChunks];
  auto fetch = [&](int n) {
    const int row = n * kTileN + r;
#pragma unroll
    for (int c = 0; c < kSrcChunks; ++c) nxt[c] = make_uint4(0, 0, 0, 0);
    if (row < padded) {
#pragma unroll
      for (int c = 0; c < kSrcChunks; ++c) nxt[c] = __ldg(prows + (row0 + row) * kSrcChunks + c);
    }
  };
  fetch(0);
  __syncthreads();  // the previous item's wgmmas have read the A block
  load_a();
  for (int n = 0; n < n_tiles; ++n) {
    if (n > 0) __syncthreads();  // the previous tile's wgmmas have read the B tile
#pragma unroll
    for (int c = 0; c < kSrcChunks; ++c) put_piece<KIND>(b_addr, kSubtileBytes, r, c, nxt[c]);
    fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core's async-proxy reads
    __syncthreads();
    Acc d[64];
    wgmma_fence();
    {
      const uint64_t ad = wgmma_desc_kmajor_sw128(a_addr), bd = wgmma_desc_kmajor_sw128(b_addr);
#pragma unroll
      for (int ks = 0; ks < K::kKSteps; ++ks) {  // 32 B of K per step, 4 steps per 128 B panel: the scan's order
        const uint32_t ao = ((ks >> 2) * kABlockPanel + (ks & 3) * 32) >> 4;
        const uint32_t bo = ((ks >> 2) * kSubtileBytes + (ks & 3) * 32) >> 4;
        if constexpr (KIND == 0) {
          wgmma_m64n128k16_bf16(d, ad + ao, bd + bo, ks != 0);
        } else if constexpr (KIND == 1) {
          wgmma_m64n128k32_s8(d, ad + ao, bd + bo, ks != 0);
        } else {
          wgmma_m64n128k16_f16(d, ad + ao, bd + bo, ks != 0);
        }
      }
      wgmma_commit();
    }
    if (n + 1 < n_tiles) fetch(n + 1);  // in flight while the chain runs
    wgmma_wait<0>();
    reg_fence_all(d);
    epi(d, n);
  }
}

}  // namespace bms
