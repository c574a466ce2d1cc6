// search_pages.cu -- searching with stored pages as the queries ("pages like this one"): the source pages' packed rows
// copied into the scan's query layout, their dequantised rows for the first stages, the per-source allow masks of a
// candidate rerank, and the per-source score normalisation.  The scoring and the selection are search_core's (api.cu).
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include "common.cuh"

namespace bms {

// item of row r: the last i with start[i] <= r (start ascending, start[0] = 0, r < start[n])
__device__ __forceinline__ int64_t item_of(const int64_t* __restrict__ start, int64_t n, int64_t r) {
  int64_t lo = 0, hi = n - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (__ldg(start + mid) <= r) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Query layout from corpus pages: destination row r of source i (rows ds[i] .. ds[i+1]) is row r - ds[i] of page src[i]
// while that is below the page's true length (ss[i+1] - ss[i]), else zero; rows from ds[n] to dst_rows are zero, and rows
// before ds[0] (another packer's) are not touched.  One thread per 16-byte piece; the bytes are copied as stored.  rows may be mapped host memory (a host-resident corpus): only
// the source pages' true rows are read.
__global__ void __launch_bounds__(256)
pack_src_pages_kernel(const uint4* __restrict__ rows, int64_t pieces_per_row, const int64_t* __restrict__ page_start,
                      const int64_t* __restrict__ src, const int64_t* __restrict__ ss, const int64_t* __restrict__ ds,
                      int64_t n_src, int64_t dst_rows, uint4* __restrict__ dst) {
  const int64_t total = dst_rows * pieces_per_row;
  const int64_t used = __ldg(ds + n_src) * pieces_per_row;
  for (int64_t t = __ldg(ds) * pieces_per_row + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; t < total;
       t += int64_t(gridDim.x) * blockDim.x) {
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (t < used) {
      const int64_t r = t / pieces_per_row, piece = t - r * pieces_per_row;
      const int64_t i = item_of(ds, n_src, r);
      const int64_t k = r - __ldg(ds + i);
      if (k < __ldg(ss + i + 1) - __ldg(ss + i)) v = rows[(__ldg(page_start + __ldg(src + i)) + k) * pieces_per_row + piece];
    }
    dst[t] = v;
  }
}

// The true rows of the source pages back to back as float32 (row r of the output = row r - ss[i] of page src[i]), each
// element the packed value widened exactly (bf16, int8 code, e4m3 value, sign bit as +-1) times scale in fp32.  One warp
// per row, lane l owns elements 4l..4l+3.
__global__ void __launch_bounds__(256)
page_rows_kernel(const void* __restrict__ rows, int dtype, const int64_t* __restrict__ page_start,
                 const int64_t* __restrict__ src, const int64_t* __restrict__ ss, int64_t n_src, float scale,
                 float4* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t n_rows = __ldg(ss + n_src);
  for (int64_t r = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; r < n_rows;
       r += (int64_t(gridDim.x) * blockDim.x) >> 5) {
    const int64_t i = item_of(ss, n_src, r);
    const int64_t row = __ldg(page_start + __ldg(src + i)) + (r - __ldg(ss + i));
    float4 v;
    if (dtype == B200MS_BF16) {
      const uint2 w = static_cast<const uint2*>(rows)[row * 32 + lane];
      v = make_float4(__uint_as_float(w.x << 16), __uint_as_float(w.x & 0xffff0000u), __uint_as_float(w.y << 16),
                      __uint_as_float(w.y & 0xffff0000u));
    } else if (dtype == B200MS_I8) {
      const uint32_t w = static_cast<const uint32_t*>(rows)[row * 32 + lane];
      v = make_float4(float(int8_t(w)), float(int8_t(w >> 8)), float(int8_t(w >> 16)), float(int8_t(w >> 24)));
    } else if (dtype == B200MS_F8) {
      const uint32_t w = static_cast<const uint32_t*>(rows)[row * 32 + lane];
      float e[4];
      for (int j = 0; j < 4; ++j)
        e[j] = __half2float(__half(__nv_cvt_fp8_to_halfraw(__nv_fp8_storage_t((w >> (8 * j)) & 0xffu), __NV_E4M3)));
      v = make_float4(e[0], e[1], e[2], e[3]);
    } else {  // B1: element e is bit 7 - e%8 of byte e/8 (MSB first); lane l's elements sit in byte l/2
      const uint32_t byte = static_cast<const uint8_t*>(rows)[row * 16 + lane / 2];
      const uint32_t nib = (lane & 1) ? byte & 0xfu : byte >> 4;
      v = make_float4((nib & 8u) ? 1.f : -1.f, (nib & 4u) ? 1.f : -1.f, (nib & 2u) ? 1.f : -1.f, (nib & 1u) ? 1.f : -1.f);
    }
    out[r * 32 + lane] = make_float4(v.x * scale, v.y * scale, v.z * scale, v.w * scale);
  }
}

// Candidate mode with allow masks: clear the valid bit of slot j (list q = j / stride) when page cand[j] is not allowed
// by q's mask row (mask_index NULL: row 0; -1: unfiltered).  One warp per 32-slot word, so no word is shared.
__global__ void __launch_bounds__(256)
mask_cand_slots_kernel(const int64_t* __restrict__ cand, int64_t n_slots, int64_t stride, int64_t n_pages,
                       const uint32_t* __restrict__ allow, const int32_t* __restrict__ mask_index, int64_t words,
                       uint32_t* __restrict__ slot_mask) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  bool keep = true;
  if (j < n_slots) {
    const int64_t id = cand[j];
    const int row = mask_index ? mask_index[j / stride] : 0;
    if (row >= 0 && id >= 0 && id < n_pages) keep = (allow[int64_t(row) * words + (id >> 5)] >> (id & 31)) & 1u;
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, keep);
  if ((threadIdx.x & 31) == 0 && j < n_slots) slot_mask[j >> 5] &= bal;
}

// Per source q of true length len = page_len[src[q]]: a reported score s becomes s / len (__fdiv_rn; a NaN is kept as
// reported); a source without rows reports nothing (count 0, every slot -inf / -1).
__global__ void normalise_pages_kernel(const int64_t* __restrict__ src, const int32_t* __restrict__ page_len, int n_src,
                                       int k, float* __restrict__ scores, int64_t* __restrict__ ids,
                                       int32_t* __restrict__ counts) {
  const int q = blockIdx.x;
  const int32_t len = page_len[src[q]];
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    float& s = scores[int64_t(q) * k + j];
    if (len <= 0) {
      s = -__int_as_float(0x7f800000);
      ids[int64_t(q) * k + j] = -1;
    } else if (!isnan(s)) {
      s = __fdiv_rn(s, float(len));
    }
  }
  if (threadIdx.x == 0 && len <= 0) counts[q] = 0;
}

int launch_pack_src_pages(b200ms_t* h, const int64_t* src_dev, const int64_t* ss_dev, const int64_t* ds_dev, int64_t n_src,
                          int64_t row0, int64_t dst_rows, void* dst, cudaStream_t s) {
  if (dst_rows <= row0) return B200MS_OK;
  const Corpus& c = h->corpus;
  const int64_t ppr = b200ms_row_bytes(c.dtype) / 16;
  pack_src_pages_kernel<<<grid_stride_blocks(h, (dst_rows - row0) * ppr, 256, 16), 256, 0, s>>>(
      static_cast<const uint4*>(c.rows), ppr, static_cast<const int64_t*>(h->page_start.p), src_dev, ss_dev, ds_dev, n_src,
      dst_rows, static_cast<uint4*>(dst));
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch pack_src_pages");
}

int launch_page_rows(b200ms_t* h, const int64_t* src_dev, const int64_t* ss_dev, int64_t n_src, int64_t n_rows, float scale,
                     float* out, cudaStream_t s) {
  if (n_rows <= 0) return B200MS_OK;
  const Corpus& c = h->corpus;
  page_rows_kernel<<<grid_stride_blocks(h, n_rows * 32, 256, 16), 256, 0, s>>>(
      c.rows, c.dtype, static_cast<const int64_t*>(h->page_start.p), src_dev, ss_dev, n_src, scale,
      reinterpret_cast<float4*>(out));
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch page_rows");
}

int launch_mask_cand_slots(b200ms_t* h, const int64_t* cand, int64_t n_slots, int64_t stride, const uint32_t* allow,
                           const int32_t* mask_index, uint32_t* slot_mask, cudaStream_t s) {
  if (n_slots <= 0) return B200MS_OK;
  mask_cand_slots_kernel<<<unsigned((n_slots + 255) / 256), 256, 0, s>>>(cand, n_slots, stride, h->corpus.n_pages, allow,
                                                                         mask_index, (h->corpus.n_pages + 31) / 32, slot_mask);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch mask_cand_slots");
}

int launch_normalise_pages(b200ms_t* h, const int64_t* src_dev, int n_src, int k, float* scores, int64_t* ids,
                           int32_t* counts, cudaStream_t s) {
  normalise_pages_kernel<<<n_src, 128, 0, s>>>(src_dev, static_cast<const int32_t*>(h->page_len.p), n_src, k, scores, ids,
                                               counts);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch normalise_pages");
}

}  // namespace bms
