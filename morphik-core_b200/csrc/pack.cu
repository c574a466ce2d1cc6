// pack.cu -- quantise / layout kernels on either side of the scorer.
//
//   sign-bit quantise + MSB-first pack : morphik_rust binary_quantize_batch_packed (morphik_rust/src/binary_ops.rs:147-222;
//                                        authoritative Python fallback core/utils/fast_ops.py:191-227): bit = float32(x) > 0
//   page / query padding               : new (the reference stores ragged BIT(128)[] arrays / per-page .npy files,
//                                        multi_vector_store.py:240-251, fast_multivector_store.py:673-707)
//
// One warp converts one destination row (lane l owns elements 4l..4l+3); HBM traffic is one coalesced read of the
// source row and one coalesced write of the destination row -- these kernels are copy-bound.
#include <cuda_bf16.h>
#include <cuda_fp8.h>

#include "common.cuh"
#include "ptx.cuh"

namespace bms {

// NaN -> 0: it has neither sign nor magnitude (fmaxf(NaN, -127) alone would make it -127, the strongest negative value)
__device__ __forceinline__ int quant_i8(float x, float scale) {
  const float r = rintf(x * scale);  // round-half-even, like numpy.rint in the oracle
  return isnan(r) ? 0 : int(fminf(fmaxf(r, -127.f), 127.f));
}

__device__ __forceinline__ void store_row4(void* dst, int dst_dtype, int64_t row, int lane, float4 v, float i8_scale) {
  if (dst_dtype == B200MS_BF16) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y);
    const __nv_bfloat162 hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 out;
    out.x = *reinterpret_cast<const uint32_t*>(&lo);
    out.y = *reinterpret_cast<const uint32_t*>(&hi);
    reinterpret_cast<uint2*>(dst)[row * 32 + lane] = out;
  } else if (dst_dtype == B200MS_I8) {
    const uint32_t b0 = uint32_t(quant_i8(v.x, i8_scale)) & 0xffu, b1 = uint32_t(quant_i8(v.y, i8_scale)) & 0xffu;
    const uint32_t b2 = uint32_t(quant_i8(v.z, i8_scale)) & 0xffu, b3 = uint32_t(quant_i8(v.w, i8_scale)) & 0xffu;
    reinterpret_cast<uint32_t*>(dst)[row * 32 + lane] = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
  } else if (dst_dtype == B200MS_F8) {  // e4m3, round-to-nearest-even, saturating at +-448 (NaN stays NaN)
    const uint32_t b0 = __nv_cvt_float_to_fp8(v.x * i8_scale, __NV_SATFINITE, __NV_E4M3);
    const uint32_t b1 = __nv_cvt_float_to_fp8(v.y * i8_scale, __NV_SATFINITE, __NV_E4M3);
    const uint32_t b2 = __nv_cvt_float_to_fp8(v.z * i8_scale, __NV_SATFINITE, __NV_E4M3);
    const uint32_t b3 = __nv_cvt_float_to_fp8(v.w * i8_scale, __NV_SATFINITE, __NV_E4M3);
    reinterpret_cast<uint32_t*>(dst)[row * 32 + lane] = b0 | (b1 << 8) | (b2 << 16) | (b3 << 24);
  } else {  // B200MS_B1: element e -> byte e/8, bit 7 - e%8 (MSB first); strict > 0 (0.0, -0.0, NaN -> 0)
    const uint32_t nib = (uint32_t(v.x > 0.f) << 3) | (uint32_t(v.y > 0.f) << 2) | (uint32_t(v.z > 0.f) << 1) |
                         uint32_t(v.w > 0.f);
    const uint32_t other = __shfl_down_sync(0xffffffffu, nib, 1);
    const uint32_t byte = (nib << 4) | other;  // valid on even lanes: elements 8i..8i+7 for i = lane/2
    const int w = lane & 3;                    // lanes 0..3 assemble the four 32-bit words of the row
    const uint32_t word = __shfl_sync(0xffffffffu, byte, 8 * w) | (__shfl_sync(0xffffffffu, byte, 8 * w + 2) << 8) |
                          (__shfl_sync(0xffffffffu, byte, 8 * w + 4) << 16) |
                          (__shfl_sync(0xffffffffu, byte, 8 * w + 6) << 24);
    if (lane < 4) reinterpret_cast<uint32_t*>(dst)[row * 4 + lane] = word;
  }
}

// items = pages (pad_mode 0: padding rows repeat the item's last true row) or queries (pad_mode 1: zero rows).
// src_start/dst_start: [n_items+1] row offsets in the ragged source / padded destination.  Rows of dst past
// dst_start[n_items] (up to dst_rows) are zero-filled.
__global__ void __launch_bounds__(256)
pack_rows_kernel(const void* __restrict__ src, int src_dtype, const int64_t* __restrict__ src_start,
                 const int64_t* __restrict__ dst_start, int64_t n_items, int64_t dst_rows, int pad_mode,
                 void* __restrict__ dst, int dst_dtype, float i8_scale) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t warp_stride = (int64_t(gridDim.x) * blockDim.x) >> 5;
  const int64_t used_rows = n_items > 0 ? __ldg(dst_start + n_items) : 0;
  for (int64_t r = warp_global; r < dst_rows; r += warp_stride) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < used_rows) {
      int64_t lo = 0, hi = n_items - 1;  // last item with dst_start[item] <= r
      while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (__ldg(dst_start + mid) <= r) lo = mid; else hi = mid - 1;
      }
      const int64_t s0 = __ldg(src_start + lo), s1 = __ldg(src_start + lo + 1);
      const int64_t k = r - __ldg(dst_start + lo);
      if (k < s1 - s0) {
        v = load_row4(src, src_dtype, s0 + k, lane);
      } else if (pad_mode == 0 && s1 > s0) {
        v = load_row4(src, src_dtype, s1 - 1, lane);
      }
    }
    store_row4(dst, dst_dtype, r, lane, v, i8_scale);
  }
}

__global__ void __launch_bounds__(256)
chunk_page_kernel(const int64_t* __restrict__ page_start, int64_t n_pages, int32_t* __restrict__ chunk_page) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t warp_stride = (int64_t(gridDim.x) * blockDim.x) >> 5;
  for (int64_t p = warp_global; p < n_pages; p += warp_stride) {
    const int64_t c0 = __ldg(page_start + p) / kGroup, c1 = __ldg(page_start + p + 1) / kGroup;
    for (int64_t c = c0 + lane; c < c1; c += 32) chunk_page[c] = int32_t(p);
  }
}

// Candidate (rerank) mode: unit j = chunk range of page cand_ids[j] (empty for id < 0); slot_mask bit j = id valid.
__global__ void cand_units_kernel(const int64_t* __restrict__ cand_ids, int n_cand, const int64_t* __restrict__ page_start,
                                  int64_t n_pages, int32_t* __restrict__ unit_start, int32_t* __restrict__ unit_end,
                                  uint32_t* __restrict__ slot_mask) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t id = j < n_cand ? cand_ids[j] : -1;
  const bool ok = id >= 0 && id < n_pages;
  if (j < n_cand && unit_start) {
    unit_start[j] = ok ? int32_t(page_start[id] / kGroup) : 0;
    unit_end[j] = ok ? int32_t(page_start[id + 1] / kGroup) : 0;
  }
  if (slot_mask) {
    const uint32_t bal = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0 && j < n_cand) slot_mask[j >> 5] = bal;
  }
}

// zero_pad_compat for candidate lists: n_lists lists of n_cand slots (list l at slots [l*stride, l*stride + n_cand)) are
// "batched" `batch` slots at a time in first-stage order, exactly as score_multi_vector batches the candidate pages
// (fast_multivector_store.py:553-555, batch_size 128); bit = page shorter than the longest page of its batch.
// One block per list; the list's page lengths are staged in shared memory (n_cand <= 4096 = B200MS_MAX_K).
constexpr int kClampMaxCand = 4096;
__global__ void __launch_bounds__(256)
clamp_slots_kernel(const int64_t* __restrict__ cand_ids, int n_cand, int64_t stride, int batch,
                   const int32_t* __restrict__ page_len, int64_t n_pages, uint32_t* __restrict__ clamp_bits) {
  __shared__ int32_t s_len[kClampMaxCand];
  __shared__ int32_t s_max[kClampMaxCand];
  const int64_t base = int64_t(blockIdx.x) * stride;  // a multiple of 32 (0 for a single list)
  for (int i = threadIdx.x; i < n_cand; i += blockDim.x) {
    const int64_t id = cand_ids[base + i];
    s_len[i] = (id >= 0 && id < n_pages) ? __ldg(page_len + id) : 0;
  }
  __syncthreads();
  const int nb = (n_cand + batch - 1) / batch;
  for (int b = threadIdx.x; b < nb; b += blockDim.x) {
    int mx = 0;
    const int e = (b + 1) * batch < n_cand ? (b + 1) * batch : n_cand;
    for (int i = b * batch; i < e; ++i) mx = max(mx, s_len[i]);
    s_max[b] = mx;
  }
  __syncthreads();
  for (int w = threadIdx.x; w < (n_cand + 31) / 32; w += blockDim.x) {
    uint32_t bits = 0;
    for (int j = 0; j < 32 && w * 32 + j < n_cand; ++j) {
      const int i = w * 32 + j;
      if (s_len[i] < s_max[i / batch]) bits |= 1u << j;
    }
    clamp_bits[base / 32 + w] = bits;
  }
}

int launch_clamp_slots(b200ms_t* h, const int64_t* cand_ids, int n_cand, int n_lists, int64_t list_stride, int batch,
                       uint32_t* clamp_bits, cudaStream_t s) {
  if (n_cand <= 0 || n_lists <= 0) return B200MS_OK;
  if (n_cand > kClampMaxCand)
    return set_error(h, B200MS_EINVAL, "zero_pad_compat: at most 4096 candidates per list (the reference reranks <= 75)");
  if (batch < 1) batch = 1;
  clamp_slots_kernel<<<n_lists, 256, 0, s>>>(cand_ids, n_cand, list_stride, batch, static_cast<const int32_t*>(h->page_len.p),
                                            h->corpus.n_pages, clamp_bits);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch clamp_slots");
}

// [n_lists, n_cand] -> [n_lists, stride] (stride = roundup(n_cand, 32)), tail slots = -1
__global__ void pad_cands_kernel(const int64_t* __restrict__ src, int n_cand, int64_t stride, int64_t total, int64_t* __restrict__ dst) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t l = i / stride, j = i % stride;
  dst[i] = j < n_cand ? src[l * n_cand + j] : int64_t(-1);
}

int launch_pad_cands(b200ms_t* h, const int64_t* src, int n_cand, int n_lists, int64_t stride, int64_t* dst, cudaStream_t s) {
  const int64_t total = stride * n_lists;
  if (total <= 0) return B200MS_OK;
  pad_cands_kernel<<<unsigned((total + 255) / 256), 256, 0, s>>>(src, n_cand, stride, total, dst);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch pad_cands");
}

int launch_cand_units(b200ms_t* h, const CorpusView& v, const int64_t* cand_ids, int n_cand, int32_t* unit_start,
                      int32_t* unit_end, uint32_t* slot_mask, cudaStream_t s) {
  if (n_cand <= 0) return B200MS_OK;
  cand_units_kernel<<<(n_cand + 255) / 256, 256, 0, s>>>(cand_ids, n_cand, v.page_start, v.n_pages, unit_start, unit_end,
                                                        slot_mask);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch cand_units");
}

// hamming_distance_batch (core/utils/fast_ops.py:242-248, morphik_rust/src/binary_ops.rs:266-292): popcount(q XOR c_i)
// of one packed 16-byte query against n packed candidates -- one thread per candidate, 128-bit loads.
__global__ void __launch_bounds__(256)
hamming_batch_kernel(const uint4* __restrict__ q, const uint4* __restrict__ cand, int64_t n, uint32_t* __restrict__ out) {
  const uint4 qq = __ldg(q);
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    const uint4 c = __ldg(cand + i);
    out[i] = __popc(c.x ^ qq.x) + __popc(c.y ^ qq.y) + __popc(c.z ^ qq.z) + __popc(c.w ^ qq.w);
  }
}

int launch_hamming_batch(b200ms_t* h, const void* q, const void* cand, int64_t n, uint32_t* out, cudaStream_t s) {
  if (n <= 0) return B200MS_OK;
  int64_t blocks = (n + 255) / 256;
  if (blocks > int64_t(h->num_sms) * 8) blocks = int64_t(h->num_sms) * 8;
  hamming_batch_kernel<<<int(blocks), 256, 0, s>>>(static_cast<const uint4*>(q), static_cast<const uint4*>(cand), n, out);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch hamming_batch");
}

int launch_pack_rows(b200ms_t* h, const void* src, int src_dtype, const int64_t* src_start_dev,
                     const int64_t* dst_start_dev, int64_t n_items, int64_t dst_rows, int pad_mode, void* dst,
                     int dst_dtype, float i8_scale, cudaStream_t s) {
  if (dst_rows <= 0) return B200MS_OK;
  pack_rows_kernel<<<grid_stride_blocks(h, dst_rows, 8, 16), 256, 0, s>>>(
      src, src_dtype, src_start_dev, dst_start_dev, n_items, dst_rows, pad_mode, dst, dst_dtype, i8_scale);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch pack_rows");
}

int launch_chunk_page(b200ms_t* h, const int64_t* page_start_dev, int64_t n_pages, int32_t* chunk_page, cudaStream_t s) {
  if (n_pages <= 0) return B200MS_OK;
  chunk_page_kernel<<<grid_stride_blocks(h, n_pages, 8, 16), 256, 0, s>>>(page_start_dev, n_pages, chunk_page);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch chunk_page");
}

}  // namespace bms
