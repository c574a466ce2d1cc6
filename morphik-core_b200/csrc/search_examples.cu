// search_examples.cu -- relevance feedback ("more like these, less like that"): the kernels that turn one scan's group scores
// of several weighted examples per request into one fused score row per request, and the device-side union of a request's
// first-stage candidate lists.  The scan and the selection are search_core's (api.cu); the per-example score is exactly the
// one the selection and b200ms_search_pages_device report (topk_keys.cuh's page_key / finish_sum, then scale and length).
#include "common.cuh"
#include "topk_keys.cuh"

namespace bms {

// dst row i = src row idx[i]: the requests' mask-index entries or candidate lists spread to their examples
template <typename T>
__global__ void __launch_bounds__(256)
gather_rows_kernel(const T* __restrict__ src, int64_t row_len, const int32_t* __restrict__ idx, int64_t total,
                   T* __restrict__ dst) {
  for (int64_t t = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; t < total; t += int64_t(gridDim.x) * blockDim.x) {
    const int64_t i = t / row_len;
    dst[t] = src[int64_t(__ldg(idx + i)) * row_len + (t - i * row_len)];
  }
}

// One thread per (request r, item p).  An example's score is the selection's reported page score (the sum of its group
// scores in SumOf<T>, finish_sum, float, times score_scale) over its true length, as b200ms_search_pages_device reports it;
// the fused score adds w * score in example order.  Every step is an explicit _rn operation, so that no FMA contraction
// changes a bit and numpy float32 reproduces it.  An item r's allow row forbids is neither read (a filtered scan leaves its
// scores stale) nor written (the selection skips it).
template <typename T>
__global__ void __launch_bounds__(256)
fuse_examples_kernel(const T* __restrict__ gs, int64_t ld, const ExampleItem* __restrict__ items,
                     const int32_t* __restrict__ req_off, int n_req, int64_t n_items, const uint32_t* __restrict__ allow,
                     const int32_t* __restrict__ mask_index, int64_t mask_stride, float score_scale,
                     float* __restrict__ fused, int64_t fused_ld) {
  for (int r = blockIdx.y; r < n_req; r += gridDim.y) {
    const uint32_t* a = allow;
    if (allow) {
      const int64_t row = mask_index ? __ldg(mask_index + r) : r;
      a = row >= 0 ? allow + row * mask_stride : nullptr;
    }
    const int e0 = __ldg(req_off + r), e1 = __ldg(req_off + r + 1);
    for (int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; p < n_items; p += int64_t(gridDim.x) * blockDim.x) {
      if (a && !((__ldg(a + (p >> 5)) >> (p & 31)) & 1u)) continue;
      float acc = 0.0f;
      for (int e = e0; e < e1; ++e) {
        const int g0 = __ldg(&items[e].g0), g1 = __ldg(&items[e].g1);
        if (g1 <= g0) continue;
        const int64_t col = __ldg(&items[e].col0) + p;
        typename SumOf<T>::type sum = 0;
        for (int g = g0; g < g1; ++g) sum += __ldg(gs + int64_t(g) * ld + col);
        const float score = __fdiv_rn(__fmul_rn(float(finish_sum(sum)), score_scale), __ldg(&items[e].len));
        acc = __fadd_rn(acc, __fmul_rn(__ldg(&items[e].w), score));
      }
      fused[int64_t(r) * fused_ld + p] = acc;
    }
  }
}

// One CTA per request: its entries are the slots of lists list_off[r] .. list_off[r+1], row-major.  Pass 1 records every
// distinct id's first entry in an open-addressing table (keys ~0 = empty, first entries atomicMin'ed); pass 2 walks the
// entries in order and keeps those at their id's first entry, ranked by a block-wide prefix count.  The result depends
// only on the input, not on the order the atomics land in.
constexpr int kUnionThreads = 1024;
constexpr unsigned long long kUnionEmpty = ~0ull;

__device__ __forceinline__ int64_t union_slot(unsigned long long* keys, int64_t cap, int64_t id, bool insert) {
  int64_t slot = int64_t((uint64_t(id) * 0x9E3779B97F4A7C15ull) >> 17) & (cap - 1);
  for (;;) {
    const unsigned long long k =
        insert ? atomicCAS(keys + slot, kUnionEmpty, (unsigned long long)id) : __ldcg(keys + slot);
    if (k == (unsigned long long)id || (insert && k == kUnionEmpty)) return slot;
    slot = (slot + 1) & (cap - 1);
  }
}

__global__ void __launch_bounds__(kUnionThreads)
union_candidates_kernel(const int64_t* __restrict__ cand, int n_cand, const int32_t* __restrict__ list_off,
                        unsigned long long* keys_all, uint32_t* first_all, int64_t cap, int64_t* __restrict__ out,
                        int width) {
  __shared__ uint32_t warp_cnt[kUnionThreads / 32];
  const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int64_t beg = int64_t(list_off[r]) * n_cand, n = int64_t(list_off[r + 1]) * n_cand - beg;
  unsigned long long* keys = keys_all + int64_t(r) * cap;
  uint32_t* first = first_all + int64_t(r) * cap;
  for (int64_t i = tid; i < n; i += kUnionThreads) {
    const int64_t id = cand[beg + i];
    if (id >= 0) atomicMin(first + union_slot(keys, cap, id, true), uint32_t(i));
  }
  __syncthreads();
  int64_t count = 0;
  for (int64_t c = 0; c < n; c += kUnionThreads) {
    const int64_t i = c + tid;
    const int64_t id = i < n ? cand[beg + i] : -1;
    const bool keep = id >= 0 && __ldcg(first + union_slot(keys, cap, id, false)) == uint32_t(i);
    const uint32_t bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int64_t rank = count + __popc(bal & ((1u << lane) - 1u));
    int total = 0;
    for (int w = 0; w < kUnionThreads / 32; ++w) {
      if (w < wid) rank += warp_cnt[w];
      total += warp_cnt[w];
    }
    if (keep && rank < width) out[int64_t(r) * width + rank] = id;
    count += total;
    __syncthreads();
  }
  for (int64_t j = (count < width ? count : width) + tid; j < width; j += kUnionThreads) out[int64_t(r) * width + j] = -1;
}

template <typename T>
int launch_gather_rows(b200ms_t* h, const T* src, int64_t row_len, const int32_t* idx, int n_rows, T* dst, cudaStream_t s) {
  const int64_t total = row_len * n_rows;
  if (total <= 0) return B200MS_OK;
  gather_rows_kernel<T><<<grid_stride_blocks(h, total, 256, 16), 256, 0, s>>>(src, row_len, idx, total, dst);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch gather_rows");
}
template int launch_gather_rows<int32_t>(b200ms_t*, const int32_t*, int64_t, const int32_t*, int, int32_t*, cudaStream_t);
template int launch_gather_rows<int64_t>(b200ms_t*, const int64_t*, int64_t, const int32_t*, int, int64_t*, cudaStream_t);

int launch_fuse_examples(b200ms_t* h, const void* gs, int score_dtype, int64_t ld, const ExampleItem* items,
                         const int32_t* req_off, int n_req, int64_t n_items, const uint32_t* allow, const int32_t* mask_index,
                         int64_t mask_stride, float score_scale, float* fused, int64_t fused_ld, cudaStream_t s) {
  if (n_req <= 0 || n_items <= 0) return B200MS_OK;
  // enough CTAs to cover the SMs a few times over, spread over the requests
  const int gy = n_req < 65535 ? n_req : 65535;
  int64_t gx = (n_items + 255) / 256;
  const int64_t want = (int64_t(h->num_sms) * 8 + gy - 1) / gy;
  if (gx > want) gx = want;
  const dim3 grid(unsigned(gx < 1 ? 1 : gx), unsigned(gy));
  if (score_dtype == B200MS_F32)
    fuse_examples_kernel<float><<<grid, 256, 0, s>>>(static_cast<const float*>(gs), ld, items, req_off, n_req, n_items, allow,
                                                     mask_index, mask_stride, score_scale, fused, fused_ld);
  else
    fuse_examples_kernel<int><<<grid, 256, 0, s>>>(static_cast<const int*>(gs), ld, items, req_off, n_req, n_items, allow,
                                                   mask_index, mask_stride, score_scale, fused, fused_ld);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch fuse_examples");
}

int launch_union_candidates(b200ms_t* h, const int64_t* cand, int n_cand, const int32_t* list_off_dev, int n_req,
                            int64_t max_entries, int64_t* out, int width, cudaStream_t s) {
  if (n_req <= 0) return B200MS_OK;
  int64_t cap = 64;  // at most half full
  while (cap < 2 * max_entries) cap <<= 1;
  const size_t keys_bytes = size_t(n_req) * size_t(cap) * 8, bytes = keys_bytes + size_t(n_req) * size_t(cap) * 4;
  if (int e = reserve(h, h->ex_union, bytes)) return e;
  if (int e = check_cuda(h, cudaMemsetAsync(h->ex_union.p, 0xff, bytes, s), "union_candidates: memset")) return e;
  unsigned long long* keys = static_cast<unsigned long long*>(h->ex_union.p);
  uint32_t* first = reinterpret_cast<uint32_t*>(static_cast<uint8_t*>(h->ex_union.p) + keys_bytes);
  union_candidates_kernel<<<n_req, kUnionThreads, 0, s>>>(cand, n_cand, list_off_dev, keys, first, cap, out, width);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch union_candidates");
}

}  // namespace bms
