// compact.cu -- b200ms_compact_rows: move runs of rows down inside ONE buffer until they are contiguous from row 0.
//
// What a delete leaves behind (DELETE ... WHERE document_id, multi_vector_store.py:929-933): the surviving pages as runs of
// rows with holes between them.  Every row moves to a lower or equal address, so source and destination overlap, and a
// destination one CTA writes may be the source another CTA has not read yet: a plain grid-stride gather over the whole
// buffer is wrong (and passes small tests, where one wave of CTAs reads everything before anyone writes).
//
// The destination is walked in ascending windows, one launch (or two) per window on the stream, so windows run in order:
//   * src(d), the source row of destination row d, ascends with d and src(d) >= d.  With disp = src(d0) - d0 at the window's
//     first row, every source of the window [d0, d0 + n) lies at or past d0 + disp.
//   * disp large enough: DIRECT window of n <= disp rows -- its sources all lie at or past its end, so no CTA of the launch
//     writes what another reads, and earlier windows only wrote below d0.
//   * else: BOUNCE window of at most kWindowBytes -- gathered into the library's bounce buffer, then copied out.
// Later windows read at or past their own start, which no earlier window wrote.  Rows that already sit in place (leading
// runs that start at their destination) are skipped.  tests/compact_model.py restates the walk in numpy and checks it
// against an out-of-place copy, including that no window reads a row an earlier launch or its own launch overwrote.
//
// The gather kernel locates a destination row's run by binary search over the prefix sum of the run lengths (restricted to
// the runs the window touches), as ht_gather_kernel locates pages, and moves 16-byte pieces, kUnroll independent loads in
// flight per thread before their stores.
#include <algorithm>

#include "common.cuh"

namespace bms {

constexpr int kUnroll = 4;
constexpr int64_t kWindowBytes = int64_t(64) << 20;       // bounce buffer = largest bounce window
constexpr int64_t kMinDirectBytes = kWindowBytes / 4;     // a smaller displacement goes through the bounce buffer
constexpr int64_t kMaxDirectBytes = kWindowBytes * 16;    // piece indexes inside a window stay 32-bit

// dst[piece lp of window row lr] = src[the same piece of source row start[i] + (d0 + lr - pre[i])], i = the run with
// pre[i] <= d0 + lr < pre[i + 1], searched in [r_lo, r_hi].  ppr = 16-byte pieces per row.
__global__ void __launch_bounds__(256)
compact_gather_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, const int64_t* __restrict__ pre,
                      const int64_t* __restrict__ start, int r_lo, int r_hi, int64_t d0, uint32_t ppr, uint32_t n_pieces) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t p0 = blockIdx.x * blockDim.x + threadIdx.x; p0 < n_pieces; p0 += stride * kUnroll) {
    uint4 v[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const uint32_t p = p0 + k * stride;
      if (p < n_pieces) {
        const uint32_t lr = p / ppr;
        const int64_t d = d0 + lr;
        int lo = r_lo, hi = r_hi;
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (pre[mid] <= d) lo = mid; else hi = mid - 1;
        }
        v[k] = src[(start[lo] + (d - pre[lo])) * ppr + (p - lr * ppr)];
      }
    }
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const uint32_t p = p0 + k * stride;
      if (p < n_pieces) dst[p] = v[k];
    }
  }
}

static int launch_gather(b200ms_t* h, const void* rows, void* dst, const int64_t* pre_dev, const int64_t* start_dev, int r_lo,
                         int r_hi, int64_t d0, int64_t n_rows, int64_t row_bytes, cudaStream_t s) {
  const uint32_t ppr = uint32_t(row_bytes / 16), n_pieces = uint32_t(n_rows * ppr);
  int64_t grid = (int64_t(n_pieces) + 256 * kUnroll - 1) / (256 * kUnroll);
  grid = std::min<int64_t>(grid, int64_t(h->num_sms) * 8);
  compact_gather_kernel<<<int(grid), 256, 0, s>>>(static_cast<const uint4*>(rows), static_cast<uint4*>(dst), pre_dev, start_dev,
                                                 r_lo, r_hi, d0, ppr, n_pieces);
  h->launches++;
  return check_cuda(h, cudaGetLastError(), "launch compact_gather_kernel");
}

}  // namespace bms

using namespace bms;

#define B200MS_API extern "C" __attribute__((visibility("default")))

B200MS_API int b200ms_compact_rows(b200ms_t* h, void* rows, int64_t row_bytes, const int64_t* run_start, const int64_t* run_rows,
                                   int64_t n_runs, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  if (n_runs < 0 || n_runs >= (int64_t(1) << 31) || row_bytes <= 0 || row_bytes % 16 || row_bytes > kWindowBytes ||
      (n_runs > 0 && (!rows || !run_start || !run_rows)) || (reinterpret_cast<uintptr_t>(rows) & 15))
    return set_error(h, B200MS_EINVAL, "compact_rows: bad arguments (row_bytes a multiple of 16, rows 16-byte aligned)");
  // meta = [pre (n_runs + 1) | start (n_runs)]: destination and source row of every run's first row
  std::vector<int64_t> meta(size_t(2 * n_runs + 1));
  int64_t* pre = meta.data();
  int64_t* start = pre + n_runs + 1;
  pre[0] = 0;
  for (int64_t i = 0; i < n_runs; ++i) {
    if (run_rows[i] < 0 || run_start[i] < (i ? run_start[i - 1] + run_rows[i - 1] : 0) ||
        run_start[i] > (int64_t(1) << 62) / row_bytes - run_rows[i])
      return set_error(h, B200MS_EINVAL, "compact_rows: run " + std::to_string(i) + " is negative, overlaps the run before it or "
                                             "is out of order");
    pre[i + 1] = pre[i] + run_rows[i];
    start[i] = run_start[i];
  }
  const int64_t total = pre[n_runs];
  int64_t r = 0;
  while (r < n_runs && start[r] == pre[r]) ++r;  // in place already
  if (r == n_runs) return B200MS_OK;
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  if (int e = upload(h, h->compact_meta, meta.data(), meta.size() * 8, s)) return e;
  const int64_t* pre_dev = static_cast<const int64_t*>(h->compact_meta.p);
  const int64_t* start_dev = pre_dev + n_runs + 1;
  const int64_t window_rows = kWindowBytes / row_bytes;
  const int64_t min_direct_rows = (kMinDirectBytes + row_bytes - 1) / row_bytes;
  const int64_t max_direct_rows = kMaxDirectBytes / row_bytes;
  uint8_t* base = static_cast<uint8_t*>(rows);
  // the run holding destination row x: the last i with pre[i] <= x (runs without rows are never picked)
  auto run_of = [&](int64_t x) { return int64_t(std::upper_bound(pre, pre + n_runs + 1, x) - pre) - 1; };
  for (int64_t d = pre[r]; d < total;) {
    const int64_t r_lo = run_of(d);
    const int64_t disp = start[r_lo] + (d - pre[r_lo]) - d;
    const bool direct = disp >= min_direct_rows;
    const int64_t n = std::min(direct ? std::min(disp, max_direct_rows) : window_rows, total - d);
    const int64_t r_hi = run_of(d + n - 1);
    if (direct) {
      if (int e = launch_gather(h, rows, base + d * row_bytes, pre_dev, start_dev, int(r_lo), int(r_hi), d, n, row_bytes, s)) return e;
    } else {
      if (int e = reserve(h, h->compact_bounce, size_t(kWindowBytes))) return e;
      if (int e = launch_gather(h, rows, h->compact_bounce.p, pre_dev, start_dev, int(r_lo), int(r_hi), d, n, row_bytes, s)) return e;
      if (int e = check_cuda(h, cudaMemcpyAsync(base + d * row_bytes, h->compact_bounce.p, size_t(n * row_bytes),
                                                cudaMemcpyDeviceToDevice, s), "compact_rows: copy out of the bounce buffer"))
        return e;
    }
    d += n;
  }
  return B200MS_OK;
}
