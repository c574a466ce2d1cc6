// scan_plan.cu -- the work units of a filtered full scan: only the pages the call's allow masks name are read.
//
// Replaces nothing of the reference's arithmetic: the WHERE document_id IN (...) of the SQL scan
// (core/vector_store/multi_vector_store.py:752-757) keeps Postgres from reading other documents' rows, and this does the
// same for the MaxSim scan.  The selection never reads the score of a page whose allow bit is clear (page_key, doc_item), so
// a scan that skips those pages returns the same results bit for bit.
//
// Built per call on the caller's stream, without a synchronisation (mask contents may change behind the same pointer):
//   1. union   u = OR of the mask rows the call's queries name (a query without a mask: every page), bits past n_pages
//              cleared; rows = padded rows of the allowed pages
//   2. count   unit_rows = clamp(rows / (4 * SMs), kTileN, the handle's unit_rows): set_corpus's rule applied to the allowed
//              rows, so that a sparse filter still spreads over every SM.  Inside every unit of the corpus' own plan, a
//              filtered unit is a run of allowed pages that are adjacent in memory (empty pages have no rows and break
//              nothing), cut after the page at which its rows reach unit_rows.  Units never cross a unit boundary of the
//              corpus' plan: each of its units is walked by one thread, and a mask that allows every page gives that plan back.
//   3. scan    offsets of every corpus unit's filtered units (fixed-order block scan: the unit arrays are deterministic)
//   4. write   unit_start[] / unit_end[] compacted, their count in a device word the scorers read; for 1-bit corpora also
//              the ascending list of allowed pages (the POPC kernel walks pages, not units).
#include "common.cuh"
#include "scan.cuh"

namespace bms {

struct ScanHdr {  // device words of one plan
  int32_t n_units;
  int32_t n_allowed;  // pages in the list (1-bit corpora)
  unsigned long long rows;
};

__global__ void __launch_bounds__(256)
scan_union_kernel(const uint32_t* __restrict__ allow, const int32_t* __restrict__ mask_index, int n_q, int64_t n_pages,
                  const int64_t* __restrict__ page_start, uint32_t* __restrict__ u, ScanHdr* __restrict__ hdr) {
  const int64_t words = (n_pages + 31) >> 5;
  unsigned long long rows = 0;
  for (int64_t w = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; w < words; w += int64_t(gridDim.x) * blockDim.x) {
    uint32_t b = 0;
    if (!mask_index) {
      b = __ldg(allow + w);
    } else {
      for (int q = 0; q < n_q; ++q) {
        const int mi = __ldg(mask_index + q);
        b |= mi < 0 ? ~0u : __ldg(allow + int64_t(mi) * words + w);
      }
    }
    if (w == words - 1 && (n_pages & 31)) b &= (1u << (n_pages & 31)) - 1u;
    u[w] = b;
    while (b) {
      const int64_t p = w * 32 + (__ffs(b) - 1);
      b &= b - 1;
      rows += (unsigned long long)(page_start[p + 1] - page_start[p]);
    }
  }
  for (int off = 16; off > 0; off >>= 1) rows += __shfl_xor_sync(0xffffffffu, rows, off);
  if ((threadIdx.x & 31) == 0 && rows) atomicAdd(&hdr->rows, rows);  // an integer total: the order of additions is immaterial
}

__device__ __forceinline__ int64_t filtered_unit_rows(unsigned long long rows, int num_sms, int64_t cap) {
  int64_t ur = int64_t(rows) / (4 * int64_t(num_sms > 0 ? num_sms : 1));
  if (ur < kTileN) ur = kTileN;
  return ur > cap ? cap : ur;
}

// The filtered units inside unit f of the corpus' plan, in order: emit(i, first chunk, end chunk); returns their count.
template <class Emit>
__device__ __forceinline__ int walk_unit(int f, const int32_t* __restrict__ unit_start, const int32_t* __restrict__ chunk_page,
                                         const int64_t* __restrict__ page_start, const uint32_t* __restrict__ u,
                                         int64_t unit_rows, Emit emit) {
  const int c0 = unit_start[f], c1 = unit_start[f + 1];
  if (c1 <= c0) return 0;
  const int p0 = chunk_page[c0], p1 = chunk_page[c1 - 1];
  int n = 0, start = -1;
  int64_t acc = 0, r0 = page_start[p0];
  for (int p = p0; p <= p1; ++p) {
    const int64_t r1 = page_start[p + 1];
    if (r1 > r0) {
      if ((u[p >> 5] >> (p & 31)) & 1u) {
        if (start < 0) start = int(r0 / kGroup);
        acc += r1 - r0;
        if (acc >= unit_rows) {
          emit(n++, start, int(r1 / kGroup));
          start = -1;
          acc = 0;
        }
      } else if (start >= 0) {
        emit(n++, start, int(r0 / kGroup));
        start = -1;
        acc = 0;
      }
    }
    r0 = r1;
  }
  if (start >= 0) emit(n++, start, c1);
  return n;
}

__global__ void __launch_bounds__(256)
scan_count_kernel(int n_full, const int32_t* __restrict__ unit_start, const int32_t* __restrict__ chunk_page,
                  const int64_t* __restrict__ page_start, const uint32_t* __restrict__ u, const ScanHdr* __restrict__ hdr,
                  int num_sms, int64_t cap, int32_t* __restrict__ cnt) {
  const int64_t ur = filtered_unit_rows(hdr->rows, num_sms, cap);
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < n_full; f += gridDim.x * blockDim.x)
    cnt[f] = walk_unit(f, unit_start, chunk_page, page_start, u, ur, [](int, int, int) {});
}

// word_off == NULL: no page list
__global__ void __launch_bounds__(kScanThreads)
scan_offsets_kernel(const int32_t* __restrict__ cnt, int n_full, int64_t* __restrict__ off, const uint32_t* __restrict__ u,
                    int64_t words, int64_t* __restrict__ word_off, ScanHdr* __restrict__ hdr) {
  block_scan([&](int64_t f) { return int64_t(cnt[f]); }, n_full, off);
  if (word_off) block_scan([&](int64_t w) { return int64_t(__popc(u[w])); }, words, word_off);
  __syncthreads();
  if (threadIdx.x == 0) {
    hdr->n_units = int32_t(off[n_full]);
    hdr->n_allowed = word_off ? int32_t(word_off[words]) : 0;
  }
}

__global__ void __launch_bounds__(256)
scan_write_kernel(int n_full, const int32_t* __restrict__ unit_start, const int32_t* __restrict__ chunk_page,
                  const int64_t* __restrict__ page_start, const uint32_t* __restrict__ u, const ScanHdr* __restrict__ hdr,
                  int num_sms, int64_t cap, const int64_t* __restrict__ off, int32_t* __restrict__ us, int32_t* __restrict__ ue,
                  int64_t words, const int64_t* __restrict__ word_off, int64_t* __restrict__ pages) {
  const int64_t ur = filtered_unit_rows(hdr->rows, num_sms, cap);
  const int64_t tid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x, stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t f = tid; f < n_full; f += stride) {
    const int64_t o = off[f];
    walk_unit(int(f), unit_start, chunk_page, page_start, u, ur, [&](int i, int a, int b) {
      us[o + i] = a;
      ue[o + i] = b;
    });
  }
  if (!word_off) return;
  for (int64_t w = tid; w < words; w += stride) {
    uint32_t b = u[w];
    int64_t o = word_off[w];
    while (b) {
      pages[o++] = w * 32 + (__ffs(b) - 1);
      b &= b - 1;
    }
  }
}

int reserve_scan_plan(b200ms_t* h, const Corpus& c) {
  const size_t n = size_t(c.n_pages > 0 ? c.n_pages : 1), words = (n + 31) / 32, nf = size_t(c.n_units) + 1;
  if (int e = reserve(h, h->scan_union, words * 4)) return e;
  if (int e = reserve(h, h->scan_cnt, nf * 4)) return e;
  if (int e = reserve(h, h->scan_off, nf * 8)) return e;
  if (int e = reserve(h, h->scan_start, n * 4)) return e;  // a unit holds at least one page
  if (int e = reserve(h, h->scan_end, n * 4)) return e;
  if (int e = reserve(h, h->scan_hdr, sizeof(ScanHdr))) return e;
  if (c.dtype != B200MS_B1) return B200MS_OK;
  if (int e = reserve(h, h->scan_word_off, (words + 1) * 8)) return e;
  return reserve(h, h->scan_pages, n * 8);
}

int launch_scan_plan(b200ms_t* h, const uint32_t* allow, const int32_t* mask_index, int n_q, cudaStream_t s, UnitPlan* plan) {
  const Corpus& c = h->corpus;
  const int64_t words = (c.n_pages + 31) / 32;
  const int n_full = c.n_units;
  const bool list = c.dtype == B200MS_B1;
  const int32_t* unit_start = static_cast<const int32_t*>(h->unit_start.p);
  const int32_t* chunk_page = static_cast<const int32_t*>(h->chunk_page.p);
  const int64_t* page_start = static_cast<const int64_t*>(h->page_start.p);
  uint32_t* u = static_cast<uint32_t*>(h->scan_union.p);
  ScanHdr* hdr = static_cast<ScanHdr*>(h->scan_hdr.p);
  int32_t* cnt = static_cast<int32_t*>(h->scan_cnt.p);
  int64_t* off = static_cast<int64_t*>(h->scan_off.p);
  int64_t* word_off = list ? static_cast<int64_t*>(h->scan_word_off.p) : nullptr;
  int32_t* us = static_cast<int32_t*>(h->scan_start.p);
  int32_t* ue = static_cast<int32_t*>(h->scan_end.p);
  int64_t* pages = list ? static_cast<int64_t*>(h->scan_pages.p) : nullptr;
  const int wide = 4 * (h->num_sms > 0 ? h->num_sms : 1);
  auto blocks = [&](int64_t items) { return int((items + 255) / 256 < wide ? (items + 255) / 256 : wide); };
  if (int e = check_cuda(h, cudaMemsetAsync(hdr, 0, sizeof(ScanHdr), s), "scan plan: memset")) return e;
  scan_union_kernel<<<blocks(words), 256, 0, s>>>(allow, mask_index, n_q, c.n_pages, page_start, u, hdr);
  scan_count_kernel<<<blocks(n_full), 256, 0, s>>>(n_full, unit_start, chunk_page, page_start, u, hdr, h->num_sms,
                                                  h->unit_rows, cnt);
  scan_offsets_kernel<<<1, kScanThreads, 0, s>>>(cnt, n_full, off, u, words, word_off, hdr);
  scan_write_kernel<<<blocks(list && words > n_full ? words : n_full), 256, 0, s>>>(
      n_full, unit_start, chunk_page, page_start, u, hdr, h->num_sms, h->unit_rows, off, us, ue, words, word_off, pages);
  h->launches += 4;
  if (int e = check_cuda(h, cudaGetLastError(), "launch scan plan")) return e;
  plan->start = us;
  plan->end = ue;
  plan->n_units = int(c.n_pages);
  plan->n_units_dev = &hdr->n_units;
  plan->pages = pages;
  plan->n_pages_dev = list ? &hdr->n_allowed : nullptr;
  plan->slot_mode = 0;
  return B200MS_OK;
}

int read_scan_stats(b200ms_t* h, int64_t* units, int64_t* rows) {
  ScanHdr hdr{h->corpus.n_units, 0, (unsigned long long)h->corpus.n_rows};
  if (h->scan_planned)
    if (int e = check_cuda(h, cudaMemcpy(&hdr, h->scan_hdr.p, sizeof(hdr), cudaMemcpyDeviceToHost), "last_scan_stats: copy"))
      return e;
  if (units) *units = hdr.n_units;
  if (rows) *rows = int64_t(hdr.rows);
  return B200MS_OK;
}

}  // namespace bms
