// api.cu -- the extern "C" surface declared in include/b200ms.h: handle management, corpus attachment
// (chunk table, work-unit plan, TMA descriptor), query packing and the fused search entry points.
// Host-side C++ only orchestrates; all arithmetic on embeddings happens in the CUDA kernels.
// (Multi-GPU entry points -- NCCL communicator, all-gather of top-k lists, pipelined sharded search -- live in comm.cu.)
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "common.cuh"

namespace bms {

static std::mutex g_err_mu;
static std::string g_err;

static const char* const kHostFullScan =
    "host-resident corpus (b200ms_set_corpus_host): only candidate scoring (b200ms_rerank_device / b200ms_rerank_batch_device) "
    "is supported; full scans would stream the whole corpus over PCIe";

int set_error(b200ms_t* h, int code, const std::string& msg) {
  if (h) h->err = msg;
  std::lock_guard<std::mutex> lk(g_err_mu);
  g_err = msg;
  return code;
}

int check_cuda(b200ms_t* h, cudaError_t e, const char* what) {
  if (e == cudaSuccess) return B200MS_OK;
  // a failed runtime call (e.g. cudaFuncSetAttribute) also leaves its error as the thread's last error: clear it, or the
  // next launch check on this thread -- in any later call -- would report it as its own failure
  cudaGetLastError();
  return set_error(h, B200MS_ECUDA, std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")");
}

int reserve(b200ms_t* h, DeviceBuf& b, size_t bytes) {
  if (bytes <= b.cap) return B200MS_OK;
  if (h) {
    if (h->capturing) return set_error(h, B200MS_ESTATE, "scratch buffer would grow inside a graph capture");
    h->generation++;  // captured graphs hold the old address
  }
  if (b.p) cudaFree(b.p);
  b.p = nullptr;
  b.cap = 0;
  size_t want = bytes + bytes / 4;
  want = (want + 1023) & ~size_t(1023);
  if (cudaMalloc(&b.p, want) != cudaSuccess) {
    cudaGetLastError();
    want = (bytes + 1023) & ~size_t(1023);
    if (cudaError_t e = cudaMalloc(&b.p, want); e != cudaSuccess) {
      b.p = nullptr;
      cudaGetLastError();
      return set_error(h, B200MS_ENOMEM, "cudaMalloc of " + std::to_string(want) + " scratch bytes failed");
    }
  }
  b.cap = want;
  return B200MS_OK;
}

int reserve_pinned(b200ms_t* h, PinnedBuf& b, size_t bytes) {
  if (bytes <= b.cap) return B200MS_OK;
  if (h) h->generation++;
  if (b.p) cudaFreeHost(b.p);
  b.p = nullptr;
  b.cap = 0;
  const size_t want = ((bytes + bytes / 4) + 4095) & ~size_t(4095);
  // cudaHostAllocMapped: with unified addressing the same pointer is valid in kernels (zero-copy reads / writes over PCIe)
  if (cudaError_t e = cudaHostAlloc(&b.p, want, cudaHostAllocMapped | cudaHostAllocPortable); e != cudaSuccess) {
    b.p = nullptr;
    cudaGetLastError();
    return set_error(h, B200MS_ENOMEM, "cudaHostAlloc of " + std::to_string(want) + " pinned bytes failed");
  }
  b.cap = want;
  return B200MS_OK;
}

// MaxDynamicSharedMemorySize is a property of the FUNCTION in the device's context, shared by every handle of the process:
// it must only ever be raised.  (A per-handle cache let a second handle "set" a small value for the merge kernel and thereby
// LOWER the limit a first handle relied on -- its next large merge then failed with cudaErrorInvalidValue.)  Launches that fit
// the 48 KB default need no call at all.
int ensure_smem(b200ms_t* h, const void* kernel, int smem, const char* what) {
  if (smem <= 16 * 1024) return B200MS_OK;  // static + dynamic cannot pass the 48 KB default below this
  struct Entry {
    int static_bytes;
    int raised;  // largest MaxDynamicSharedMemorySize set so far (0 = never set)
  };
  static std::mutex mu;
  static std::unordered_map<uint64_t, Entry> table;  // (device, kernel)
  const uint64_t key = (uint64_t(uint32_t(h ? h->device : 0)) << 56) ^ uint64_t(reinterpret_cast<uintptr_t>(kernel));
  std::lock_guard<std::mutex> lk(mu);
  auto it = table.find(key);
  if (it == table.end()) {
    cudaFuncAttributes fa;
    if (int e = check_cuda(h, cudaFuncGetAttributes(&fa, kernel), what)) return e;
    it = table.emplace(key, Entry{int(fa.sharedSizeBytes), 0}).first;
  }
  Entry& en = it->second;
  // the default limit (48 KB) covers the kernel's STATIC shared memory as well as the dynamic request
  if (en.raised == 0 && smem + en.static_bytes <= 48 * 1024) return B200MS_OK;
  if (en.raised >= smem) return B200MS_OK;
  if (int e = check_cuda(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), what)) return e;
  en.raised = smem;
  return B200MS_OK;
}

int upload(b200ms_t* h, DeviceBuf& b, const void* src, size_t bytes, cudaStream_t s) {
  if (int e = reserve(h, b, bytes ? bytes : 16)) return e;
  if (bytes == 0) return B200MS_OK;
  return check_cuda(h, cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, s), "upload metadata");
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Resolved once per process, thread-safe (handles on different threads may attach corpora concurrently).
static EncodeTiledFn encode_fn(b200ms_t* h) {
  static std::once_flag once;
  static EncodeTiledFn fn = nullptr;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess && p) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    } else {
      cudaGetLastError();
    }
  });
  if (!fn) set_error(h, B200MS_ECUDA, "cuTensorMapEncodeTiled not available from the driver");
  return fn;
}

// [n_rows, row_bytes] row-major view; box = one 128-byte K panel x box_rows rows, 128-byte swizzle (what the wgmma
// K-major SWIZZLE_128B descriptor expects).  Out-of-range rows read as zero.  row_bytes is 256 for bf16 rows and 128 for
// the one-byte dtypes by default; the FDE matrix passes its own (fde_dim * 2).
int make_tmap_rows(b200ms_t* h, CUtensorMap* out, const void* base, int dtype, int64_t n_rows, int box_rows, int64_t row_bytes) {
  EncodeTiledFn fn = encode_fn(h);
  if (!fn) return B200MS_ECUDA;
  const bool bf16 = dtype == B200MS_BF16;
  if (row_bytes <= 0) row_bytes = bf16 ? 256 : 128;
  const cuuint64_t dims[2] = {cuuint64_t(bf16 ? row_bytes / 2 : row_bytes), cuuint64_t(n_rows > 0 ? n_rows : 1)};
  const cuuint64_t strides[1] = {cuuint64_t(row_bytes)};
  const cuuint32_t box[2] = {cuuint32_t(bf16 ? 64 : 128), cuuint32_t(box_rows)};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(out, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2,
                        const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(h, B200MS_ECUDA, "cuTensorMapEncodeTiled failed with CUresult " + std::to_string(int(r)));
  return B200MS_OK;
}

static bool corpus_dtype_ok(int d) { return d == B200MS_BF16 || d == B200MS_I8 || d == B200MS_B1 || d == B200MS_F8; }
static bool src_dtype_ok(int d) { return d == B200MS_F32 || d == B200MS_BF16; }

DeviceGuard::DeviceGuard(int dev) {
  cudaGetDevice(&prev);
  if (prev != dev) cudaSetDevice(dev);
}
DeviceGuard::~DeviceGuard() {
  int cur = -1;
  cudaGetDevice(&cur);
  if (prev >= 0 && cur != prev) cudaSetDevice(prev);
}

StreamOrder::StreamOrder(b200ms_t* h, cudaStream_t s) : h_(h), s_(s) {
  if (h->capturing) return;
  if (s != h->stream) {  // the handle's own stream is only ever captured inside run_host_graph (h->capturing)
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &st) != cudaSuccess) {  // the legacy stream while another stream captures globally
      cudaGetLastError();
      return;
    }
    if (st != cudaStreamCaptureStatusNone) return;
  }
  if (h->order_pending && s != h->order_stream)
    err_ = check_cuda(h, cudaStreamWaitEvent(s, h->order_ev, 0), "wait for the handle's previous call");
  active_ = err_ == B200MS_OK;
}

StreamOrder::~StreamOrder() {
  if (!active_) return;
  if (synced_) {
    h_->order_pending = false;
  } else if (cudaEventRecord(h_->order_ev, s_) == cudaSuccess) {
    h_->order_stream = s_;
    h_->order_pending = true;
  } else {
    cudaGetLastError();
  }
}

void group_tokens(const int32_t* lens, int64_t n, const int32_t* goff, int64_t n_groups, int32_t* ntok) {
  for (int64_t i = 0; i < n; ++i) {
    int64_t left = lens[i];
    for (int64_t g = goff[i]; g < goff[i + 1] && g < n_groups; ++g) {
      ntok[g] = int32_t(left > kGroup ? kGroup : left);
      left -= ntok[g];
    }
  }
}

SearchMeta build_search_meta(const int32_t* lens, int64_t n, bool with_groups) {
  SearchMeta m;
  if (!lens || n < 0) n = 0;
  const size_t n1 = size_t(n) + 1;
  m.n = n;
  m.off_ds = n1 * 8;
  m.off_goff = 2 * n1 * 8;
  m.off_ntok = m.off_goff + ((n1 * 4 + 15) & ~size_t(15));
  if (with_groups) {
    m.groups = b200ms_query_groups(lens, int(n));
    m.groups_padded = groups_padded(m.groups);
  }
  m.host.assign(with_groups ? m.off_ntok + size_t(m.groups_padded > 0 ? m.groups_padded : 4) * 4 : m.off_goff, 0);
  int64_t* ss = reinterpret_cast<int64_t*>(m.host.data());
  int64_t* ds = reinterpret_cast<int64_t*>(m.host.data() + m.off_ds);
  for (int64_t i = 0; i < n; ++i) {
    const int64_t len = lens[i] > 0 ? lens[i] : 0;
    ss[i + 1] = ss[i] + len;
    ds[i + 1] = ds[i] + b200ms_padded_len(len);
  }
  m.rows = ss[n];
  m.padded_rows = ds[n];
  if (with_groups) {
    int32_t* goff = reinterpret_cast<int32_t*>(m.host.data() + m.off_goff);
    for (int64_t i = 0; i <= n; ++i) goff[i] = int32_t(ds[i] / kGroup);
    group_tokens(lens, n, goff, m.groups, reinterpret_cast<int32_t*>(m.host.data() + m.off_ntok));
  }
  return m;
}

}  // namespace bms

using namespace bms;

// search_core of a device entry point, ordered after the handle's previous call
static int search_ordered(b200ms_t* h, const SearchRequest& r, cudaStream_t s) {
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  return search_core(h, r, build_search_meta(r.q_lens, r.n_q), s);
}

#define B200MS_API extern "C" __attribute__((visibility("default")))

B200MS_API int b200ms_version(void) { return B200MS_VERSION; }

B200MS_API int b200ms_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

B200MS_API const char* b200ms_last_error(const b200ms_t* h) {
  if (h) return h->err.c_str();
  std::lock_guard<std::mutex> lk(g_err_mu);
  return g_err.c_str();
}

B200MS_API int b200ms_create(int device, b200ms_t** out) {
  if (!out) return set_error(nullptr, B200MS_EINVAL, "create: out is NULL");
  *out = nullptr;
  int n = 0;
  if (cudaError_t e = cudaGetDeviceCount(&n); e != cudaSuccess || n == 0) {
    cudaGetLastError();
    return set_error(nullptr, B200MS_ECUDA, "create: no CUDA device available (this library has no CPU fallback)");
  }
  if (device < 0 || device >= n) return set_error(nullptr, B200MS_EINVAL, "create: bad device index");
  DeviceGuard g(device);
  cudaDeviceProp prop;
  if (int e = check_cuda(nullptr, cudaGetDeviceProperties(&prop, device), "cudaGetDeviceProperties")) return e;
  if (prop.major != 9 || prop.minor != 0) {
    return set_error(nullptr, B200MS_ECUDA, std::string("create: device is sm_") + std::to_string(prop.major * 10 + prop.minor) +
                                                ", this library is built for sm_90a (H100) only");
  }
  b200ms_t* h = new b200ms_t();
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  h->smem_optin = int(prop.sharedMemPerBlockOptin);
  if (const char* e = getenv("B200MS_B1_TENSOR")) h->b1_tensor = atoi(e);
  if (const char* e = getenv("B200MS_ZERO_COPY")) h->zero_copy = atoi(e);
  if (const char* e = getenv("B200MS_UNIT_ROWS")) { if (atoll(e) > 0) h->unit_rows = atoll(e); }
  if (int e = check_cuda(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking), "cudaStreamCreate")) {
    delete h;
    return e;
  }
  if (int e = check_cuda(h, cudaEventCreateWithFlags(&h->order_ev, cudaEventDisableTiming), "create: cudaEventCreate")) {
    b200ms_destroy(h);
    return e;
  }
  for (int i = 0; i < b200ms_t::kEvRing; ++i) {
    if (cudaEventCreate(&h->ev0[i]) != cudaSuccess || cudaEventCreate(&h->ev1[i]) != cudaSuccess) {
      const int e = check_cuda(nullptr, cudaGetLastError(), "create: cudaEventCreate");
      b200ms_destroy(h);
      return e ? e : B200MS_ECUDA;
    }
  }
  *out = h;
  return B200MS_OK;
}

B200MS_API int b200ms_destroy(b200ms_t* h) {
  if (!h) return B200MS_OK;
  DeviceGuard g(h->device);
  cudaDeviceSynchronize();
  comm_teardown(h);
  for (auto& g2 : h->host_graphs)
    if (g2.exec) cudaGraphExecDestroy(g2.exec);
  DeviceBuf* bufs[] = {&h->chunk_page, &h->unit_start, &h->page_start, &h->page_len, &h->clamp_pages, &h->clamp_slots,
                       &h->meta, &h->meta_b, &h->q_raw, &h->q_packed, &h->scores, &h->mask, &h->mask_index, &h->out_all,
                       &h->cand_pad, &h->cand_start, &h->cand_end, &h->cand_mask, &h->topk_keys, &h->topk_ids, &h->docs_best, &h->docs_mask, &h->docs_top, &h->docs_pick, &h->b1_q_i8, &h->b1_tok_const, &h->f8_q_f16,
                       &h->fde_simhash, &h->fde_ams_index, &h->fde_ams_sign, &h->fde_tmp, &h->fde_q_bf16, &h->fde_final_index,
                       &h->fde_final_sign, &h->ht_bitmap, &h->ht_wpre, &h->ht_uniq, &h->ht_stage_off, &h->ht_hdr,
                       &h->ht_remap, &h->ht_ps, &h->ht_chunk_page, &h->ht_scores, &h->ht_stage, &h->scan_union, &h->scan_cnt,
                       &h->scan_off, &h->scan_start, &h->scan_end, &h->scan_hdr, &h->scan_word_off, &h->scan_pages,
                       &h->compact_meta, &h->compact_bounce, &h->mmr_state, &h->mmr_partials, &h->src_pages,
                       &h->ex_meta, &h->ex_lists, &h->ex_fused, &h->ex_union, &h->dm_table, &h->dm_scores, &h->dm_allow, &h->dup_cols};
  for (DeviceBuf* b : bufs)
    if (b->p) cudaFree(b->p);
  release_blocks(h);
  for (cudaEvent_t e : h->ht_ev) cudaEventDestroy(e);
  if (h->stage.p) cudaFreeHost(h->stage.p);
  for (int i = 0; i < b200ms_t::kEvRing; ++i) {
    if (h->ev0[i]) cudaEventDestroy(h->ev0[i]);
    if (h->ev1[i]) cudaEventDestroy(h->ev1[i]);
  }
  if (h->order_ev) cudaEventDestroy(h->order_ev);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return B200MS_OK;
}

B200MS_API int64_t b200ms_padded_len(int64_t len) { return len <= 0 ? 0 : (len + kGroup - 1) / kGroup * kGroup; }

B200MS_API int64_t b200ms_padded_rows(const int32_t* page_lens, int64_t n_pages) {
  int64_t t = 0;
  for (int64_t i = 0; i < n_pages; ++i) t += b200ms_padded_len(page_lens[i]);
  return t;
}

B200MS_API int64_t b200ms_row_bytes(int dtype) {
  switch (dtype) {
    case B200MS_F32: return 512;
    case B200MS_BF16: return 256;
    case B200MS_I8: return 128;
    case B200MS_F8: return 128;
    case B200MS_B1: return 16;
    default: return 0;
  }
}

B200MS_API int64_t b200ms_query_groups(const int32_t* q_lens, int n_q) {
  int64_t g = 0;
  for (int i = 0; i < n_q; ++i) g += (int64_t(q_lens[i] > 0 ? q_lens[i] : 0) + kGroup - 1) / kGroup;
  return g;
}

B200MS_API int64_t b200ms_launch_count(const b200ms_t* h) { return h ? h->launches : 0; }

B200MS_API int b200ms_set_option(b200ms_t* h, const char* name, int64_t value) {
  if (!h || !name) return B200MS_EINVAL;
  const std::string n(name);
  if (n == "b1_tensor" && value >= 0 && value <= 2) {
    h->b1_tensor = int(value);
  } else if (n == "zero_pad_compat" && value >= 0 && value <= (int64_t(1) << 30)) {
    h->zero_pad_batch = int(value);
  } else if (n == "zero_copy" && value >= 0 && value <= 1) {
    h->zero_copy = int(value);
  } else if (n == "fde_gemm" && value >= 0 && value <= 1) {
    h->fde_gemm = int(value);
  } else if (n == "host_graph" && value >= 0 && value <= 1) {
    h->host_graph = int(value);
  } else if (n == "unit_rows" && value > 0) {
    h->unit_rows = value;
  } else if (n == "max_ctas" && value >= 0) {
    h->max_ctas = int(value);
  } else if (n == "host_stage_bytes" && value > 0) {
    h->host_stage_bytes = value;
  } else {
    return set_error(h, B200MS_EINVAL, "set_option: unknown option or bad value: " + n);
  }
  h->generation++;
  return B200MS_OK;
}

B200MS_API int b200ms_set_tuning(b200ms_t* h, int64_t unit_rows, int max_ctas) {
  if (!h) return B200MS_EINVAL;
  if (unit_rows > 0)
    if (int e = b200ms_set_option(h, "unit_rows", unit_rows)) return e;
  if (max_ctas >= 0) return b200ms_set_option(h, "max_ctas", max_ctas);
  return B200MS_OK;
}

B200MS_API int64_t b200ms_corpus_pages(const b200ms_t* h) { return h ? h->corpus.n_pages : 0; }
B200MS_API int64_t b200ms_corpus_rows(const b200ms_t* h) { return h ? h->corpus.n_rows : 0; }

// ------------------------------------------------------------------------------------------------ quantise / pack
// Pack the items of m (queries: up to groups_padded * 32 rows, tail rows zeroed; pages: m.padded_rows) with one upload of
// m's [ss | ds] part.  m is pageable host memory: cudaMemcpyAsync staged it before returning, so it may die afterwards.
static int pack_items(b200ms_t* h, const void* src, int src_dtype, const SearchMeta& m, bool queries, void* dst, int dst_dtype,
                      float i8_scale, cudaStream_t s) {
  if (int e = upload(h, h->meta_b, m.host.data(), m.off_goff, s)) return e;
  const int64_t* dev = static_cast<const int64_t*>(h->meta_b.p);
  return launch_pack_rows(h, src, src_dtype, dev, dev + m.n + 1, m.n, queries ? m.groups_padded * kGroup : m.padded_rows,
                          queries ? 1 : 0, dst, dst_dtype, i8_scale, s);
}

B200MS_API int b200ms_sign_pack(b200ms_t* h, const void* x, int src_dtype, int64_t rows, uint8_t* out, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (!src_dtype_ok(src_dtype) || rows < 0 || (rows > 0 && (!x || !out)))
    return set_error(h, B200MS_EINVAL, "sign_pack: bad arguments");
  if (rows == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  const int64_t st[2] = {0, rows};
  if (int e = upload(h, h->meta_b, st, sizeof(st), s)) return e;
  const int64_t* d = static_cast<const int64_t*>(h->meta_b.p);
  return launch_pack_rows(h, x, src_dtype, d, d, 1, rows, 0, out, B200MS_B1, 1.f, s);
}

B200MS_API int b200ms_hamming_batch(b200ms_t* h, const uint8_t* q_bits, const uint8_t* cand_bits, int64_t n, uint32_t* out,
                                    void* stream) {
  if (!h) return B200MS_EINVAL;
  if (n < 0 || (n > 0 && (!q_bits || !cand_bits || !out)) || (reinterpret_cast<uintptr_t>(q_bits) & 15) ||
      (reinterpret_cast<uintptr_t>(cand_bits) & 15))
    return set_error(h, B200MS_EINVAL, "hamming_batch: bad arguments (16-byte aligned packed rows)");
  DeviceGuard g(h->device);
  StreamOrder order(h, static_cast<cudaStream_t>(stream));
  if (int e = order.error()) return e;
  return launch_hamming_batch(h, q_bits, cand_bits, n, out, static_cast<cudaStream_t>(stream));
}

B200MS_API int b200ms_pack_pages(b200ms_t* h, const void* src, int src_dtype, const int32_t* page_lens, int64_t n_pages,
                                 void* dst, int dst_dtype, float i8_scale, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (!src_dtype_ok(src_dtype) || !corpus_dtype_ok(dst_dtype) || n_pages < 0 || (n_pages > 0 && (!page_lens || !dst)))
    return set_error(h, B200MS_EINVAL, "pack_pages: bad arguments");
  if (n_pages == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  StreamOrder order(h, static_cast<cudaStream_t>(stream));
  if (int e = order.error()) return e;
  return pack_items(h, src, src_dtype, build_search_meta(page_lens, n_pages, false), false, dst, dst_dtype, i8_scale,
                    static_cast<cudaStream_t>(stream));
}

B200MS_API int b200ms_pack_queries(b200ms_t* h, const void* q, int src_dtype, const int32_t* q_lens, int n_q,
                                   void* q_packed, int dst_dtype, float i8_scale, int32_t* group_offsets_out,
                                   int* n_groups_out, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (!src_dtype_ok(src_dtype) || !corpus_dtype_ok(dst_dtype) || n_q < 0 || (n_q > 0 && (!q_lens || !q_packed)))
    return set_error(h, B200MS_EINVAL, "pack_queries: bad arguments");
  DeviceGuard g(h->device);
  StreamOrder order(h, static_cast<cudaStream_t>(stream));
  if (int e = order.error()) return e;
  const SearchMeta m = build_search_meta(q_lens, n_q);
  if (m.groups_padded > 0)
    if (int e = pack_items(h, q, src_dtype, m, true, q_packed, dst_dtype, i8_scale, static_cast<cudaStream_t>(stream))) return e;
  if (group_offsets_out) memcpy(group_offsets_out, m.goff(), (size_t(n_q) + 1) * 4);
  if (n_groups_out) *n_groups_out = int(m.groups);
  return B200MS_OK;
}

// ------------------------------------------------------------------------------------------------ corpus
// ps_host: the corpus' padded page offsets [n_pages + 1]; page_start must already hold them on the device (ordered before s)
int bms::build_scan_tables(b200ms_t* h, Corpus& c, const int64_t* ps_host, cudaStream_t s) {
  // work units: runs of whole pages of about unit_rows rows; unit_start in chunks
  // (small corpora: shrink the units so that every SM still gets about four of them -- a 100-page corpus as 25 units
  // of 4096 rows would leave 123 SMs idle)
  int64_t unit_rows = c.n_rows / (4 * int64_t(h->num_sms > 0 ? h->num_sms : 1));
  if (unit_rows < kTileN) unit_rows = kTileN;
  if (unit_rows > h->unit_rows) unit_rows = h->unit_rows;
  std::vector<int32_t> us;
  us.push_back(0);
  int64_t acc = 0;
  for (int64_t i = 0; i < c.n_pages; ++i) {
    acc += ps_host[i + 1] - ps_host[i];
    if (acc >= unit_rows) {
      us.push_back(int32_t(ps_host[i + 1] / kGroup));
      acc = 0;
    }
  }
  if (us.back() != int32_t(c.n_chunks)) us.push_back(int32_t(c.n_chunks));
  c.n_units = int(us.size()) - 1;
  if (int e = upload(h, h->unit_start, us.data(), us.size() * 4, s)) return e;
  if (int e = reserve(h, h->chunk_page, size_t(c.n_chunks > 0 ? c.n_chunks : 1) * 4)) return e;
  if (int e = reserve_scan_plan(h, c)) return e;
  if (int e = launch_chunk_page(h, static_cast<const int64_t*>(h->page_start.p), c.n_pages,
                                static_cast<int32_t*>(h->chunk_page.p), s))
    return e;
  c.scan_tables = true;
  return B200MS_OK;
}

// Page tables of a corpus; an HBM corpus also gets its work-unit plan, chunk table and TMA descriptor.  A host-resident one
// (rows = the device address of mapped pinned memory) is only ever read by the candidate gather, which needs page_start.
static int attach_corpus(b200ms_t* h, const void* rows, int dtype, const int32_t* page_lens, int64_t n_pages, bool host) {
  DeviceGuard g(h->device);
  cudaStream_t s = h->stream;
  StreamOrder order(h, s);  // a call still in flight may read the tables rewritten below
  if (int e = order.error()) return e;
  Corpus c;
  c.rows = rows;
  c.dtype = dtype;
  c.n_pages = n_pages;
  c.host = host;
  std::vector<int64_t> ps(size_t(n_pages) + 1);
  ps[0] = 0;
  for (int64_t i = 0; i < n_pages; ++i) {
    ps[i + 1] = ps[i] + b200ms_padded_len(page_lens[i]);
    if (page_lens[i] <= 0) c.has_empty = true;
    if (ps[i + 1] - ps[i] > c.max_page_rows) c.max_page_rows = ps[i + 1] - ps[i];
  }
  c.n_rows = ps[n_pages];
  c.n_chunks = c.n_rows / kGroup;
  if (c.n_chunks >= (int64_t(1) << 31)) return set_error(h, B200MS_EINVAL, "set_corpus: more than 2^31 chunks");
  if (int e = upload(h, h->page_start, ps.data(), ps.size() * 8, s)) return e;
  if (int e = upload(h, h->page_len, page_lens, size_t(n_pages) * 4, s)) return e;
  h->page_len_host.assign(page_lens, page_lens + n_pages);
  if (host) {
    if (int e = check_cuda(h, cudaStreamSynchronize(s), "set_corpus_host: stream sync")) return e;
    order.finished();
    h->corpus = c;
    h->generation++;
    return B200MS_OK;
  }
  if (int e = build_scan_tables(h, c, ps.data(), s)) return e;
  if (dtype != B200MS_B1 && c.n_rows > 0) {
    if (int e = make_tmap_rows(h, &c.tmap, rows, dtype, c.n_rows, kTileN)) return e;
    c.has_tmap = true;
  }
  if (int e = check_cuda(h, cudaStreamSynchronize(s), "set_corpus: stream sync")) return e;
  order.finished();
  h->corpus = c;
  h->generation++;
  return B200MS_OK;
}

B200MS_API int b200ms_set_corpus(b200ms_t* h, const void* rows, int dtype, const int32_t* page_lens, int64_t n_pages) {
  if (!h) return B200MS_EINVAL;
  if (!corpus_dtype_ok(dtype) || n_pages < 0 || (n_pages > 0 && (!rows || !page_lens)))
    return set_error(h, B200MS_EINVAL, "set_corpus: bad arguments");
  if (n_pages > 0 && (reinterpret_cast<uintptr_t>(rows) & 1023))
    return set_error(h, B200MS_EINVAL, "set_corpus: rows must be 1024-byte aligned");
  return attach_corpus(h, rows, dtype, page_lens, n_pages, false);
}

B200MS_API int b200ms_set_corpus_host(b200ms_t* h, const void* rows_host, int dtype, const int32_t* page_lens, int64_t n_pages) {
  if (!h) return B200MS_EINVAL;
  if (!corpus_dtype_ok(dtype) || n_pages < 0 || (n_pages > 0 && (!rows_host || !page_lens)))
    return set_error(h, B200MS_EINVAL, "set_corpus_host: bad arguments");
  if (reinterpret_cast<uintptr_t>(rows_host) & 15)
    return set_error(h, B200MS_EINVAL, "set_corpus_host: rows must be 16-byte aligned");
  DeviceGuard g(h->device);
  const void* dev = nullptr;
  if (rows_host) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, rows_host) != cudaSuccess) {
      cudaGetLastError();
      return set_error(h, B200MS_EINVAL, "set_corpus_host: cudaPointerGetAttributes failed on rows");
    }
    if (a.type != cudaMemoryTypeHost || !a.devicePointer)
      return set_error(h, B200MS_EINVAL, "set_corpus_host: rows must be pinned, device-mapped host memory (b200ms_host_alloc)");
    dev = a.devicePointer;
  }
  return attach_corpus(h, dev, dtype, page_lens, n_pages, true);
}

B200MS_API int b200ms_host_alloc(b200ms_t* h, int64_t bytes, void** out) {
  if (!h) return B200MS_EINVAL;
  if (!out || bytes < 0) return set_error(h, B200MS_EINVAL, "host_alloc: bad arguments");
  *out = nullptr;
  DeviceGuard g(h->device);
  // exact size: the caller's corpus may be most of host RAM
  if (cudaError_t e = cudaHostAlloc(out, size_t(bytes > 0 ? bytes : 16), cudaHostAllocMapped | cudaHostAllocPortable);
      e != cudaSuccess) {
    *out = nullptr;
    cudaGetLastError();
    return set_error(h, B200MS_ENOMEM, "cudaHostAlloc of " + std::to_string(bytes) + " pinned bytes failed");
  }
  return B200MS_OK;
}

B200MS_API int b200ms_host_free(b200ms_t* h, void* p) {
  if (!p) return B200MS_OK;
  if (!h) {  // the handle is already gone: pinned blocks are portable, any context frees them
    if (cudaFreeHost(p) == cudaSuccess) return B200MS_OK;
    return check_cuda(nullptr, cudaGetLastError(), "cudaFreeHost");
  }
  DeviceGuard g(h->device);
  return check_cuda(h, cudaFreeHost(p), "cudaFreeHost");
}

B200MS_API int b200ms_last_gather_stats(b200ms_t* h, int64_t* unique_pages, int64_t* bytes, int* rounds, float* ms) {
  if (!h) return B200MS_EINVAL;
  DeviceGuard g(h->device);
  float total = 0.f;
  for (int r = 0; r < h->ht_rounds; ++r) {
    float t = 0.f;
    if (cudaEventSynchronize(h->ht_ev[2 * r + 1]) != cudaSuccess ||
        cudaEventElapsedTime(&t, h->ht_ev[2 * r], h->ht_ev[2 * r + 1]) != cudaSuccess)
      return check_cuda(h, cudaGetLastError(), "last_gather_stats: gather events");
    total += t;
  }
  if (unique_pages) *unique_pages = h->ht_unique;
  if (bytes) *bytes = h->ht_bytes;
  if (rounds) *rounds = h->ht_rounds;
  if (ms) *ms = total;
  return B200MS_OK;
}

B200MS_API int b200ms_last_scan_stats(b200ms_t* h, int64_t* units, int64_t* rows) {
  if (!h) return B200MS_EINVAL;
  DeviceGuard g(h->device);
  if (h->order_pending)
    if (int e = check_cuda(h, cudaEventSynchronize(h->order_ev), "last_scan_stats: wait for the scan")) return e;
  return read_scan_stats(h, units, rows);
}

// zero_pad_compat, full scan: pages are "batched" in page-id order, zero_pad_batch at a time (score_multi_vector's
// batch_size, 128 upstream); a page shorter than the longest of its batch gets its per-token maxima clamped at 0.
// Built on the host once per (corpus, batch size) and cached on the device.
static int ensure_clamp_pages(b200ms_t* h, cudaStream_t s, const uint32_t** out) {
  *out = nullptr;
  if (h->zero_pad_batch <= 0 || h->corpus.dtype == B200MS_B1) return B200MS_OK;  // SQL max_sim has no padding quirk
  Corpus& c = h->corpus;
  const int64_t n = c.n_pages;
  if (c.clamp_batch != h->zero_pad_batch) {
    std::vector<uint32_t> bits(size_t((n + 31) / 32) + 1, 0u);
    const int64_t B = h->zero_pad_batch;
    for (int64_t b0 = 0; b0 < n; b0 += B) {
      const int64_t b1 = b0 + B < n ? b0 + B : n;
      int32_t mx = 0;
      for (int64_t p = b0; p < b1; ++p) mx = h->page_len_host[p] > mx ? h->page_len_host[p] : mx;
      for (int64_t p = b0; p < b1; ++p)
        if (h->page_len_host[p] < mx) bits[size_t(p >> 5)] |= 1u << (p & 31);
    }
    if (int e = upload(h, h->clamp_pages, bits.data(), bits.size() * 4, s)) return e;
    c.clamp_batch = h->zero_pad_batch;
  }
  *out = static_cast<const uint32_t*>(h->clamp_pages.p);
  return B200MS_OK;
}

// ------------------------------------------------------------------------------------------------ hot path
// Candidate mode of the wgmma scorers: unit j = the chunk range of candidate slot j, scores indexed by j.  The units come
// from unit_ids, page ids of v (cs.ids, or their staging-block remap for a host-resident corpus); the zero_pad_compat
// clamp bits always come from cs.ids, the corpus page ids.
static int candidate_plan(b200ms_t* h, const CorpusView& v, const int64_t* unit_ids, const CandSpec& cs, int n_q,
                          bool zero_pad, cudaStream_t s, UnitPlan* plan) {
  const int n_slots = int(cs.n_slots(n_q));
  if (int e = reserve(h, h->cand_start, size_t(n_slots) * 4)) return e;
  if (int e = reserve(h, h->cand_end, size_t(n_slots) * 4)) return e;
  if (int e = launch_cand_units(h, v, unit_ids, n_slots, static_cast<int32_t*>(h->cand_start.p),
                                static_cast<int32_t*>(h->cand_end.p), nullptr, s))
    return e;
  plan->start = static_cast<const int32_t*>(h->cand_start.p);
  plan->end = static_cast<const int32_t*>(h->cand_end.p);
  plan->n_units = n_slots;
  plan->slot_mode = 1;
  if (zero_pad && h->zero_pad_batch > 0) {  // the reference's quirk, exactly: batches of zero_pad_batch candidates in first-stage order
    if (int e = reserve(h, h->clamp_slots, size_t((n_slots + 31) / 32 + 1) * 4)) return e;
    if (int e = launch_clamp_slots(h, cs.ids, cs.n_cand, cs.per_query ? n_q : 1, cs.stride(), h->zero_pad_batch,
                                   static_cast<uint32_t*>(h->clamp_slots.p), s))
      return e;
    plan->clamp_bits = static_cast<const uint32_t*>(h->clamp_slots.p);
  }
  return B200MS_OK;
}

// Per-query candidate lists on wgmma: one launch per 128-token query tile, the tile's queries against THEIR candidate
// lists only (a contiguous slot range).
static int score_wgmma_per_query(b200ms_t* h, const CorpusView& v, const UnitPlan& plan, const CandSpec& cs,
                                 const void* q_packed, int n_groups, const int32_t* goff, const int32_t* ntok_dev, int n_q,
                                 void* group_scores, int64_t ld, cudaStream_t s) {
  const int n_mtiles = int(groups_padded(n_groups)) / 4;
  int q_lo = 0;
  for (int m = 0; m < n_mtiles; ++m) {
    const int g0 = 4 * m, g1 = 4 * m + 4;
    while (q_lo < n_q && goff[q_lo + 1] <= g0) ++q_lo;  // first query with a group in this tile
    int q_hi = q_lo;
    while (q_hi < n_q && goff[q_hi] < g1) ++q_hi;        // one past the last
    if (q_hi <= q_lo) continue;
    UnitPlan sub = plan;
    const int64_t s0 = int64_t(q_lo) * cs.stride();
    sub.start += s0;
    sub.end += s0;
    sub.n_units = int(int64_t(q_hi - q_lo) * cs.stride());
    if (sub.clamp_bits) sub.clamp_bits += s0 / 32;
    void* sc = static_cast<uint8_t*>(group_scores) + size_t(s0) * 4;
    if (int e = launch_score_wgmma(h, v, sub, q_packed, n_groups, ntok_dev, sc, ld, s, m, m + 1)) return e;
  }
  return B200MS_OK;
}

// Scores the rows of v.  unit_ids: the candidate slots as page ids of v (cs.ids unless v is a staging block); fill = false
// skips the zero-fill (a later gather round of a host-resident corpus adds its slots to the same matrix).  scan (full scans
// only): the filtered plan to walk in place of the corpus' own; the scores of the pages it leaves out are not written.
// zero_pad = false: no zero_pad_compat clamp whatever the option says (page and example searches).
static int score_impl(b200ms_t* h, const void* q_packed, int n_groups, const int32_t* goff, int n_q, const int32_t* ntok_dev,
                      void* group_scores, int64_t ld, const CandSpec& cs, cudaStream_t s, const CorpusView& v,
                      const int64_t* unit_ids, bool fill = true, const UnitPlan* scan = nullptr, bool zero_pad = true) {
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "score: no corpus attached (call b200ms_set_corpus first)");
  const int64_t n_items = cs.ids ? cs.n_slots(n_q) : c.n_pages;
  if (n_groups < 0 || ld < n_items || cs.n_cand < 0 || (n_groups > 0 && (!q_packed || !group_scores)))
    return set_error(h, B200MS_EINVAL, "score: bad arguments");
  if (n_groups == 0 || n_items == 0 || c.n_pages == 0) return B200MS_OK;
  const bool b1 = c.dtype == B200MS_B1;
  if (b1 && (!goff || !ntok_dev || n_q <= 0)) return set_error(h, B200MS_EINVAL, "score: B1 needs the per-group token counts");
  // b1_tensor: 0 = POPC kernel, 1 = wgmma kernel (bits expanded to int8, maxsim_wgmma.cu), 2 (default) = by group count:
  // the POPC pipe costs one pass per 32-token group, the wgmma kernel about the same for up to 4 groups.  Full scans of
  // 65 536 pages x 1024 rows (tools/time_scan.py --b1-groups) on an NVIDIA H100 80GB HBM3 at a 700 W power limit: 1 group
  // 1.65 ms POPC vs 3.80 ms wgmma, 2 groups 3.16 vs 3.81, 3 groups 4.85 vs 3.81, 8 groups 12.76 vs 4.75.  Rerank of a
  // candidate list stays on the POPC kernel.
  const bool b1_wgmma = b1 && !cs.ids && (h->b1_tensor == 1 || (h->b1_tensor == 2 && n_groups >= 3));
  // zero-fill what no launch writes: the tile kernels skip pages with zero rows and unused candidate slots; the per-query
  // POPC launches write only their own query's groups and slots
  const bool zero_fill = b1 ? (b1_wgmma && c.has_empty) || cs.per_query : c.has_empty || cs.ids;
  if (zero_fill && fill)
    if (int e = zero_scores(h, group_scores, groups_padded(n_groups), ld, s, "score: memset")) return e;
  UnitPlan plan = scan ? *scan : full_scan_plan(h);
  if (!cs.ids) h->scan_planned = scan != nullptr;
  if (!b1) {
    if (int e = cs.ids    ? candidate_plan(h, v, unit_ids, cs, n_q, zero_pad, s, &plan)
                : zero_pad ? ensure_clamp_pages(h, s, &plan.clamp_bits)
                           : B200MS_OK)
      return e;
  }
  // ev0 / ev1 bracket the scoring launches only (b200ms_score_times_ms): bench.py derives the roofline's achieved figure
  // from this time
  const int slot = int(h->ev_count % b200ms_t::kEvRing);
  if (!h->capturing)
    if (int e = check_cuda(h, cudaEventRecord(h->ev0[slot], s), "score: event record")) return e;
  int e = B200MS_OK;
  if (b1_wgmma) {
    e = launch_score_b1_wgmma(h, plan, q_packed, ntok_dev, n_groups, group_scores, ld, s);
  } else if (b1 && cs.per_query) {
    for (int q = 0; q < n_q && !e; ++q)
      if (goff[q + 1] > goff[q])
        e = launch_score_b1(h, v, unit_ids + int64_t(q) * cs.stride(), cs.n_cand, q_packed, n_groups, ntok_dev,
                            static_cast<int32_t*>(group_scores) + int64_t(q) * cs.stride(), ld, s, goff[q], goff[q + 1]);
  } else if (b1) {
    e = launch_score_b1(h, v, unit_ids, cs.n_cand, q_packed, n_groups, ntok_dev, group_scores, ld, s, 0, n_groups, scan);
  } else if (cs.per_query) {
    e = score_wgmma_per_query(h, v, plan, cs, q_packed, n_groups, goff, ntok_dev, n_q, group_scores, ld, s);
  } else {
    e = launch_score_wgmma(h, v, plan, q_packed, n_groups, ntok_dev, group_scores, ld, s);
  }
  if (e) return e;
  if (!h->capturing) {
    if (int e2 = check_cuda(h, cudaEventRecord(h->ev1[slot], s), "score: event record")) return e2;
    h->ev_count++;
  }
  return B200MS_OK;
}

B200MS_API int b200ms_score(b200ms_t* h, const void* q_packed, int n_groups, const int32_t* q_lens,
                            const int32_t* group_offsets, int n_q, void* group_scores, int64_t ld, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (h->corpus.host) return set_error(h, B200MS_ESTATE, kHostFullScan);
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  const int32_t* ntok_dev = nullptr;  // dense corpora without q_lens / group_offsets: every packed row is a token
  if (h->corpus.dtype == B200MS_B1 && (!q_lens || !group_offsets || n_q <= 0))
    return set_error(h, B200MS_EINVAL, "score: B1 needs q_lens and group_offsets");
  if (q_lens && group_offsets && n_q > 0) {
    const int64_t gp = groups_padded(n_groups);
    std::vector<int32_t> ntok(size_t(gp > 0 ? gp : 4), 0);
    group_tokens(q_lens, n_q, group_offsets, n_groups, ntok.data());
    if (int e = upload(h, h->meta, ntok.data(), ntok.size() * 4, s)) return e;
    ntok_dev = static_cast<const int32_t*>(h->meta.p);
  }
  return score_impl(h, q_packed, n_groups, group_offsets, n_q, ntok_dev, group_scores, ld, CandSpec{}, s, corpus_view(h),
                    nullptr);
}

static int score_time_of(b200ms_t* h, int64_t idx, float* ms) {
  const int slot = int(idx % b200ms_t::kEvRing);
  if (cudaEventSynchronize(h->ev1[slot]) != cudaSuccess) return check_cuda(h, cudaGetLastError(), "cudaEventSynchronize");
  if (cudaEventElapsedTime(ms, h->ev0[slot], h->ev1[slot]) != cudaSuccess) return check_cuda(h, cudaGetLastError(), "cudaEventElapsedTime");
  return B200MS_OK;
}

B200MS_API float b200ms_last_score_ms(b200ms_t* h) {
  if (!h) return float(B200MS_EINVAL);
  if (h->ev_count == 0) return float(set_error(h, B200MS_ESTATE, "last_score_ms: no scoring call recorded"));
  DeviceGuard g(h->device);
  float ms = 0.f;
  if (int e = score_time_of(h, h->ev_count - 1, &ms)) return float(e);
  return ms;
}

B200MS_API int64_t b200ms_score_call_count(const b200ms_t* h) { return h ? h->ev_count : 0; }

B200MS_API int b200ms_score_times_ms(b200ms_t* h, float* out_ms, int n) {
  if (!h || !out_ms || n < 0) return B200MS_EINVAL;
  if (n > b200ms_t::kEvRing || n > h->ev_count) return set_error(h, B200MS_EINVAL, "score_times_ms: n exceeds the recorded history (ring of 256)");
  DeviceGuard g(h->device);
  for (int i = 0; i < n; ++i)
    if (int e = score_time_of(h, h->ev_count - n + i, &out_ms[i])) return e;
  return n;
}

// b200ms_topk / b200ms_topk_masked: allow = one mask (mask_index NULL) or a [n_masks, words] matrix with a row per query
static int topk_impl(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                     const int32_t* group_offsets, int n_q, const uint32_t* allow_mask, const int32_t* mask_index, int k,
                     float scale, int64_t id_base, float* top_scores, int64_t* top_ids, int32_t* top_counts, void* stream) {
  if ((score_dtype != B200MS_F32 && score_dtype != B200MS_I32) || n_pages < 0 || ld < n_pages || n_q < 0 || k < 1 ||
      k > B200MS_MAX_K || (n_q > 0 && (!group_offsets || !top_scores || !top_ids || !top_counts)) ||
      (n_q > 0 && n_pages > 0 && !group_scores))
    return set_error(h, B200MS_EINVAL, "topk: bad arguments (1 <= k <= 4096)");
  if (n_q == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  if (int e = upload(h, h->meta, group_offsets, size_t(n_q + 1) * 4, s)) return e;
  return launch_topk(h, group_scores, score_dtype, n_pages, ld, static_cast<const int32_t*>(h->meta.p), n_q, allow_mask,
                     k, scale, id_base, nullptr, top_scores, top_ids, top_counts, s, mask_index, (n_pages + 31) / 32);
}

B200MS_API int b200ms_topk(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                           const int32_t* group_offsets, int n_q, const uint32_t* allow_mask, int k, float scale,
                           int64_t id_base, float* top_scores, int64_t* top_ids, int32_t* top_counts, void* stream) {
  if (!h) return B200MS_EINVAL;
  return topk_impl(h, group_scores, score_dtype, n_pages, ld, group_offsets, n_q, allow_mask, nullptr, k, scale, id_base,
                   top_scores, top_ids, top_counts, stream);
}

B200MS_API int b200ms_topk_masked(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                                  const int32_t* group_offsets, int n_q, const uint32_t* allow_masks_dev, int n_masks,
                                  const int32_t* mask_index_dev, int k, float scale, int64_t id_base, float* top_scores,
                                  int64_t* top_ids, int32_t* top_counts, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  if (n_masks < 0 || (n_masks > 0 && (!allow_masks_dev || !mask_index_dev)))
    return set_error(h, B200MS_EINVAL, "topk_masked: n_masks > 0 needs the mask matrix and one index per query");
  return topk_impl(h, group_scores, score_dtype, n_pages, ld, group_offsets, n_q, n_masks > 0 ? allow_masks_dev : nullptr,
                   n_masks > 0 ? mask_index_dev : nullptr, k, scale, id_base, top_scores, top_ids, top_counts, cuda_stream);
}

B200MS_API int b200ms_merge_topk(b200ms_t* h, const float* cand_scores, const int64_t* cand_ids, int n_q, int m, int k,
                                 float* top_scores, int64_t* top_ids, int32_t* top_counts, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (n_q < 0 || m < 1 || m > 2 * B200MS_MAX_K || k < 1 || k > B200MS_MAX_K ||
      (n_q > 0 && (!cand_scores || !cand_ids || !top_scores || !top_ids || !top_counts)))
    return set_error(h, B200MS_EINVAL, "merge_topk: bad arguments (m <= 8192, k <= 4096)");
  DeviceGuard g(h->device);
  StreamOrder order(h, static_cast<cudaStream_t>(stream));
  if (int e = order.error()) return e;
  return launch_merge_topk(h, cand_scores, cand_ids, n_q, m, k, top_scores, top_ids, top_counts,
                           static_cast<cudaStream_t>(stream));
}

namespace bms {

int zero_scores(b200ms_t* h, void* scores, int64_t gp, int64_t ld, cudaStream_t s, const char* what) {
  return check_cuda(h, cudaMemsetAsync(scores, 0, size_t(gp) * size_t(ld) * 4, s), what);
}

// A filtered full scan reads only the pages some query of the call may see.  The other pages keep whatever the score matrix
// held before, and that is never read: the selection skips a page whose allow bit is clear before it touches the page's
// score, in the flat form (page_key) and in the document form (doc_item) alike.  A corpus whose own plan is one wave of
// units gains nothing from a shorter one, so it keeps it (and a small search its launch count).
int plan_full_scan(b200ms_t* h, const uint32_t* allow, const int32_t* mask_index, int n_q, cudaStream_t s, UnitPlan* plan) {
  *plan = full_scan_plan(h);
  h->scan_planned = allow && h->corpus.n_units > (h->max_ctas > 0 ? h->max_ctas : h->num_sms);
  return h->scan_planned ? launch_scan_plan(h, allow, mask_index, n_q, s, plan) : B200MS_OK;
}

int search_scan(b200ms_t* h, const SearchRequest& r, const SearchMeta& m, cudaStream_t s, const void* meta_dev, ScanResult* out) {
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, "search: no corpus attached (call b200ms_set_corpus first)");
  if (c.host && !r.cand.ids) return set_error(h, B200MS_ESTATE, kHostFullScan);
  if (c.host && h->capturing) return set_error(h, B200MS_ESTATE, "search: a host-resident corpus cannot be graph-captured");
  const int n_q = r.n_q;
  if (n_q < 1 || !r.q_lens || (!r.q && !r.src_pages) || r.k < 1 || r.k > B200MS_MAX_K || !r.top_scores || !r.top_ids || !r.top_counts)
    return set_error(h, B200MS_EINVAL, "search: bad arguments (n_q >= 1, 1 <= k <= 4096)");
  if (r.docs) {
    const DocSpec& d = *r.docs;
    if (!d.page_doc || !d.page_counts || d.per_doc < 1 || d.per_doc > B200MS_MAX_PER_DOC || d.n_docs < 0 ||
        (c.n_pages > 0 && d.n_docs < 1) || d.n_docs > c.n_pages || (r.cand.ids && !r.cand.per_query))
      return set_error(h, B200MS_EINVAL, "search_docs: bad arguments (page_doc and outputs, 1 <= per_doc <= 64, 1 <= n_docs <= n_pages)");
  }
  CandSpec cs = r.cand;
  if (cs.per_query && cs.stride() != cs.n_cand) {  // caller's lists are [n_q, n_cand]: give every list a 32-slot-aligned stride
    if (int e = reserve(h, h->cand_pad, size_t(cs.stride()) * size_t(n_q) * 8)) return e;
    if (int e = launch_pad_cands(h, r.cand.ids, cs.n_cand, n_q, cs.stride(), static_cast<int64_t*>(h->cand_pad.p), s)) return e;
    cs.ids = static_cast<const int64_t*>(h->cand_pad.p);
  }
  const int64_t n_items = cs.ids ? cs.n_slots(n_q) : c.n_pages;
  const auto [gp, ld] = score_layout(m, n_items);
  if (int e = reserve(h, h->q_packed, size_t(gp) * kGroup * size_t(b200ms_row_bytes(c.dtype)))) return e;
  if (int e = reserve(h, h->scores, size_t(gp) * size_t(ld) * 4)) return e;
  if (!meta_dev) {
    if (int e = upload(h, h->meta, m.host.data(), m.host.size(), s)) return e;
    meta_dev = h->meta.p;
  }
  const uint8_t* md = static_cast<const uint8_t*>(meta_dev);
  const int64_t* ss_dev = reinterpret_cast<const int64_t*>(md);
  const int64_t* ds_dev = reinterpret_cast<const int64_t*>(md + m.off_ds);
  const int32_t* goff_dev = reinterpret_cast<const int32_t*>(md + m.off_goff);
  const int32_t* ntok_dev = reinterpret_cast<const int32_t*>(md + m.off_ntok);
  if (m.groups_padded > 0) {  // query rows [0, ds[n_rows_q]), then the stored pages' rows; the last packer zeroes the tail
    const int64_t rows = m.groups_padded * kGroup;
    const int n_rows_q = r.src_pages ? r.src_first : n_q;
    const int64_t q_end = n_rows_q == n_q ? rows : reinterpret_cast<const int64_t*>(m.host.data() + m.off_ds)[n_rows_q];
    if (n_rows_q > 0)
      if (int e = launch_pack_rows(h, r.q, r.q_dtype, ss_dev, ds_dev, n_rows_q, q_end, 1, h->q_packed.p, c.dtype, r.i8_q_scale, s))
        return e;
    if (n_rows_q < n_q)
      if (int e = launch_pack_src_pages(h, r.src_pages, ss_dev + n_rows_q, ds_dev + n_rows_q, n_q - n_rows_q, q_end, rows,
                                        h->q_packed.p, s))
        return e;
  }
  const int ng = int(m.groups);
  if (!c.host) {
    UnitPlan scan;
    const bool full_scan = !cs.ids && ng > 0;
    if (full_scan)
      if (int e = plan_full_scan(h, r.allow, r.mask_index, n_q, s, &scan)) return e;
    if (int e = score_impl(h, h->q_packed.p, ng, m.goff(), n_q, ntok_dev, h->scores.p, ld, cs, s, corpus_view(h), cs.ids, true,
                           full_scan && h->scan_planned ? &scan : nullptr, !r.page_scale))
      return e;
  } else if (ng > 0 && n_items > 0) {
    struct Ctx {
      const void* q;
      int ng;
      const int32_t* goff;
      int n_q;
      const int32_t* ntok;
      int64_t ld;
      const CandSpec* cs;
      cudaStream_t s;
      bool zero_pad;
    } ctx{h->q_packed.p, ng, m.goff(), n_q, ntok_dev, ld, &cs, s, !r.page_scale};
    auto round = [](b200ms_t* hh, const CorpusView& v, const int64_t* unit_ids, void* scores, bool fill, void* p) {
      const Ctx& x = *static_cast<const Ctx*>(p);
      return score_impl(hh, x.q, x.ng, x.goff, x.n_q, x.ntok, scores, x.ld, *x.cs, x.s, v, unit_ids, fill, nullptr, x.zero_pad);
    };
    if (int e = score_host_tier(h, cs, n_q, gp, ld, h->scores.p, s, round, &ctx)) return e;
  }
  if (ng == 0 || n_items == 0)
    if (int e = zero_scores(h, h->scores.p, gp, ld, s, "search: memset")) return e;
  out->cs = cs;
  out->ld = ld;
  out->goff_dev = goff_dev;
  out->sdt = (c.dtype == B200MS_BF16 || c.dtype == B200MS_F8) ? B200MS_F32 : B200MS_I32;
  return B200MS_OK;
}

int search_core(b200ms_t* h, const SearchRequest& r, const SearchMeta& m, cudaStream_t s, const void* meta_dev) {
  ScanResult sr;
  if (int e = search_scan(h, r, m, s, meta_dev, &sr)) return e;
  const Corpus& c = h->corpus;
  const int n_q = r.n_q;
  const CandSpec& cs = sr.cs;
  const int64_t ld = sr.ld;
  const int32_t* goff_dev = sr.goff_dev;
  const int sdt = sr.sdt;
  if (r.docs)
    return cs.ids ? launch_topk_docs(h, h->scores.p, sdt, cs.n_cand, ld, goff_dev, n_q, nullptr, nullptr, cs.ids, cs.stride(),
                                     c.n_pages, *r.docs, r.k, r.score_scale, 0, s)
                  : launch_topk_docs(h, h->scores.p, sdt, c.n_pages, ld, goff_dev, n_q, r.allow, r.mask_index, nullptr, 0,
                                     c.n_pages, *r.docs, r.k, r.score_scale, r.id_base, s);
  if (!cs.ids) {
    return launch_topk(h, h->scores.p, sdt, c.n_pages, ld, goff_dev, n_q, r.allow, r.k, r.score_scale, r.id_base, nullptr,
                       r.top_scores, r.top_ids, r.top_counts, s, r.mask_index, (c.n_pages + 31) / 32);
  }
  // candidate mode: rank the slots (ties -> lower slot = better first-stage rank), report the page ids; unused slots masked
  const int n_slots = int(cs.n_slots(n_q));
  if (int e = reserve(h, h->cand_mask, size_t((n_slots + 31) / 32 + 1) * 4)) return e;
  if (int e = launch_cand_units(h, corpus_view(h), cs.ids, n_slots, nullptr, nullptr, static_cast<uint32_t*>(h->cand_mask.p), s))
    return e;
  if (r.allow && cs.per_query)
    if (int e = launch_mask_cand_slots(h, cs.ids, n_slots, cs.stride(), r.allow, r.mask_index,
                                       static_cast<uint32_t*>(h->cand_mask.p), s))
      return e;
  return launch_topk(h, h->scores.p, sdt, cs.n_cand, ld, goff_dev, n_q, static_cast<const uint32_t*>(h->cand_mask.p), r.k,
                     r.score_scale, 0, cs.ids, r.top_scores, r.top_ids, r.top_counts, s, nullptr, 0, cs.stride());
}

}  // namespace bms

B200MS_API int b200ms_rerank_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                    const int64_t* cand_ids_dev, int n_cand, int k, float i8_q_scale, float score_scale,
                                    float* top_scores_dev, int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (!src_dtype_ok(src_dtype) || !cand_ids_dev || n_cand < 1)
    return set_error(h, B200MS_EINVAL, "rerank_device: bad arguments (F32/BF16 queries, n_cand >= 1)");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, q_lens, n_q, k, i8_q_scale, score_scale, top_scores_dev, top_ids_dev, top_counts_dev};
  r.cand = CandSpec{cand_ids_dev, n_cand, 0};
  return search_ordered(h, r, static_cast<cudaStream_t>(stream));
}

B200MS_API int b200ms_rerank_batch_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                          const int64_t* cand_ids_dev, int n_cand, int k, float i8_q_scale, float score_scale,
                                          float* top_scores_dev, int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream) {
  if (!h) return B200MS_EINVAL;
  const CandSpec cand{cand_ids_dev, n_cand, 1};
  if (!src_dtype_ok(src_dtype) || !cand_ids_dev || n_cand < 1 || n_q < 1 || cand.n_slots(n_q) >= (int64_t(1) << 30))
    return set_error(h, B200MS_EINVAL, "rerank_batch_device: bad arguments (F32/BF16 queries, n_cand >= 1, n_q*n_cand < 2^30)");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, q_lens, n_q, k, i8_q_scale, score_scale, top_scores_dev, top_ids_dev, top_counts_dev};
  r.cand = cand;
  return search_ordered(h, r, static_cast<cudaStream_t>(stream));
}

B200MS_API int b200ms_search_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q, int k,
                                    const uint32_t* allow_mask_dev, float i8_q_scale, float score_scale, int64_t id_base,
                                    float* top_scores_dev, int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (!src_dtype_ok(src_dtype)) return set_error(h, B200MS_EINVAL, "search_device: src dtype must be F32 or BF16");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, q_lens, n_q, k, i8_q_scale, score_scale, top_scores_dev, top_ids_dev, top_counts_dev, id_base};
  r.allow = allow_mask_dev;
  return search_ordered(h, r, static_cast<cudaStream_t>(stream));
}

B200MS_API int b200ms_search_device_masked(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                           int k, const uint32_t* allow_masks_dev, int n_masks,
                                           const int32_t* mask_index_dev, float i8_q_scale, float score_scale,
                                           int64_t id_base, float* top_scores_dev, int64_t* top_ids_dev,
                                           int32_t* top_counts_dev, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (!src_dtype_ok(src_dtype)) return set_error(h, B200MS_EINVAL, "search_device_masked: src dtype must be F32 or BF16");
  if (n_masks < 0 || (n_masks > 0 && (!allow_masks_dev || !mask_index_dev)))
    return set_error(h, B200MS_EINVAL, "search_device_masked: n_masks > 0 needs the mask matrix and one index per query");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, q_lens, n_q, k, i8_q_scale, score_scale, top_scores_dev, top_ids_dev, top_counts_dev, id_base};
  if (n_masks > 0) {
    r.allow = allow_masks_dev;
    r.mask_index = mask_index_dev;
  }
  return search_ordered(h, r, static_cast<cudaStream_t>(stream));
}

// ---- grouping results by document
static bool docs_dims_ok(int k, int per_doc, int64_t n_docs, int64_t n_pages) {
  return k >= 1 && k <= B200MS_MAX_K && per_doc >= 1 && per_doc <= B200MS_MAX_PER_DOC && n_docs >= 0 &&
         (n_pages == 0 || n_docs >= 1) && n_docs <= n_pages;
}

B200MS_API int b200ms_topk_docs(b200ms_t* h, const void* group_scores, int score_dtype, int64_t n_pages, int64_t ld,
                                const int32_t* group_offsets, int n_q, const uint32_t* allow_mask, const int32_t* page_doc,
                                int64_t n_docs, int k, int per_doc, float scale, int64_t id_base, float* doc_page_scores,
                                int64_t* doc_page_ids, int32_t* doc_page_counts, int32_t* doc_counts, void* stream) {
  if (!h) return B200MS_EINVAL;
  if ((score_dtype != B200MS_F32 && score_dtype != B200MS_I32) || n_pages < 0 || ld < n_pages || n_q < 0 ||
      !docs_dims_ok(k, per_doc, n_docs, n_pages) || !page_doc || !doc_page_scores || !doc_page_ids || !doc_page_counts ||
      !doc_counts || (n_q > 0 && !group_offsets) || (n_q > 0 && n_pages > 0 && !group_scores))
    return set_error(h, B200MS_EINVAL, "topk_docs: bad arguments (1 <= k <= 4096, 1 <= per_doc <= 64, 1 <= n_docs <= n_pages)");
  if (n_q == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  if (int e = upload(h, h->meta, group_offsets, size_t(n_q + 1) * 4, s)) return e;
  const DocSpec d{page_doc, n_docs, per_doc, doc_page_scores, doc_page_ids, doc_page_counts, doc_counts};
  return launch_topk_docs(h, group_scores, score_dtype, n_pages, ld, static_cast<const int32_t*>(h->meta.p), n_q, allow_mask,
                          nullptr, nullptr, 0, n_pages, d, k, scale, id_base, s);
}

B200MS_API int b200ms_search_docs_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q, int k,
                                         int per_doc, const int32_t* page_doc, int64_t n_docs, const uint32_t* allow_masks_dev,
                                         int n_masks, const int32_t* mask_index_dev, float i8_q_scale, float score_scale,
                                         int64_t id_base, float* doc_page_scores, int64_t* doc_page_ids,
                                         int32_t* doc_page_counts, int32_t* doc_counts, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (!src_dtype_ok(src_dtype)) return set_error(h, B200MS_EINVAL, "search_docs_device: src dtype must be F32 or BF16");
  if (n_masks < 0 || (n_masks > 0 && (!allow_masks_dev || !mask_index_dev)))
    return set_error(h, B200MS_EINVAL, "search_docs_device: n_masks > 0 needs the mask matrix and one index per query");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, q_lens, n_q, k, i8_q_scale, score_scale, doc_page_scores, doc_page_ids, doc_counts, id_base};
  if (n_masks > 0) {
    r.allow = allow_masks_dev;
    r.mask_index = mask_index_dev;
  }
  const DocSpec d{page_doc, n_docs, per_doc, doc_page_scores, doc_page_ids, doc_page_counts, doc_counts};
  r.docs = &d;
  return search_ordered(h, r, static_cast<cudaStream_t>(stream));
}

B200MS_API int b200ms_rerank_docs_batch_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                               const int64_t* cand_ids_dev, int n_cand, int k, int per_doc,
                                               const int32_t* page_doc, int64_t n_docs, float i8_q_scale, float score_scale,
                                               float* doc_page_scores, int64_t* doc_page_ids, int32_t* doc_page_counts,
                                               int32_t* doc_counts, void* stream) {
  if (!h) return B200MS_EINVAL;
  const CandSpec cand{cand_ids_dev, n_cand, 1};
  if (!src_dtype_ok(src_dtype) || !cand_ids_dev || n_cand < 1 || n_q < 1 || cand.n_slots(n_q) >= (int64_t(1) << 30))
    return set_error(h, B200MS_EINVAL,
                     "rerank_docs_batch_device: bad arguments (F32/BF16 queries, n_cand >= 1, n_q*n_cand < 2^30)");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, q_lens, n_q, k, i8_q_scale, score_scale, doc_page_scores, doc_page_ids, doc_counts};
  r.cand = cand;
  const DocSpec d{page_doc, n_docs, per_doc, doc_page_scores, doc_page_ids, doc_page_counts, doc_counts};
  r.docs = &d;
  return search_ordered(h, r, static_cast<cudaStream_t>(stream));
}

// ---- documents ranked by document-level MaxSim
static int doc_maxsim_ordered(b200ms_t* h, const bms::DocMaxSimCall& x, int src_dtype, cudaStream_t s) {
  if (!h) return B200MS_EINVAL;
  if (!src_dtype_ok(src_dtype)) return set_error(h, B200MS_EINVAL, "doc_maxsim: src dtype must be F32 or BF16");
  DeviceGuard g(h->device);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  return doc_maxsim(h, x, s);
}

B200MS_API int b200ms_search_doc_maxsim_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                               int k, int per_doc, const int32_t* page_doc, int64_t n_docs,
                                               const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                               float i8_q_scale, float score_scale, int64_t id_base, float* doc_scores,
                                               int64_t* doc_ids, int64_t* page_ids, float* page_shares,
                                               int32_t* page_counts, int32_t* doc_counts, void* cuda_stream) {
  bms::DocMaxSimCall x{q_dev, src_dtype, q_lens, n_q, k, per_doc, page_doc, n_docs, allow_masks_dev, n_masks, mask_index_dev,
                       nullptr, 0, i8_q_scale, score_scale, id_base, doc_scores, doc_ids, page_shares, page_ids, page_counts,
                       doc_counts};
  return doc_maxsim_ordered(h, x, src_dtype, static_cast<cudaStream_t>(cuda_stream));
}

B200MS_API int b200ms_rerank_doc_maxsim_batch_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens,
                                                     int n_q, const int64_t* cand_ids_dev, int n_cand, int k, int per_doc,
                                                     const int32_t* page_doc, int64_t n_docs, const uint32_t* allow_masks_dev,
                                                     int n_masks, const int32_t* mask_index_dev, float i8_q_scale,
                                                     float score_scale, int64_t id_base, float* doc_scores, int64_t* doc_ids,
                                                     int64_t* page_ids, float* page_shares, int32_t* page_counts,
                                                     int32_t* doc_counts, void* cuda_stream) {
  if (h && !cand_ids_dev)
    return set_error(h, B200MS_EINVAL, "rerank_doc_maxsim_batch_device: bad arguments (candidate lists [n_q, n_cand >= 1])");
  bms::DocMaxSimCall x{q_dev, src_dtype, q_lens, n_q, k, per_doc, page_doc, n_docs, allow_masks_dev, n_masks, mask_index_dev,
                       cand_ids_dev, n_cand, i8_q_scale, score_scale, id_base, doc_scores, doc_ids, page_shares, page_ids,
                       page_counts, doc_counts};
  return doc_maxsim_ordered(h, x, src_dtype, static_cast<cudaStream_t>(cuda_stream));
}

// ---- searching with stored pages as the queries
// The source pages of a call: every id names a page of the attached corpus; their true lengths into *lens
static int check_src_pages(b200ms_t* h, const int64_t* src, int n_src, const char* what, std::vector<int32_t>* lens) {
  const Corpus& c = h->corpus;
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, std::string(what) + ": no corpus attached");
  if (!src || n_src < 1) return set_error(h, B200MS_EINVAL, std::string(what) + ": bad arguments (n_src >= 1 source pages)");
  lens->resize(size_t(n_src));
  for (int i = 0; i < n_src; ++i) {
    if (src[i] < 0 || src[i] >= c.n_pages)
      return set_error(h, B200MS_EINVAL, std::string(what) + ": source page " + std::to_string(src[i]) + " is not a page of the corpus (" +
                                             std::to_string(c.n_pages) + " pages)");
    (*lens)[size_t(i)] = h->page_len_host[size_t(src[i])];
  }
  return B200MS_OK;
}

static int check_masks(b200ms_t* h, const uint32_t* masks, int n_masks, const int32_t* index, const char* what) {
  if (n_masks < 0 || (n_masks > 0 && (!masks || !index)))
    return set_error(h, B200MS_EINVAL, std::string(what) + ": n_masks > 0 needs the mask matrix and one index per source");
  return B200MS_OK;
}

// pack the sources' rows -> score -> top-k (search_core) -> divide every source's scores by its length
static int search_pages_ordered(b200ms_t* h, const int64_t* src_host, SearchRequest& r, cudaStream_t s) {
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  if (int e = upload(h, h->src_pages, src_host, size_t(r.n_q) * 8, s)) return e;
  r.src_pages = static_cast<const int64_t*>(h->src_pages.p);
  r.page_scale = true;
  if (int e = search_core(h, r, build_search_meta(r.q_lens, r.n_q), s)) return e;
  return launch_normalise_pages(h, r.src_pages, r.n_q, r.k, r.top_scores, r.top_ids, r.top_counts, s);
}

B200MS_API int b200ms_search_pages_device(b200ms_t* h, const int64_t* src_pages_host, int n_src, int k,
                                          const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                          float score_scale, int64_t id_base, float* top_scores_dev, int64_t* top_ids_dev,
                                          int32_t* top_counts_dev, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  if (h->corpus.host) return set_error(h, B200MS_ESTATE, kHostFullScan);
  std::vector<int32_t> lens;
  if (int e = check_src_pages(h, src_pages_host, n_src, "search_pages_device", &lens)) return e;
  if (int e = check_masks(h, allow_masks_dev, n_masks, mask_index_dev, "search_pages_device")) return e;
  if (k < 1 || k > B200MS_MAX_K || !top_scores_dev || !top_ids_dev || !top_counts_dev)
    return set_error(h, B200MS_EINVAL, "search_pages_device: bad arguments (1 <= k <= 4096, outputs)");
  DeviceGuard g(h->device);
  SearchRequest r{nullptr, h->corpus.dtype, lens.data(), n_src, k, 1.f, score_scale, top_scores_dev, top_ids_dev, top_counts_dev,
                  id_base};
  if (n_masks > 0) {
    r.allow = allow_masks_dev;
    r.mask_index = mask_index_dev;
  }
  return search_pages_ordered(h, src_pages_host, r, static_cast<cudaStream_t>(cuda_stream));
}

B200MS_API int b200ms_rerank_pages_batch_device(b200ms_t* h, const int64_t* src_pages_host, int n_src,
                                                const int64_t* cand_ids_dev, int n_cand, int k,
                                                const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                                float score_scale, float* top_scores_dev, int64_t* top_ids_dev,
                                                int32_t* top_counts_dev, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  std::vector<int32_t> lens;
  if (int e = check_src_pages(h, src_pages_host, n_src, "rerank_pages_batch_device", &lens)) return e;
  if (int e = check_masks(h, allow_masks_dev, n_masks, mask_index_dev, "rerank_pages_batch_device")) return e;
  const CandSpec cand{cand_ids_dev, n_cand, 1};
  if (!cand_ids_dev || n_cand < 1 || cand.n_slots(n_src) >= (int64_t(1) << 30) || k < 1 || k > B200MS_MAX_K || !top_scores_dev ||
      !top_ids_dev || !top_counts_dev)
    return set_error(h, B200MS_EINVAL, "rerank_pages_batch_device: bad arguments (n_cand >= 1, n_src*n_cand < 2^30, 1 <= k <= 4096)");
  DeviceGuard g(h->device);
  SearchRequest r{nullptr, h->corpus.dtype, lens.data(), n_src, k, 1.f, score_scale, top_scores_dev, top_ids_dev, top_counts_dev};
  r.cand = cand;
  if (n_masks > 0) {
    r.allow = allow_masks_dev;
    r.mask_index = mask_index_dev;
  }
  return search_pages_ordered(h, src_pages_host, r, static_cast<cudaStream_t>(cuda_stream));
}

B200MS_API int b200ms_page_rows_device(b200ms_t* h, const int64_t* src_pages_host, int n_src, float scale, float* out,
                                       void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  std::vector<int32_t> lens;
  if (int e = check_src_pages(h, src_pages_host, n_src, "page_rows_device", &lens)) return e;
  // [src ids | true-row offsets], one upload
  std::vector<int64_t> meta(size_t(2 * n_src + 1), 0);
  for (int i = 0; i < n_src; ++i) {
    meta[size_t(i)] = src_pages_host[i];
    meta[size_t(n_src + i + 1)] = meta[size_t(n_src + i)] + lens[size_t(i)];
  }
  const int64_t n_rows = meta.back();
  if (n_rows > 0 && !out) return set_error(h, B200MS_EINVAL, "page_rows_device: out is NULL");
  if (n_rows == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  if (int e = upload(h, h->src_pages, meta.data(), meta.size() * 8, s)) return e;
  const int64_t* d = static_cast<const int64_t*>(h->src_pages.p);
  return launch_page_rows(h, d, d + n_src, n_src, n_rows, scale, out, s);
}

// ---- relevance feedback: weighted examples, one fused score per request
// The examples of a call: n_qe query embeddings (rows of q_dev, lengths q_lens) then n_src stored pages; example i belongs to
// request ex_req[i] and carries weight ex_w[i].  Their true lengths (tokens, rows) into *lens, in example order.
static int check_examples(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_qe, const int64_t* src,
                          int n_src, const int32_t* ex_req, const float* ex_w, int n_req, const char* what,
                          std::vector<int32_t>* lens) {
  const Corpus& c = h->corpus;
  const std::string w(what);
  if (c.dtype < 0) return set_error(h, B200MS_ESTATE, w + ": no corpus attached");
  if (n_qe < 0 || n_src < 0 || n_qe + n_src < 1 || n_req < 1 || !ex_req || !ex_w ||
      (n_qe > 0 && (!q_dev || !q_lens || !src_dtype_ok(src_dtype))) || (n_src > 0 && !src))
    return set_error(h, B200MS_EINVAL, w + ": bad arguments (one or more examples, n_req >= 1, F32/BF16 query rows)");
  lens->clear();
  for (int i = 0; i < n_qe; ++i) {
    if (q_lens[i] < 0) return set_error(h, B200MS_EINVAL, w + ": a query example has a negative length");
    lens->push_back(q_lens[i]);
  }
  for (int i = 0; i < n_src; ++i) {
    if (src[i] < 0 || src[i] >= c.n_pages)
      return set_error(h, B200MS_EINVAL, w + ": example page " + std::to_string(src[i]) + " is not a page of the corpus (" +
                                             std::to_string(c.n_pages) + " pages)");
    lens->push_back(h->page_len_host[size_t(src[i])]);
  }
  std::vector<char> positive(size_t(n_req), 0);
  for (int i = 0; i < n_qe + n_src; ++i) {
    if (ex_req[i] < 0 || ex_req[i] >= n_req)
      return set_error(h, B200MS_EINVAL, w + ": example " + std::to_string(i) + " names request " + std::to_string(ex_req[i]) +
                                             " outside [0, " + std::to_string(n_req) + ")");
    if (!std::isfinite(ex_w[i]) || ex_w[i] == 0.f)
      return set_error(h, B200MS_EINVAL, w + ": example " + std::to_string(i) + " has a zero or non-finite weight");
    if (ex_w[i] > 0.f) positive[size_t(ex_req[i])] = 1;
  }
  for (int q = 0; q < n_req; ++q)
    if (!positive[size_t(q)])
      return set_error(h, B200MS_EINVAL, w + ": request " + std::to_string(q) + " has no example of positive weight");
  return B200MS_OK;
}

struct ExampleCall {
  const int64_t* src_host;
  int n_src, n_qe;
  const int32_t* ex_req;
  const float* ex_w;
  int n_req;
  const int64_t* cand;  // NULL: full scan; else the requests' lists [n_req, n_cand]
  int n_cand;
  const uint32_t* masks;  // n_masks > 0: one row per request through mask_index
  int n_masks;
  const int32_t* mask_index;
};

// Every example of every request scored in ONE search_scan (each example a query of it: query embeddings packed from q,
// pages from their packed rows; in candidate mode every example scores its request's list), then one fused score row per
// request (launch_fuse_examples) and one selection over those rows (launch_topk: one group per request, F32, scale 1).
static int search_examples_ordered(b200ms_t* h, SearchRequest& r, const ExampleCall& x, cudaStream_t s) {
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  const Corpus& c = h->corpus;
  const int n_ex = r.n_q, n_req = x.n_req;
  const SearchMeta m = build_search_meta(r.q_lens, n_ex);
  const int32_t* goff = m.goff();
  const int64_t stride = x.cand ? CandSpec{x.cand, x.n_cand, 1}.stride() : 0;
  // one upload: [source page ids int64 | the examples by request | req_off int32 [n_req+1] | 0..n_req int32 | ex_req int32]
  const size_t off_items = size_t(x.n_src) * 8, off_req = off_items + size_t(n_ex) * sizeof(ExampleItem);
  const size_t off_iota = off_req + size_t(n_req + 1) * 4, off_exreq = off_iota + size_t(n_req + 1) * 4;
  std::vector<uint8_t> blk(off_exreq + size_t(n_ex) * 4);
  if (x.n_src > 0) memcpy(blk.data(), x.src_host, off_items);
  ExampleItem* items = reinterpret_cast<ExampleItem*>(blk.data() + off_items);
  int32_t* req_off = reinterpret_cast<int32_t*>(blk.data() + off_req);
  int32_t* iota = reinterpret_cast<int32_t*>(blk.data() + off_iota);
  memcpy(blk.data() + off_exreq, x.ex_req, size_t(n_ex) * 4);
  for (int q = 0; q <= n_req; ++q) req_off[q] = 0, iota[q] = q;
  for (int i = 0; i < n_ex; ++i) req_off[x.ex_req[i] + 1]++;
  for (int q = 0; q < n_req; ++q) req_off[q + 1] += req_off[q];
  std::vector<int32_t> fill(req_off, req_off + n_req);
  for (int i = 0; i < n_ex; ++i)  // stable: a request's examples stay in example order
    items[fill[size_t(x.ex_req[i])]++] = ExampleItem{goff[i], goff[i + 1], float(r.q_lens[i]), x.ex_w[i], int64_t(i) * stride};
  if (int e = upload(h, h->ex_meta, blk.data(), blk.size(), s)) return e;
  const uint8_t* md = static_cast<const uint8_t*>(h->ex_meta.p);
  const ExampleItem* items_dev = reinterpret_cast<const ExampleItem*>(md + off_items);
  const int32_t* req_off_dev = reinterpret_cast<const int32_t*>(md + off_req);
  const int32_t* iota_dev = reinterpret_cast<const int32_t*>(md + off_iota);
  const int32_t* ex_req_dev = reinterpret_cast<const int32_t*>(md + off_exreq);
  if (x.n_src > 0) {
    r.src_pages = reinterpret_cast<const int64_t*>(md);
    r.src_first = x.n_qe;
  }
  r.page_scale = true;
  const uint32_t* allow = x.n_masks > 0 ? x.masks : nullptr;
  const int32_t* mask_index = x.n_masks > 0 ? x.mask_index : nullptr;
  int64_t* req_lists = nullptr;
  if (x.cand) {  // [n_req + n_ex, stride]: the requests' lists padded to 32-slot strides, then every example's request's list
    if (int e = reserve(h, h->ex_lists, size_t(n_req + n_ex) * size_t(stride) * 8)) return e;
    req_lists = static_cast<int64_t*>(h->ex_lists.p);
    int64_t* ex_lists = req_lists + int64_t(n_req) * stride;
    if (int e = launch_pad_cands(h, x.cand, x.n_cand, n_req, stride, req_lists, s)) return e;
    if (int e = launch_gather_rows<int64_t>(h, req_lists, stride, ex_req_dev, n_ex, ex_lists, s)) return e;
    r.cand = CandSpec{ex_lists, int(stride), 1};
  } else if (allow) {  // the filtered scan reads the pages any example's request may return
    if (int e = reserve(h, h->ex_lists, size_t(n_ex) * 4)) return e;
    int32_t* ex_mask_index = static_cast<int32_t*>(h->ex_lists.p);
    if (int e = launch_gather_rows<int32_t>(h, mask_index, 1, ex_req_dev, n_ex, ex_mask_index, s)) return e;
    r.allow = allow;
    r.mask_index = ex_mask_index;
  }
  ScanResult sr;
  if (int e = search_scan(h, r, m, s, nullptr, &sr)) return e;
  if (!x.cand) {
    const int64_t words = (c.n_pages + 31) / 32, fld = words * 32 > 32 ? words * 32 : 32;
    if (int e = reserve(h, h->ex_fused, size_t(n_req) * size_t(fld) * 4)) return e;
    float* fused = static_cast<float*>(h->ex_fused.p);
    if (int e = launch_fuse_examples(h, h->scores.p, sr.sdt, sr.ld, items_dev, req_off_dev, n_req, c.n_pages, allow, mask_index,
                                     words, r.score_scale, fused, fld, s))
      return e;
    return launch_topk(h, fused, B200MS_F32, c.n_pages, fld, iota_dev, n_req, allow, r.k, 1.f, r.id_base, nullptr, r.top_scores,
                       r.top_ids, r.top_counts, s, mask_index, words);
  }
  // candidate mode: request r's slots are r * stride + j; its valid-slot bits (unused slots and pages its mask row forbids
  // cleared) filter both the fusion and the selection
  const int64_t n_slots = int64_t(n_req) * stride;
  uint32_t* slot_mask = nullptr;
  if (int e = reserve(h, h->cand_mask, size_t((n_slots + 31) / 32 + 1) * 4)) return e;
  slot_mask = static_cast<uint32_t*>(h->cand_mask.p);
  if (int e = launch_cand_units(h, corpus_view(h), req_lists, int(n_slots), nullptr, nullptr, slot_mask, s)) return e;
  if (allow)
    if (int e = launch_mask_cand_slots(h, req_lists, n_slots, stride, allow, mask_index, slot_mask, s)) return e;
  if (int e = reserve(h, h->ex_fused, size_t(n_slots) * 4)) return e;
  float* fused = static_cast<float*>(h->ex_fused.p);
  if (int e = launch_fuse_examples(h, h->scores.p, sr.sdt, sr.ld, items_dev, req_off_dev, n_req, x.n_cand, slot_mask, nullptr,
                                   stride / 32, r.score_scale, fused, stride, s))
    return e;
  // all requests' fused slots form ONE row (request r's at r * stride, where the selection looks for them); with ld 0 that
  // row is every request's one group
  return launch_topk(h, fused, B200MS_F32, x.n_cand, 0, iota_dev, n_req, slot_mask, r.k, 1.f, 0, req_lists, r.top_scores,
                     r.top_ids, r.top_counts, s, nullptr, 0, stride);
}

B200MS_API int b200ms_search_examples_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_qe,
                                             const int64_t* src_pages_host, int n_src, const int32_t* ex_req_host,
                                             const float* ex_weight_host, int n_req, int k, const uint32_t* allow_masks_dev,
                                             int n_masks, const int32_t* mask_index_dev, float i8_q_scale, float score_scale,
                                             int64_t id_base, float* top_scores_dev, int64_t* top_ids_dev,
                                             int32_t* top_counts_dev, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  if (h->corpus.host) return set_error(h, B200MS_ESTATE, kHostFullScan);
  std::vector<int32_t> lens;
  if (int e = check_examples(h, q_dev, src_dtype, q_lens, n_qe, src_pages_host, n_src, ex_req_host, ex_weight_host, n_req,
                             "search_examples_device", &lens))
    return e;
  if (int e = check_masks(h, allow_masks_dev, n_masks, mask_index_dev, "search_examples_device")) return e;
  if (k < 1 || k > B200MS_MAX_K || !top_scores_dev || !top_ids_dev || !top_counts_dev)
    return set_error(h, B200MS_EINVAL, "search_examples_device: bad arguments (1 <= k <= 4096, outputs)");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, lens.data(), n_qe + n_src, k, i8_q_scale, score_scale, top_scores_dev, top_ids_dev,
                  top_counts_dev, id_base};
  const ExampleCall x{src_pages_host, n_src, n_qe, ex_req_host, ex_weight_host, n_req, nullptr, 0, allow_masks_dev, n_masks,
                      mask_index_dev};
  return search_examples_ordered(h, r, x, static_cast<cudaStream_t>(cuda_stream));
}

B200MS_API int b200ms_rerank_examples_batch_device(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens,
                                                   int n_qe, const int64_t* src_pages_host, int n_src,
                                                   const int32_t* ex_req_host, const float* ex_weight_host, int n_req,
                                                   const int64_t* cand_ids_dev, int n_cand, int k,
                                                   const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                                   float i8_q_scale, float score_scale, float* top_scores_dev,
                                                   int64_t* top_ids_dev, int32_t* top_counts_dev, void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  std::vector<int32_t> lens;
  if (int e = check_examples(h, q_dev, src_dtype, q_lens, n_qe, src_pages_host, n_src, ex_req_host, ex_weight_host, n_req,
                             "rerank_examples_batch_device", &lens))
    return e;
  if (int e = check_masks(h, allow_masks_dev, n_masks, mask_index_dev, "rerank_examples_batch_device")) return e;
  const CandSpec cand{cand_ids_dev, n_cand, 1};
  if (!cand_ids_dev || n_cand < 1 || cand.n_slots(n_req + n_qe + n_src) >= (int64_t(1) << 30) || k < 1 || k > B200MS_MAX_K ||
      !top_scores_dev || !top_ids_dev || !top_counts_dev)
    return set_error(h, B200MS_EINVAL,
                     "rerank_examples_batch_device: bad arguments (n_cand >= 1, (n_req + examples)*n_cand < 2^30, 1 <= k <= 4096)");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, lens.data(), n_qe + n_src, k, i8_q_scale, score_scale, top_scores_dev, top_ids_dev,
                  top_counts_dev};
  const ExampleCall x{src_pages_host, n_src, n_qe, ex_req_host, ex_weight_host, n_req, cand_ids_dev, n_cand, allow_masks_dev,
                      n_masks, mask_index_dev};
  return search_examples_ordered(h, r, x, static_cast<cudaStream_t>(cuda_stream));
}

B200MS_API int b200ms_union_candidates_device(b200ms_t* h, const int64_t* cand_ids_dev, int n_lists, int n_cand,
                                              const int32_t* list_off_host, int n_req, int64_t* out_dev, int width,
                                              void* cuda_stream) {
  if (!h) return B200MS_EINVAL;
  if (n_req < 1 || n_lists < 0 || n_cand < 1 || width < 1 || !list_off_host || !out_dev || (n_lists > 0 && !cand_ids_dev) ||
      int64_t(n_lists) * n_cand >= (int64_t(1) << 30))
    return set_error(h, B200MS_EINVAL, "union_candidates_device: bad arguments (n_req >= 1, n_cand >= 1, width >= 1, n_lists*n_cand < 2^30)");
  int64_t most = 0;
  bool ok = list_off_host[0] == 0 && list_off_host[n_req] == n_lists;
  for (int q = 0; q < n_req && ok; ++q) {
    ok = list_off_host[q + 1] >= list_off_host[q];
    most = std::max(most, int64_t(list_off_host[q + 1] - list_off_host[q]) * n_cand);
  }
  if (!ok)
    return set_error(h, B200MS_EINVAL, "union_candidates_device: list_off must rise from 0 to n_lists");
  DeviceGuard g(h->device);
  cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  if (int e = upload(h, h->ex_meta, list_off_host, size_t(n_req + 1) * 4, s)) return e;
  return launch_union_candidates(h, cand_ids_dev, n_cand, static_cast<const int32_t*>(h->ex_meta.p), n_req, most, out_dev,
                                 width, s);
}

// Small unmasked zero-copy calls repeat with the same shapes (interactive queries): the second call of a shape is captured
// into a CUDA graph -- pack -> score -> top-k become ONE launch, the third call onwards replays it.  Everything the kernels
// read or write sits at fixed addresses (mapped staging block, handle scratch); h->generation changes when any moves.
// enqueue() puts the search on stream s; it runs plainly on the first use of a shape and whenever capture fails.
template <class Enqueue>
static int run_host_graph(b200ms_t* h, uint64_t key, cudaStream_t s, Enqueue&& enqueue) {
  b200ms::HostGraph* hg = nullptr;  // NOLINT
  for (auto& g : h->host_graphs)
    if (g.key == key) hg = &g;
  if (!hg) {
    if (h->host_graphs.size() >= 16) {  // evict the least recently used shape
      size_t lru = 0;
      for (size_t i = 1; i < h->host_graphs.size(); ++i)
        if (h->host_graphs[i].last_use < h->host_graphs[lru].last_use) lru = i;
      if (h->host_graphs[lru].exec) cudaGraphExecDestroy(h->host_graphs[lru].exec);
      h->host_graphs.erase(h->host_graphs.begin() + long(lru));
    }
    h->host_graphs.emplace_back();
    hg = &h->host_graphs.back();
    hg->key = key;
  }
  hg->last_use = ++h->graph_clock;
  if (hg->exec && hg->generation != h->generation) {  // a buffer moved / corpus or option changed: start over
    cudaGraphExecDestroy(hg->exec);
    hg->exec = nullptr;
    hg->seen = 0;
  }
  if (hg->exec) {
    if (int e = check_cuda(h, cudaGraphLaunch(hg->exec, s), "search_host: graph launch")) return e;
    h->launches += hg->launches;
    return B200MS_OK;
  }
  if (hg->seen < 1) {
    hg->seen++;
    return enqueue();
  }
  const uint64_t gen0 = h->generation;
  const int64_t l0 = h->launches;
  if (int e = check_cuda(h, cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal), "search_host: begin capture")) return e;
  h->capturing = true;
  const int e = enqueue();
  h->capturing = false;
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(s, &graph);
  bool ok = !e && ce == cudaSuccess && graph && gen0 == h->generation;
  if (ok) ok = cudaGraphInstantiate(&hg->exec, graph, 0) == cudaSuccess;
  if (graph) cudaGraphDestroy(graph);
  if (!ok) {
    cudaGetLastError();
    hg->exec = nullptr;
    hg->seen = -1000000;  // this shape does not capture: plain launches from now on
    return enqueue();
  }
  hg->generation = h->generation;
  hg->launches = int(h->launches - l0);
  return check_cuda(h, cudaGraphLaunch(hg->exec, s), "search_host: graph launch");
}

// the shape of a host search: everything a captured graph bakes in besides the staging and scratch addresses
static uint64_t host_graph_key(const SearchRequest& r) {
  uint64_t key = 1469598103934665603ull;
  auto mix = [&](uint64_t v) { key = (key ^ v) * 1099511628211ull; };
  mix(uint64_t(r.n_q));
  mix(uint64_t(r.k));
  for (int i = 0; i < r.n_q; ++i) mix(uint64_t(uint32_t(r.q_lens[i])));
  mix(uint64_t(r.id_base));
  uint32_t fb;
  memcpy(&fb, &r.score_scale, 4);
  mix(fb);
  memcpy(&fb, &r.i8_q_scale, 4);
  mix(fb);
  return key;
}

// Host entry point.  Two transports, same kernels:
//   zero-copy (small calls, the interactive case: <= 256 query rows and <= 64 KB of results): the query rows and the
//     per-call metadata are written into ONE handle-owned mapped pinned block that the pack / top-k kernels read in
//     place, and the top-k kernel writes its results straight into the same block -- no copy-engine operation and no
//     metadata upload on the critical path (round 1 spent ~12 driver calls, 4 of them pageable uploads, around a 15 us scan).
//   copy engine (batches): one H2D of the rows, one upload of the metadata block, one fused D2H of the result block.
static int search_host_impl(b200ms_t* h, const float* q_host, const int32_t* q_lens, int n_q, int k,
                            const uint32_t* masks_host, int n_masks, const int32_t* mask_index_host, float i8_q_scale,
                            float score_scale, int64_t id_base, float* top_scores_host, int64_t* top_ids_host,
                            int32_t* top_counts_host) {
  if (h->corpus.host) return set_error(h, B200MS_ESTATE, kHostFullScan);
  if (n_q < 1 || !q_lens || !q_host || k < 1 || k > B200MS_MAX_K || !top_scores_host || !top_ids_host || !top_counts_host)
    return set_error(h, B200MS_EINVAL, "search_host: bad arguments (n_q >= 1, 1 <= k <= 4096)");
  DeviceGuard g(h->device);
  cudaStream_t s = h->stream;
  StreamOrder order(h, s);  // before the first upload, and outside the graph capture of run_host_graph
  if (int e = order.error()) return e;
  const SearchMeta m = build_search_meta(q_lens, n_q);
  const ResultBlock rb(n_q, k);
  const size_t q_bytes = size_t(m.rows) * kDim * 4;
  SearchRequest r{nullptr, B200MS_F32, q_lens, n_q, k, i8_q_scale, score_scale};
  r.id_base = id_base;
  if (masks_host && n_masks > 0 && h->corpus.n_pages > 0) {
    if (mask_index_host)
      for (int i = 0; i < n_q; ++i)
        if (mask_index_host[i] < -1 || mask_index_host[i] >= n_masks)
          return set_error(h, B200MS_EINVAL, "search_host_masked: mask_index out of range");
    if (int e = upload(h, h->mask, masks_host, size_t(n_masks) * size_t((h->corpus.n_pages + 31) / 32) * 4, s)) return e;
    r.allow = static_cast<const uint32_t*>(h->mask.p);
    if (mask_index_host) {
      if (int e = upload(h, h->mask_index, mask_index_host, size_t(n_q) * 4, s)) return e;
      r.mask_index = static_cast<const int32_t*>(h->mask_index.p);
    }
  }
  const bool zc = h->zero_copy && m.rows <= 256 && rb.bytes() <= (64u << 10);
  const size_t q_off = (m.host.size() + 255) & ~size_t(255), out_off = (q_off + q_bytes + 255) & ~size_t(255);
  if (int e = reserve_pinned(h, h->stage, out_off + rb.bytes())) return e;
  uint8_t* st = static_cast<uint8_t*>(h->stage.p);
  void* out = st + out_off;  // where the kernels write the result block
  const void* meta_dev = nullptr;
  if (zc) {  // [metadata | query rows | results], all read and written in place
    memcpy(st, m.host.data(), m.host.size());
    if (q_bytes) memcpy(st + q_off, q_host, q_bytes);
    r.q = st + q_off;
    meta_dev = st;
  } else {
    if (int e = reserve(h, h->q_raw, q_bytes ? q_bytes : 512)) return e;
    if (int e = reserve(h, h->out_all, rb.bytes())) return e;
    if (q_bytes)
      if (int e = check_cuda(h, cudaMemcpyAsync(h->q_raw.p, q_host, q_bytes, cudaMemcpyHostToDevice, s), "search_host: H2D queries")) return e;
    r.q = h->q_raw.p;
    out = h->out_all.p;
  }
  r.top_scores = rb.scores(out);
  r.top_ids = rb.ids(out);
  r.top_counts = rb.counts(out);
  auto enqueue = [&] { return search_core(h, r, m, s, meta_dev); };
  if (int e = zc && h->host_graph && !r.allow ? run_host_graph(h, host_graph_key(r), s, enqueue) : enqueue()) return e;
  if (!zc)
    if (int e = check_cuda(h, cudaMemcpyAsync(st + out_off, out, rb.bytes(), cudaMemcpyDeviceToHost, s), "search_host: D2H results")) return e;
  if (int e = check_cuda(h, cudaStreamSynchronize(s), "search_host: stream sync")) return e;
  order.finished();
  rb.unpack(st + out_off, top_scores_host, top_ids_host, top_counts_host);
  return B200MS_OK;
}

B200MS_API int b200ms_search_host(b200ms_t* h, const float* q_host, const int32_t* q_lens, int n_q, int k,
                                  const uint32_t* allow_mask_host, float i8_q_scale, float score_scale, int64_t id_base,
                                  float* top_scores_host, int64_t* top_ids_host, int32_t* top_counts_host) {
  if (!h) return B200MS_EINVAL;
  return search_host_impl(h, q_host, q_lens, n_q, k, allow_mask_host, allow_mask_host ? 1 : 0, nullptr, i8_q_scale,
                          score_scale, id_base, top_scores_host, top_ids_host, top_counts_host);
}

B200MS_API int b200ms_search_host_masked(b200ms_t* h, const float* q_host, const int32_t* q_lens, int n_q, int k,
                                         const uint32_t* allow_masks_host, int n_masks, const int32_t* mask_index_host,
                                         float i8_q_scale, float score_scale, int64_t id_base, float* top_scores_host,
                                         int64_t* top_ids_host, int32_t* top_counts_host) {
  if (!h) return B200MS_EINVAL;
  if (n_masks < 0 || (n_masks > 0 && (!allow_masks_host || !mask_index_host)))
    return set_error(h, B200MS_EINVAL, "search_host_masked: n_masks > 0 needs the mask matrix and one index per query");
  return search_host_impl(h, q_host, q_lens, n_q, k, allow_masks_host, n_masks, mask_index_host, i8_q_scale, score_scale,
                          id_base, top_scores_host, top_ids_host, top_counts_host);
}
