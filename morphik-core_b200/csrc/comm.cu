// comm.cu -- the multi-GPU half of the C-ABI (SURVEY 8e / 8b "b200ms_allgather_topk"): one process per GPU, the corpus sharded
// by document, and per query batch exactly ONE collective -- an NCCL all-gather of every rank's top-k list (12 bytes per
// entry) over NVLink -- followed by a merge on every rank.  The reference has nothing comparable (single-process asyncio
// server); this is what lets a ctypes-only host run the sharded search without torch.distributed on the query path.
//
// NCCL is bound at run time (dlopen of libnccl.so.2: the copy already loaded by the host process -- e.g. torch's -- or the
// system one; B200MS_NCCL_LIB overrides), so libb200ms.so itself has no link-time dependency and still loads on a box
// without NCCL.  Only ncclGetUniqueId / ncclCommInitRank / ncclAllGather / ncclBroadcast / ncclCommDestroy are used.
//
// Pipelined search (b200ms_sharded_search_begin / _end, and the *_host_* forms): the local scan + top-k of step i run on the
// caller's stream and write straight into the exchange layout; the all-gather and the merge of step i run on the handle's
// (high-priority) communication stream behind an event, so the caller's stream can start the scan of step i+1 without
// waiting for the slowest rank -- two exchange slots, results are picked up one step later with _end.  A synchronous
// caller simply calls _end right after _begin.
#include <dlfcn.h>

#include <cstdlib>
#include <cstring>
#include <mutex>

#include "common.cuh"

namespace bms {

// ---- the slice of nccl.h this file needs (ABI-stable since NCCL 2.x)
typedef struct ncclComm* ncclComm_t;
typedef struct {
  char internal[128];
} ncclUniqueId;
typedef int ncclResult_t;  // ncclSuccess == 0
constexpr int kNcclChar = 0;  // ncclInt8 / ncclChar

struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*CommAbort)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  std::string where;
  bool ok = false;
};

static NcclApi& nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* lib = nullptr;
    std::vector<std::string> names;
    if (const char* e = getenv("B200MS_NCCL_LIB")) names.push_back(e);
    names.push_back("libnccl.so.2");
    names.push_back("libnccl.so");
    for (const std::string& n : names) {
      lib = dlopen(n.c_str(), RTLD_NOW | RTLD_GLOBAL | RTLD_NOLOAD);  // prefer the copy the host process already uses
      if (!lib) lib = dlopen(n.c_str(), RTLD_NOW | RTLD_GLOBAL);
      if (lib) {
        api.where = n;
        break;
      }
    }
    if (!lib) return;
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(lib, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(lib, "ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
    api.CommAbort = reinterpret_cast<decltype(api.CommAbort)>(dlsym(lib, "ncclCommAbort"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(lib, "ncclAllGather"));
    api.Broadcast = reinterpret_cast<decltype(api.Broadcast)>(dlsym(lib, "ncclBroadcast"));
    api.Send = reinterpret_cast<decltype(api.Send)>(dlsym(lib, "ncclSend"));
    api.Recv = reinterpret_cast<decltype(api.Recv)>(dlsym(lib, "ncclRecv"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
    api.GetVersion = reinterpret_cast<decltype(api.GetVersion)>(dlsym(lib, "ncclGetVersion"));
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.Broadcast;
  });
  return api;
}

static int check_nccl(b200ms_t* h, ncclResult_t r, const char* what) {
  if (r == 0) return B200MS_OK;
  NcclApi& a = nccl_api();
  return set_error(h, B200MS_ECUDA, std::string(what) + ": NCCL error " + std::to_string(r) + " (" +
                                        (a.GetErrorString ? a.GetErrorString(r) : "?") + ")");
}

constexpr int kSlots = 2;

struct Comm {
  ncclComm_t comm = nullptr;
  bool owned = false;
  int rank = 0, world = 1;
  cudaStream_t cstream = nullptr;  // communication stream (all-gather + merge), higher priority than the scan's stream
  // pipeline slots
  DeviceBuf xchg[kSlots], gath[kSlots], q_raw[kSlots], out_dev[kSlots], lcount[kSlots];
  PinnedBuf out_pin[kSlots];
  cudaEvent_t ev_local[kSlots] = {}, ev_gathered[kSlots] = {}, ev_done[kSlots] = {};
  bool used[kSlots] = {};
  bool host_pending[kSlots] = {};  // host pipeline: results of this slot not collected yet (b200ms_sharded_search_host_end)
  int out_nq[kSlots] = {}, out_k[kSlots] = {};
  int64_t ticket = 0;
};

static int ensure_comm_state(b200ms_t* h) {
  if (h->comm) return B200MS_OK;
  Comm* c = new Comm();
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  if (int e = check_cuda(h, cudaStreamCreateWithPriority(&c->cstream, cudaStreamNonBlocking, hi), "comm: stream create")) {
    delete c;
    return e;
  }
  for (int i = 0; i < kSlots; ++i) {
    if (cudaEventCreateWithFlags(&c->ev_local[i], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_gathered[i], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_done[i], cudaEventDisableTiming) != cudaSuccess) {
      const int e = check_cuda(h, cudaGetLastError(), "comm: event create");
      delete c;
      return e ? e : B200MS_ECUDA;
    }
  }
  h->comm = c;
  return B200MS_OK;
}

// ncclCommDestroy waits for the peers' matching call (measured: rank 0 sat in it forever while rank 1 had simply dropped its
// handle), which makes handle destruction a hidden collective.  Every operation this handle issued is complete by now (the
// caller synchronised the device), so the communicator is released with ncclCommAbort, which is local.
static void release_comm(Comm* c) {
  if (!c->comm || !c->owned || !nccl_api().ok) return;
  if (c->cstream) cudaStreamSynchronize(c->cstream);
  if (nccl_api().CommAbort) nccl_api().CommAbort(c->comm); else nccl_api().CommDestroy(c->comm);
  c->comm = nullptr;
}

void comm_teardown(b200ms_t* h) {
  Comm* c = h->comm;
  if (!c) return;
  release_comm(c);
  for (int i = 0; i < kSlots; ++i) {
    DeviceBuf* bufs[] = {&c->xchg[i], &c->gath[i], &c->q_raw[i], &c->out_dev[i], &c->lcount[i]};
    for (DeviceBuf* b : bufs)
      if (b->p) cudaFree(b->p);
    if (c->out_pin[i].p) cudaFreeHost(c->out_pin[i].p);
    if (c->ev_local[i]) cudaEventDestroy(c->ev_local[i]);
    if (c->ev_gathered[i]) cudaEventDestroy(c->ev_gathered[i]);
    if (c->ev_done[i]) cudaEventDestroy(c->ev_done[i]);
  }
  if (c->cstream) cudaStreamDestroy(c->cstream);
  delete c;
  h->comm = nullptr;
}

// all-gather the local exchange block and merge: enqueued on `s`
static int allgather_merge(b200ms_t* h, ncclComm_t comm, int world, const void* xchg_local, void* gathered, int n_q, int k,
                           float* ts, int64_t* ti, int32_t* tc, cudaStream_t s) {
  if (world > 1) {
    if (int e = check_nccl(h, nccl_api().AllGather(xchg_local, gathered, xchg_bytes(n_q, k), kNcclChar, comm, s), "ncclAllGather")) return e;
    h->launches++;  // the collective's kernel
  }
  return launch_merge_gathered(h, world > 1 ? gathered : xchg_local, world, n_q, k, ts, ti, tc, s);
}

}  // namespace bms

using namespace bms;

#define B200MS_API extern "C" __attribute__((visibility("default")))

B200MS_API int b200ms_comm_available(void) { return nccl_api().ok ? 1 : 0; }

B200MS_API int b200ms_comm_unique_id(uint8_t* id128) {
  if (!id128) return set_error(nullptr, B200MS_EINVAL, "comm_unique_id: NULL buffer");
  NcclApi& a = nccl_api();
  if (!a.ok) return set_error(nullptr, B200MS_ESTATE, "comm: libnccl.so.2 could not be loaded (set B200MS_NCCL_LIB)");
  ncclUniqueId id;
  if (int e = check_nccl(nullptr, a.GetUniqueId(&id), "ncclGetUniqueId")) return e;
  memcpy(id128, id.internal, 128);
  return B200MS_OK;
}

B200MS_API int b200ms_comm_init(b200ms_t* h, const uint8_t* id128, int rank, int world) {
  if (!h) return B200MS_EINVAL;
  if (!id128 || world < 1 || rank < 0 || rank >= world) return set_error(h, B200MS_EINVAL, "comm_init: bad arguments");
  NcclApi& a = nccl_api();
  if (world > 1 && !a.ok) return set_error(h, B200MS_ESTATE, "comm: libnccl.so.2 could not be loaded (set B200MS_NCCL_LIB)");
  DeviceGuard g(h->device);
  if (int e = ensure_comm_state(h)) return e;
  Comm* c = h->comm;
  release_comm(c);
  c->comm = nullptr;
  c->rank = rank;
  c->world = world;
  if (world > 1) {
    ncclUniqueId id;
    memcpy(id.internal, id128, 128);
    if (int e = check_nccl(h, a.CommInitRank(&c->comm, world, id, rank), "ncclCommInitRank")) return e;
    c->owned = true;
  }
  return B200MS_OK;
}

B200MS_API int b200ms_comm_adopt(b200ms_t* h, void* nccl_comm, int rank, int world) {
  if (!h) return B200MS_EINVAL;
  if (world < 1 || rank < 0 || rank >= world || (world > 1 && !nccl_comm)) return set_error(h, B200MS_EINVAL, "comm_adopt: bad arguments");
  if (world > 1 && !nccl_api().ok) return set_error(h, B200MS_ESTATE, "comm: libnccl.so.2 could not be loaded");
  DeviceGuard g(h->device);
  if (int e = ensure_comm_state(h)) return e;
  Comm* c = h->comm;
  release_comm(c);
  c->comm = static_cast<ncclComm_t>(nccl_comm);
  c->owned = false;
  c->rank = rank;
  c->world = world;
  return B200MS_OK;
}

B200MS_API int b200ms_comm_destroy(b200ms_t* h) {
  if (!h) return B200MS_EINVAL;
  DeviceGuard g(h->device);
  cudaDeviceSynchronize();
  comm_teardown(h);
  return B200MS_OK;
}

B200MS_API int b200ms_comm_rank(const b200ms_t* h) { return h && h->comm ? h->comm->rank : 0; }
B200MS_API int b200ms_comm_world(const b200ms_t* h) { return h && h->comm ? h->comm->world : 1; }
B200MS_API int64_t b200ms_xchg_bytes(int n_q, int k) { return n_q < 0 || k < 0 ? 0 : int64_t(xchg_bytes(n_q, k)); }

B200MS_API int b200ms_bcast_device(b200ms_t* h, void* buf, int64_t bytes, int root, void* stream) {
  if (!h) return B200MS_EINVAL;
  Comm* c = h->comm;
  if (!c) return set_error(h, B200MS_ESTATE, "bcast: call b200ms_comm_init first");
  if (bytes < 0 || (bytes > 0 && !buf) || root < 0 || root >= c->world) return set_error(h, B200MS_EINVAL, "bcast: bad arguments");
  if (c->world == 1 || bytes == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  StreamOrder order(h, static_cast<cudaStream_t>(stream));
  if (int e = order.error()) return e;
  h->launches++;
  return check_nccl(h, nccl_api().Broadcast(buf, buf, size_t(bytes), kNcclChar, root, c->comm, static_cast<cudaStream_t>(stream)), "ncclBroadcast");
}

// Point-to-point over the handle's communicator: ingest rows travel from the coordinating rank to the OWNING rank only.
B200MS_API int b200ms_send_device(b200ms_t* h, const void* buf, int64_t bytes, int peer, void* stream) {
  if (!h) return B200MS_EINVAL;
  Comm* c = h->comm;
  if (!c || !c->comm) return set_error(h, B200MS_ESTATE, "send: call b200ms_comm_init first (world > 1)");
  if (bytes < 0 || (bytes > 0 && !buf) || peer < 0 || peer >= c->world || peer == c->rank || !nccl_api().Send)
    return set_error(h, B200MS_EINVAL, "send: bad arguments (or ncclSend unavailable)");
  if (bytes == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  StreamOrder order(h, static_cast<cudaStream_t>(stream));
  if (int e = order.error()) return e;
  h->launches++;
  return check_nccl(h, nccl_api().Send(buf, size_t(bytes), kNcclChar, peer, c->comm, static_cast<cudaStream_t>(stream)), "ncclSend");
}

B200MS_API int b200ms_recv_device(b200ms_t* h, void* buf, int64_t bytes, int peer, void* stream) {
  if (!h) return B200MS_EINVAL;
  Comm* c = h->comm;
  if (!c || !c->comm) return set_error(h, B200MS_ESTATE, "recv: call b200ms_comm_init first (world > 1)");
  if (bytes < 0 || (bytes > 0 && !buf) || peer < 0 || peer >= c->world || peer == c->rank || !nccl_api().Recv)
    return set_error(h, B200MS_EINVAL, "recv: bad arguments (or ncclRecv unavailable)");
  if (bytes == 0) return B200MS_OK;
  DeviceGuard g(h->device);
  StreamOrder order(h, static_cast<cudaStream_t>(stream));
  if (int e = order.error()) return e;
  h->launches++;
  return check_nccl(h, nccl_api().Recv(buf, size_t(bytes), kNcclChar, peer, c->comm, static_cast<cudaStream_t>(stream)), "ncclRecv");
}

B200MS_API int b200ms_allgather_topk(b200ms_t* h, void* nccl_comm, const void* xchg_local, int n_q, int k, float* top_scores,
                                     int64_t* top_ids, int32_t* top_counts, void* stream) {
  if (!h) return B200MS_EINVAL;
  Comm* c = h->comm;
  if (!c) return set_error(h, B200MS_ESTATE, "allgather_topk: call b200ms_comm_init (or b200ms_comm_adopt) first");
  DeviceGuard g(h->device);
  const int world = c->world;
  if (n_q < 1 || k < 1 || k > B200MS_MAX_K || int64_t(world) * k > 2 * B200MS_MAX_K || !xchg_local || !top_scores || !top_ids || !top_counts)
    return set_error(h, B200MS_EINVAL, "allgather_topk: bad arguments (world * k <= 8192)");
  ncclComm_t comm = nccl_comm ? static_cast<ncclComm_t>(nccl_comm) : c->comm;
  if (world > 1 && !comm) return set_error(h, B200MS_ESTATE, "allgather_topk: no communicator");
  if (int e = reserve(h, c->gath[0], xchg_bytes(n_q, k) * size_t(world))) return e;
  StreamOrder order(h, static_cast<cudaStream_t>(stream));
  if (int e = order.error()) return e;
  return allgather_merge(h, comm, world, xchg_local, c->gath[0].p, n_q, k, top_scores, top_ids, top_counts,
                         static_cast<cudaStream_t>(stream));
}

// ---- pipelined sharded search ----------------------------------------------------------------------------------------
// r's outputs receive the merged result (on the communication stream)
static int sharded_begin(b200ms_t* h, const SearchRequest& r, const SearchMeta& m, cudaStream_t s, int* slot_out) {
  if (int e = ensure_comm_state(h)) return e;
  Comm* c = h->comm;
  const int world = c->world;
  if (r.n_q < 1 || r.k < 1 || r.k > B200MS_MAX_K || int64_t(world) * r.k > 2 * B200MS_MAX_K)
    return set_error(h, B200MS_EINVAL, "sharded_search: bad arguments (n_q >= 1, world * k <= 8192)");
  if (world > 1 && !c->comm) return set_error(h, B200MS_ESTATE, "sharded_search: call b200ms_comm_init first");
  const int slot = int(c->ticket % kSlots);
  const size_t xb = xchg_bytes(r.n_q, r.k);
  if (c->used[slot]) {
    // the slot's previous exchange must have left the send buffer before the local top-k overwrites it
    if (int e = check_cuda(h, cudaStreamWaitEvent(s, c->ev_gathered[slot], 0), "sharded_search: wait gathered")) return e;
  }
  if (int e = reserve(h, c->xchg[slot], xb)) return e;
  if (int e = reserve(h, c->gath[slot], xb * size_t(world))) return e;
  if (int e = reserve(h, c->lcount[slot], size_t(r.n_q) * 4)) return e;
  void* x = c->xchg[slot].p;
  // local scan + top-k with global ids, written straight into the exchange layout (the local counts are not exchanged:
  // unused entries carry id -1; they go to scratch so that a caller reusing its output buffers across pipelined steps
  // never has two streams writing top_counts)
  const ResultBlock xl(r.n_q, r.k);
  SearchRequest local = r;
  local.top_ids = xl.ids(x);
  local.top_scores = xl.scores(x);
  local.top_counts = static_cast<int32_t*>(c->lcount[slot].p);
  if (int e = search_core(h, local, m, s)) return e;
  if (int e = check_cuda(h, cudaEventRecord(c->ev_local[slot], s), "sharded_search: record local")) return e;
  if (int e = check_cuda(h, cudaStreamWaitEvent(c->cstream, c->ev_local[slot], 0), "sharded_search: wait local")) return e;
  if (world > 1) {
    if (int e = check_nccl(h, nccl_api().AllGather(x, c->gath[slot].p, xb, kNcclChar, c->comm, c->cstream), "ncclAllGather")) return e;
    h->launches++;
  }
  if (int e = check_cuda(h, cudaEventRecord(c->ev_gathered[slot], c->cstream), "sharded_search: record gathered")) return e;
  if (int e = launch_merge_gathered(h, world > 1 ? c->gath[slot].p : x, world, r.n_q, r.k, r.top_scores, r.top_ids,
                                    r.top_counts, c->cstream))
    return e;
  c->used[slot] = true;
  *slot_out = slot;
  return B200MS_OK;
}

static const char* const kShardedHostCorpus =
    "sharded search: the attached corpus is host-resident (b200ms_set_corpus_host); only candidate scoring is supported";

B200MS_API int64_t b200ms_sharded_search_begin(b200ms_t* h, const void* q_dev, int src_dtype, const int32_t* q_lens, int n_q,
                                               int k, const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                               float i8_q_scale, float score_scale, int64_t id_base, float* top_scores_dev,
                                               int64_t* top_ids_dev, int32_t* top_counts_dev, void* stream) {
  if (!h) return B200MS_EINVAL;
  if (h->corpus.host) return set_error(h, B200MS_ESTATE, kShardedHostCorpus);
  if ((src_dtype != B200MS_F32 && src_dtype != B200MS_BF16) || !top_scores_dev || !top_ids_dev || !top_counts_dev ||
      n_masks < 0 || (n_masks > 0 && (!allow_masks_dev || !mask_index_dev)))
    return set_error(h, B200MS_EINVAL, "sharded_search_begin: bad arguments");
  DeviceGuard g(h->device);
  SearchRequest r{q_dev, src_dtype, q_lens, n_q, k, i8_q_scale, score_scale, top_scores_dev, top_ids_dev, top_counts_dev, id_base};
  if (n_masks > 0) {
    r.allow = allow_masks_dev;
    r.mask_index = mask_index_dev;
  }
  int slot = 0;
  {
    // ordered on the caller's stream, where the local search runs; the merge on the communication stream reads only
    // this slot's buffers
    StreamOrder order(h, static_cast<cudaStream_t>(stream));
    if (int e = order.error()) return e;
    if (int e = sharded_begin(h, r, build_search_meta(q_lens, n_q), static_cast<cudaStream_t>(stream), &slot)) return e;
  }
  Comm* c = h->comm;
  if (int e = check_cuda(h, cudaEventRecord(c->ev_done[slot], c->cstream), "sharded_search: record done")) return e;
  return c->ticket++;
}

B200MS_API int b200ms_sharded_search_end(b200ms_t* h, int64_t ticket, void* stream) {
  if (!h) return B200MS_EINVAL;
  Comm* c = h->comm;
  if (!c || ticket < 0 || ticket >= c->ticket || ticket + kSlots < c->ticket)
    return set_error(h, B200MS_EINVAL, "sharded_search_end: unknown or expired ticket (at most 2 searches in flight)");
  DeviceGuard g(h->device);
  return check_cuda(h, cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), c->ev_done[int(ticket % kSlots)], 0),
                    "sharded_search_end: wait done");
}

B200MS_API int64_t b200ms_sharded_search_host_begin(b200ms_t* h, const float* q_host, const int32_t* q_lens, int n_q, int k,
                                                    const uint32_t* allow_masks_dev, int n_masks, const int32_t* mask_index_dev,
                                                    float i8_q_scale, float score_scale, int64_t id_base) {
  if (!h) return B200MS_EINVAL;
  if (h->corpus.host) return set_error(h, B200MS_ESTATE, kShardedHostCorpus);
  if (!q_host || !q_lens || n_q < 1 || n_masks < 0 || (n_masks > 0 && (!allow_masks_dev || !mask_index_dev)))
    return set_error(h, B200MS_EINVAL, "sharded_search_host_begin: bad arguments");
  DeviceGuard g(h->device);
  if (int e = ensure_comm_state(h)) return e;
  Comm* c = h->comm;
  const int slot = int(c->ticket % kSlots);
  if (c->host_pending[slot])
    return set_error(h, B200MS_ESTATE, "sharded_search_host_begin: two searches are in flight -- collect the older one with "
                                       "b200ms_sharded_search_host_end first");
  cudaStream_t s = h->stream;
  StreamOrder order(h, s);
  if (int e = order.error()) return e;
  const SearchMeta m = build_search_meta(q_lens, n_q);
  const ResultBlock rb(n_q, k);
  if (int e = reserve(h, c->q_raw[slot], size_t(m.rows > 0 ? m.rows : 1) * kDim * 4)) return e;
  if (int e = reserve(h, c->out_dev[slot], rb.bytes())) return e;
  if (int e = reserve_pinned(h, c->out_pin[slot], rb.bytes())) return e;
  if (m.rows > 0)
    if (int e = check_cuda(h, cudaMemcpyAsync(c->q_raw[slot].p, q_host, size_t(m.rows) * kDim * 4, cudaMemcpyHostToDevice, s),
                           "sharded_search_host: H2D queries"))
      return e;
  void* od = c->out_dev[slot].p;
  SearchRequest r{c->q_raw[slot].p, B200MS_F32, q_lens, n_q, k, i8_q_scale, score_scale, rb.scores(od), rb.ids(od), rb.counts(od),
                  id_base};
  if (n_masks > 0) {
    r.allow = allow_masks_dev;
    r.mask_index = mask_index_dev;
  }
  int sl = 0;
  if (int e = sharded_begin(h, r, m, s, &sl)) return e;
  if (int e = check_cuda(h, cudaMemcpyAsync(c->out_pin[slot].p, od, rb.bytes(), cudaMemcpyDeviceToHost, c->cstream),
                         "sharded_search_host: D2H results"))
    return e;
  if (int e = check_cuda(h, cudaEventRecord(c->ev_done[slot], c->cstream), "sharded_search_host: record done")) return e;
  c->out_nq[slot] = n_q;
  c->out_k[slot] = k;
  c->host_pending[slot] = true;
  return c->ticket++;
}

B200MS_API int b200ms_sharded_search_host_end(b200ms_t* h, int64_t ticket, float* top_scores_host, int64_t* top_ids_host,
                                              int32_t* top_counts_host) {
  if (!h) return B200MS_EINVAL;
  Comm* c = h->comm;
  if (!c || ticket < 0 || ticket >= c->ticket || ticket + kSlots < c->ticket || !top_scores_host || !top_ids_host || !top_counts_host)
    return set_error(h, B200MS_EINVAL, "sharded_search_host_end: unknown or expired ticket, or NULL outputs");
  DeviceGuard g(h->device);
  const int slot = int(ticket % kSlots);
  if (int e = check_cuda(h, cudaEventSynchronize(c->ev_done[slot]), "sharded_search_host_end: sync")) return e;
  ResultBlock(c->out_nq[slot], c->out_k[slot]).unpack(c->out_pin[slot].p, top_scores_host, top_ids_host, top_counts_host);
  c->host_pending[slot] = false;
  return B200MS_OK;
}
