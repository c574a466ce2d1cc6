// block.cu -- growable device blocks (b200ms_block_*): one reserved range of device virtual addresses per block, backed
// chunk by chunk with physical memory through the driver's virtual memory management calls.
//
// A corpus that is ingested and deleted from for as long as the store lives cannot be sized in advance.  In a cudaMalloc'd
// buffer, growing means a second, larger buffer and a copy (old + new resident at once), and memory freed by a compaction
// can only be handed back by allocating a smaller buffer and copying again.  Here the rows keep their address: growing maps
// more chunks behind the mapped ones, shrinking unmaps chunks from the tail and releases them to the driver.
#include <mutex>

#include "common.cuh"

struct b200ms_block {
  b200ms_t* owner = nullptr;
  CUdeviceptr base = 0;
  int64_t max_bytes = 0;
  size_t reserved = 0;                                // bytes of address space: max_bytes rounded up to whole chunks
  std::vector<CUmemGenericAllocationHandle> chunks;   // chunk i backs [base + i * chunk, base + (i + 1) * chunk)
};

namespace bms {

constexpr size_t kChunk = size_t(B200MS_BLOCK_CHUNK_BYTES);

// The driver entry points, fetched through the runtime like cuTensorMapEncodeTiled (no link dependency on libcuda).
struct VmmApi {
  decltype(&cuMemAddressReserve) reserve = nullptr;
  decltype(&cuMemAddressFree) address_free = nullptr;
  decltype(&cuMemCreate) create = nullptr;
  decltype(&cuMemRelease) release = nullptr;
  decltype(&cuMemMap) map = nullptr;
  decltype(&cuMemUnmap) unmap = nullptr;
  decltype(&cuMemSetAccess) set_access = nullptr;
  decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
  bool ok = false;
};

template <typename Fn>
static bool fetch(const char* name, Fn* out) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
    cudaGetLastError();
    return false;
  }
  *out = reinterpret_cast<Fn>(p);
  return true;
}

static const VmmApi* vmm_api(b200ms_t* h) {
  static std::once_flag once;
  static VmmApi api;
  std::call_once(once, [] {
    api.ok = fetch("cuMemAddressReserve", &api.reserve) && fetch("cuMemAddressFree", &api.address_free) &&
             fetch("cuMemCreate", &api.create) && fetch("cuMemRelease", &api.release) && fetch("cuMemMap", &api.map) &&
             fetch("cuMemUnmap", &api.unmap) && fetch("cuMemSetAccess", &api.set_access) &&
             fetch("cuMemGetAllocationGranularity", &api.granularity);
  });
  if (!api.ok) {
    set_error(h, B200MS_ECUDA, "the driver's virtual memory management entry points (cuMemCreate, cuMemMap, ...) are not available");
    return nullptr;
  }
  return &api;
}

static int check_cu(b200ms_t* h, CUresult r, const char* what) {
  if (r == CUDA_SUCCESS) return B200MS_OK;
  return set_error(h, B200MS_ECUDA, std::string(what) + " failed with CUresult " + std::to_string(int(r)));
}

static CUmemAllocationProp chunk_prop(const b200ms_t* h) {
  CUmemAllocationProp prop = {};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = h->device;
  return prop;
}

// Unmap and release the chunks at and past index `keep`, last first.
static void drop_tail(const VmmApi* v, b200ms_block* b, size_t keep) {
  while (b->chunks.size() > keep) {
    const size_t i = b->chunks.size() - 1;
    v->unmap(b->base + i * kChunk, kChunk);
    v->release(b->chunks[i]);
    b->chunks.pop_back();
  }
}

// Memory about to be unmapped may still be read or written by the handle's last call: wait for it.
static int wait_for_handle(b200ms_t* h) {
  if (!h->order_pending) return B200MS_OK;
  if (int e = check_cuda(h, cudaEventSynchronize(h->order_ev), "block: wait for the handle's previous call")) return e;
  h->order_pending = false;
  return B200MS_OK;
}

static bool owns(const b200ms_t* h, const b200ms_block* b) {
  for (const b200ms_block* x : h->blocks)
    if (x == b) return true;
  return false;
}

static int destroy_block(b200ms_t* h, const VmmApi* v, b200ms_block* b) {
  drop_tail(v, b, 0);
  const int e = check_cu(h, v->address_free(b->base, b->reserved), "cuMemAddressFree");
  delete b;
  return e;
}

void release_blocks(b200ms_t* h) {
  if (h->blocks.empty()) return;
  if (const VmmApi* v = vmm_api(h))
    for (b200ms_block* b : h->blocks) destroy_block(h, v, b);
  h->blocks.clear();
}

}  // namespace bms

using namespace bms;

#define B200MS_API extern "C" __attribute__((visibility("default")))

B200MS_API int b200ms_block_create(b200ms_t* h, int64_t max_bytes, b200ms_block_t** out) {
  if (!h) return B200MS_EINVAL;
  if (!out || max_bytes < 0) return set_error(h, B200MS_EINVAL, "block_create: bad arguments");
  *out = nullptr;
  DeviceGuard g(h->device);
  const VmmApi* v = vmm_api(h);
  if (!v) return B200MS_ECUDA;
  const CUmemAllocationProp prop = chunk_prop(h);
  size_t gran = 0;
  if (int e = check_cu(h, v->granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM), "cuMemGetAllocationGranularity")) return e;
  if (gran == 0 || kChunk % gran)
    return set_error(h, B200MS_ECUDA, "block_create: the chunk size is not a multiple of the device's allocation granularity (" +
                                          std::to_string(gran) + " bytes)");
  b200ms_block* b = new b200ms_block();
  b->owner = h;
  b->max_bytes = max_bytes;
  b->reserved = (size_t(max_bytes > 0 ? max_bytes : 1) + kChunk - 1) / kChunk * kChunk;
  if (int e = check_cu(h, v->reserve(&b->base, b->reserved, 0, 0, 0), "cuMemAddressReserve")) {
    delete b;
    return e;
  }
  h->blocks.push_back(b);
  *out = b;
  return B200MS_OK;
}

B200MS_API int b200ms_block_resize(b200ms_t* h, b200ms_block_t* b, int64_t bytes) {
  if (!h) return B200MS_EINVAL;
  if (!b || !owns(h, b) || bytes < 0 || bytes > b->max_bytes)
    return set_error(h, B200MS_EINVAL, "block_resize: bad arguments (a block of this handle, 0 <= bytes <= max_bytes)");
  DeviceGuard g(h->device);
  const VmmApi* v = vmm_api(h);
  if (!v) return B200MS_ECUDA;
  const size_t have = b->chunks.size(), want = (size_t(bytes) + kChunk - 1) / kChunk;
  if (want < have) {
    if (int e = wait_for_handle(h)) return e;
    drop_tail(v, b, want);
    return B200MS_OK;
  }
  if (want == have) return B200MS_OK;
  // refuse what cannot fit before creating anything: cuMemCreate of the last few chunks the card has would push every
  // other allocation on it (this process's scratch included) into failure
  size_t free_b = 0, total_b = 0;
  if (int e = check_cuda(h, cudaMemGetInfo(&free_b, &total_b), "block_resize: cudaMemGetInfo")) return e;
  const size_t add = (want - have) * kChunk;
  const std::string nomem = "block_resize: " + std::to_string(add) + " more bytes do not fit the device";
  if (add > free_b) return set_error(h, B200MS_ENOMEM, nomem + " (" + std::to_string(free_b) + " free)");
  const CUmemAllocationProp prop = chunk_prop(h);
  for (size_t i = have; i < want; ++i) {
    CUmemGenericAllocationHandle mem;
    if (v->create(&mem, kChunk, &prop, 0) != CUDA_SUCCESS) {  // another process took the memory in between
      drop_tail(v, b, have);
      return set_error(h, B200MS_ENOMEM, nomem + " (cuMemCreate failed)");
    }
    if (int e = check_cu(h, v->map(b->base + i * kChunk, kChunk, 0, mem, 0), "cuMemMap")) {
      v->release(mem);
      drop_tail(v, b, have);
      return e;
    }
    b->chunks.push_back(mem);
  }
  CUmemAccessDesc access = {};
  access.location = prop.location;
  access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if (int e = check_cu(h, v->set_access(b->base + have * kChunk, add, &access, 1), "cuMemSetAccess")) {
    drop_tail(v, b, have);
    return e;
  }
  return B200MS_OK;
}

B200MS_API void* b200ms_block_ptr(const b200ms_block_t* b) { return b ? reinterpret_cast<void*>(b->base) : nullptr; }

B200MS_API int64_t b200ms_block_mapped_bytes(const b200ms_block_t* b) { return b ? int64_t(b->chunks.size() * kChunk) : 0; }

B200MS_API int b200ms_block_destroy(b200ms_t* h, b200ms_block_t* b) {
  if (!h) return B200MS_EINVAL;
  if (!b || !owns(h, b)) return set_error(h, B200MS_EINVAL, "block_destroy: not a block of this handle");
  DeviceGuard g(h->device);
  const VmmApi* v = vmm_api(h);
  if (!v) return B200MS_ECUDA;
  if (int e = wait_for_handle(h)) return e;
  for (size_t i = 0; i < h->blocks.size(); ++i)
    if (h->blocks[i] == b) {
      h->blocks.erase(h->blocks.begin() + i);
      break;
    }
  return destroy_block(h, v, b);
}
