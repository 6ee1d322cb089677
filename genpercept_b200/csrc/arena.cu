// The per-device activation arena that the plans of every engine with gp_set_shared_arena on share.
//
// One virtual range as large as the device's memory is reserved at first use, so its base never moves: op lists, TMA
// descriptors and captured CUDA graphs built against it stay valid while physical memory is mapped and unmapped behind
// it.  The mapped size follows the largest arena among the live plans in the pool.  The driver's virtual-memory calls
// are reached through cudaGetDriverEntryPoint, as igemm.cu reaches cuTensorMapEncodeTiled, so the library links no
// libcuda.
#include <cuda.h>

#include <mutex>
#include <set>

#include "engine.h"

namespace gp {

namespace {

struct Driver {
  CUresult (*reserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*free_range)(CUdeviceptr, size_t) = nullptr;
  CUresult (*create)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*release)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*map)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*unmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*set_access)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*granularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
};

template <class F>
void entry(const char* name, F* fn) {
  void* f = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
    throw GpError(GP_ERR_CUDA, std::string("shared arena: the driver has no ") + name);
  *fn = reinterpret_cast<F>(f);
}

const Driver& driver() {
  static Driver d;
  static bool ok = false;
  if (!ok) {
    entry("cuMemAddressReserve", &d.reserve);
    entry("cuMemAddressFree", &d.free_range);
    entry("cuMemCreate", &d.create);
    entry("cuMemRelease", &d.release);
    entry("cuMemMap", &d.map);
    entry("cuMemUnmap", &d.unmap);
    entry("cuMemSetAccess", &d.set_access);
    entry("cuMemGetAllocationGranularity", &d.granularity);
    ok = true;
  }
  return d;
}

void check(CUresult r, const char* what) {
  if (r != CUDA_SUCCESS) throw GpError(GP_ERR_CUDA, std::string("shared arena: ") + what + " failed (CUresult " +
                                                        std::to_string((int)r) + ")");
}

struct Chunk { size_t off, size; CUmemGenericAllocationHandle h; };

struct Pool {
  int device = 0;
  CUdeviceptr base = 0;
  size_t reserved = 0, mapped = 0, gran = 0;
  std::vector<Chunk> chunks;      // back to back from base, covering [0, mapped)
  std::multiset<size_t> plans;    // arena_bytes of every live plan in the pool
  int engines = 0;
  cudaEvent_t last_use = nullptr;

  CUmemAllocationProp prop() const {
    CUmemAllocationProp p = {};
    p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    p.location.id = device;
    return p;
  }
  size_t round(size_t b) const { return (b + gran - 1) / gran * gran; }

  // Backs [off, off + size) with a new physical allocation; false (nothing changed) when the device is out of memory.
  bool map_chunk(size_t off, size_t size, Chunk* out) {
    const Driver& d = driver();
    const CUmemAllocationProp p = prop();
    CUmemGenericAllocationHandle h;
    const CUresult r = d.create(&h, size, &p, 0);
    if (r == CUDA_ERROR_OUT_OF_MEMORY) return false;
    check(r, "cuMemCreate");
    if (d.map(base + off, size, 0, h, 0) != CUDA_SUCCESS) { d.release(h); return false; }
    CUmemAccessDesc a = {};
    a.location = p.location;
    a.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if (d.set_access(base + off, size, &a, 1) != CUDA_SUCCESS) {
      d.unmap(base + off, size);
      d.release(h);
      return false;
    }
    *out = {off, size, h};
    return true;
  }

  // Maps up to `need` (a multiple of gran); false when the device cannot back it (the mapping is left as it was).
  bool grow(size_t need) {
    if (need <= mapped) return true;
    if (need > reserved) return false;
    Chunk c;
    if (!map_chunk(mapped, need - mapped, &c)) return false;
    chunks.push_back(c);
    mapped = need;
    return true;
  }

  // Unmaps down to `need` (a multiple of gran).  The caller has synchronised the device.  A chunk that straddles `need`
  // is replaced by a smaller one; its contents are not kept (no plan keeps data across calls, see gp_set_shared_arena).
  void shrink(size_t need) {
    const Driver& d = driver();
    while (mapped > need) {
      Chunk c = chunks.back();
      if (c.off >= need) {
        d.unmap(base + c.off, c.size);
        d.release(c.h);
        chunks.pop_back();
        mapped = c.off;
        continue;
      }
      // keep the old chunk unless the smaller one is in place
      const CUmemAllocationProp p = prop();
      CUmemGenericAllocationHandle h;
      if (d.create(&h, need - c.off, &p, 0) != CUDA_SUCCESS) return;
      d.unmap(base + c.off, c.size);
      CUmemAccessDesc a = {};
      a.location = p.location;
      a.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      if (d.map(base + c.off, need - c.off, 0, h, 0) != CUDA_SUCCESS ||
          d.set_access(base + c.off, need - c.off, &a, 1) != CUDA_SUCCESS) {
        d.unmap(base + c.off, need - c.off);
        d.release(h);
        d.map(base + c.off, c.size, 0, c.h, 0);
        d.set_access(base + c.off, c.size, &a, 1);
        return;
      }
      d.release(c.h);
      chunks.back() = {c.off, need - c.off, h};
      mapped = need;
    }
  }
};

std::mutex g_mu;
std::map<int, Pool> g_pools;

Pool& pool(int device) {
  auto it = g_pools.find(device);
  if (it == g_pools.end()) throw GpError(GP_ERR_STATE, "shared arena: no engine on device " + std::to_string(device) + " shares it");
  return it->second;
}

}  // namespace

void shared_arena_join(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_pools.find(device);
  if (it != g_pools.end()) { it->second.engines++; return; }
  const Driver& d = driver();
  Pool p;
  p.device = device;
  const CUmemAllocationProp pr = p.prop();
  check(d.granularity(&p.gran, &pr, CU_MEM_ALLOC_GRANULARITY_MINIMUM), "cuMemGetAllocationGranularity");
  size_t free_b = 0, total_b = 0;
  GP_CUDA(cudaMemGetInfo(&free_b, &total_b));
  p.reserved = p.round(total_b);
  check(d.reserve(&p.base, p.reserved, 0, 0, 0), "cuMemAddressReserve");
  if (cudaEventCreateWithFlags(&p.last_use, cudaEventDisableTiming) != cudaSuccess) {
    d.free_range(p.base, p.reserved);
    throw GpError(GP_ERR_CUDA, "shared arena: cudaEventCreateWithFlags failed");
  }
  p.engines = 1;
  g_pools[device] = std::move(p);
}

void shared_arena_leave(int device) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_pools.find(device);
  if (it == g_pools.end() || --it->second.engines > 0) return;
  Pool& p = it->second;
  cudaDeviceSynchronize();
  p.shrink(0);
  driver().free_range(p.base, p.reserved);
  cudaEventDestroy(p.last_use);
  g_pools.erase(it);
}

uint8_t* shared_arena_add(int device, size_t bytes) {
  std::lock_guard<std::mutex> lk(g_mu);
  Pool& p = pool(device);
  if (!p.grow(p.round(std::max(bytes, p.mapped)))) return nullptr;
  p.plans.insert(bytes);
  return reinterpret_cast<uint8_t*>(p.base);
}

void shared_arena_remove(int device, size_t bytes) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_pools.find(device);
  if (it == g_pools.end()) return;
  Pool& p = it->second;
  auto jt = p.plans.find(bytes);
  if (jt == p.plans.end()) return;
  p.plans.erase(jt);
  const size_t need = p.plans.empty() ? 0 : p.round(*p.plans.rbegin());
  if (need < p.mapped) {
    cudaDeviceSynchronize();
    p.shrink(need);
  }
}

void shared_arena_wait(int device, cudaStream_t s) {
  std::lock_guard<std::mutex> lk(g_mu);
  GP_CUDA(cudaStreamWaitEvent(s, pool(device).last_use, 0));
}

void shared_arena_record(int device, cudaStream_t s) noexcept {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_pools.find(device);
  if (it != g_pools.end()) cudaEventRecord(it->second.last_use, s);
}

}  // namespace gp

extern "C" {

gp_status gp_shared_arena_info(int device, int64_t* mapped_bytes, int64_t* reserved_bytes, int64_t* live_plans) {
  std::lock_guard<std::mutex> lk(gp::g_mu);
  auto it = gp::g_pools.find(device);
  const bool on = it != gp::g_pools.end();
  if (mapped_bytes) *mapped_bytes = on ? (int64_t)it->second.mapped : 0;
  if (reserved_bytes) *reserved_bytes = on ? (int64_t)it->second.reserved : 0;
  if (live_plans) *live_plans = on ? (int64_t)it->second.plans.size() : 0;
  return GP_OK;
}

gp_status gp_shared_arena_fill(int device, int byte, void* stream) {
  return gp::guarded_call([&]() {
    std::lock_guard<std::mutex> lk(gp::g_mu);
    gp::Pool& p = gp::pool(device);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    GP_CUDA(cudaSetDevice(device));
    GP_CUDA(cudaStreamWaitEvent(s, p.last_use, 0));
    if (p.mapped) GP_CUDA(cudaMemsetAsync(reinterpret_cast<void*>(p.base), byte & 0xFF, p.mapped, s));
    GP_CUDA(cudaEventRecord(p.last_use, s));
  });
}

}  // extern "C"
