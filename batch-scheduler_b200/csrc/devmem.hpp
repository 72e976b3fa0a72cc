// devmem.hpp — compressible device memory: an allocation made through the driver's virtual-memory calls with
// CU_MEM_ALLOCATION_COMP_GENERIC, so that on GPUs with Compute Data Compression the L2 compresses its lines on
// their way to DRAM.  Compression is invisible to every reader and writer (kernels, TMA bulk stores, cudaMemcpy*);
// only the number of bytes that reach DRAM changes.  The driver calls are resolved through the runtime
// (cudaGetDriverEntryPointByVersion), so nothing links libcuda directly.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstddef>

namespace bsk {

struct CompMem {
  void* p = nullptr;
  size_t bytes = 0;                        // mapped size: the request rounded up to the allocation granularity
  CUmemGenericAllocationHandle handle = 0;
};

namespace compmem_detail {

struct Driver {
  bool ok = false;
  decltype(&cuDeviceGet) device_get = nullptr;
  decltype(&cuDeviceGetAttribute) attribute = nullptr;
  decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
  decltype(&cuMemAddressReserve) reserve = nullptr;
  decltype(&cuMemAddressFree) address_free = nullptr;
  decltype(&cuMemCreate) create = nullptr;
  decltype(&cuMemRelease) release = nullptr;
  decltype(&cuMemGetAllocationPropertiesFromHandle) props = nullptr;
  decltype(&cuMemMap) map = nullptr;
  decltype(&cuMemUnmap) unmap = nullptr;
  decltype(&cuMemSetAccess) set_access = nullptr;
};

template <class F>
inline bool entry(const char* name, F* fn) {
  cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
  void* p = nullptr;
  if (cudaGetDriverEntryPointByVersion(name, &p, 12000, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess || !p)
    return false;
  *fn = reinterpret_cast<F>(p);
  return true;
}

inline const Driver& driver() {
  static const Driver d = [] {
    Driver r;
    r.ok = entry("cuDeviceGet", &r.device_get) && entry("cuDeviceGetAttribute", &r.attribute) &&
           entry("cuMemGetAllocationGranularity", &r.granularity) && entry("cuMemAddressReserve", &r.reserve) &&
           entry("cuMemAddressFree", &r.address_free) && entry("cuMemCreate", &r.create) &&
           entry("cuMemRelease", &r.release) && entry("cuMemGetAllocationPropertiesFromHandle", &r.props) &&
           entry("cuMemMap", &r.map) && entry("cuMemUnmap", &r.unmap) && entry("cuMemSetAccess", &r.set_access);
    return r;
  }();
  return d;
}

}  // namespace compmem_detail

// CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED of the current device (0 when it cannot be read).
inline int compmem_supported() {
  const auto& d = compmem_detail::driver();
  int ord = 0, v = 0;
  CUdevice dev;
  if (!d.ok || cudaGetDevice(&ord) != cudaSuccess || d.device_get(&dev, ord) != CUDA_SUCCESS) return 0;
  if (d.attribute(&v, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, dev) != CUDA_SUCCESS) return 0;
  return v;
}

inline void compmem_free(CompMem* m) {
  const auto& d = compmem_detail::driver();
  if (m->p) {
    // cudaFree waits for the device before it frees; unmapping is not documented to, so wait here
    cudaDeviceSynchronize();
    d.unmap((CUdeviceptr)m->p, m->bytes);
  }
  if (m->handle) d.release(m->handle);
  if (m->p) d.address_free((CUdeviceptr)m->p, m->bytes);
  *m = CompMem{};
}

// Allocates at least `bytes` of compressible memory on the current device and makes it readable and writable
// there.  Returns false, with *m empty and nothing held, when the device does not support compression, the
// driver does not grant it for this allocation, or any of the calls fails; the caller then uses cudaMalloc.
inline bool compmem_alloc(CompMem* m, size_t bytes) {
  *m = CompMem{};
  const auto& d = compmem_detail::driver();
  int ord = 0;
  if (!compmem_supported() || cudaGetDevice(&ord) != cudaSuccess) return false;
  CUmemAllocationProp prop = {};
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = ord;
  prop.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
  size_t gran = 0;
  if (d.granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS || gran == 0) return false;
  const size_t size = (bytes + gran - 1) / gran * gran;
  CUdeviceptr va = 0;
  if (d.reserve(&va, size, gran, 0, 0) != CUDA_SUCCESS) return false;
  CUmemGenericAllocationHandle h = 0;
  if (d.create(&h, size, &prop, 0) != CUDA_SUCCESS) {
    d.address_free(va, size);
    return false;
  }
  // the driver may hand out uncompressed memory for a compressible request: only a granted allocation is kept
  CUmemAllocationProp got = {};
  if (d.props(&got, h) != CUDA_SUCCESS || got.allocFlags.compressionType != CU_MEM_ALLOCATION_COMP_GENERIC ||
      d.map(va, size, 0, h, 0) != CUDA_SUCCESS) {
    d.release(h);
    d.address_free(va, size);
    return false;
  }
  m->p = (void*)va;
  m->bytes = size;
  m->handle = h;
  CUmemAccessDesc acc = {};
  acc.location = prop.location;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if (d.set_access(va, size, &acc, 1) != CUDA_SUCCESS) {
    compmem_free(m);
    return false;
  }
  return true;
}

}  // namespace bsk
