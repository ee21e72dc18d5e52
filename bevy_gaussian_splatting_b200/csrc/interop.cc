// interop.cc -- frame hand-back without a copy (SURVEY.md §8 f4): the frame target lives in an allocation that is
// exportable as an OS handle (POSIX file descriptor), which Vulkan -- and therefore wgpu-hal / Bevy's render device --
// imports with VK_KHR_external_memory_fd as the memory of the view-target image / a buffer it copies from.
//
// Replaces, on the CUDA path, the role of the render pass attachment the reference draws into
// (src/render/mod.rs:1501-1569 binds pipelines that write the view target); here bgs_render writes it through a
// CUDA device pointer.  Synchronisation: bgs_render (synchronous) or bgs_sync() returns after the frame is complete;
// a timeline semaphore exported by Vulkan can be imported into CUDA by the host later (cudaImportExternalSemaphore) --
// out of scope here.
//
// The CUDA driver API is resolved lazily with dlopen (like NCCL in gather.cc): libbgs.so itself links only cudart.
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <unistd.h>

#include <cstdio>
#include <mutex>
#include <vector>

#include "../../include/bgs.h"

namespace {

struct DrvApi {
    void* lib = nullptr;
    CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
    CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
    CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
    CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
    CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
    CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
    CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
    CUresult (*MemUnmap)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemAddressFree)(CUdeviceptr, size_t) = nullptr;
    CUresult (*MemRelease)(CUmemGenericAllocationHandle) = nullptr;
    bool ok = false;
};

DrvApi& drv() {
    static DrvApi a;
    static std::once_flag once;
    std::call_once(once, [] {
        a.lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
        if (!a.lib) return;
#define SYM(field, name) *(void**)(&a.field) = dlsym(a.lib, name)
        SYM(MemGetAllocationGranularity, "cuMemGetAllocationGranularity");
        SYM(MemCreate, "cuMemCreate");
        SYM(MemExportToShareableHandle, "cuMemExportToShareableHandle");
        SYM(MemImportFromShareableHandle, "cuMemImportFromShareableHandle");
        SYM(MemAddressReserve, "cuMemAddressReserve");
        SYM(MemMap, "cuMemMap");
        SYM(MemSetAccess, "cuMemSetAccess");
        SYM(MemUnmap, "cuMemUnmap");
        SYM(MemAddressFree, "cuMemAddressFree");
        SYM(MemRelease, "cuMemRelease");
#undef SYM
        a.ok = a.MemGetAllocationGranularity && a.MemCreate && a.MemExportToShareableHandle && a.MemImportFromShareableHandle &&
               a.MemAddressReserve && a.MemMap && a.MemSetAccess && a.MemUnmap && a.MemAddressFree && a.MemRelease;
    });
    return a;
}

struct Mapping { CUdeviceptr ptr; size_t size; CUmemGenericAllocationHandle handle; };
std::mutex g_mu;
std::vector<Mapping> g_maps;

CUmemAllocationProp props_for(int device) {
    CUmemAllocationProp p = {};
    p.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    p.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    p.location.id = device;
    p.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    return p;
}

bgs_status map_handle(int device, CUmemGenericAllocationHandle h, size_t size, size_t gran, void** out_ptr) {
    DrvApi& a = drv();
    CUdeviceptr ptr = 0;
    if (a.MemAddressReserve(&ptr, size, gran, 0, 0) != CUDA_SUCCESS) return BGS_ENOMEM;
    if (a.MemMap(ptr, size, 0, h, 0) != CUDA_SUCCESS) { a.MemAddressFree(ptr, size); return BGS_ECUDA; }
    CUmemAccessDesc acc = {};
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if (a.MemSetAccess(ptr, size, &acc, 1) != CUDA_SUCCESS) { a.MemUnmap(ptr, size); a.MemAddressFree(ptr, size); return BGS_ECUDA; }
    {
        std::lock_guard<std::mutex> lk(g_mu);
        g_maps.push_back({ptr, size, h});
    }
    *out_ptr = (void*)ptr;
    return BGS_OK;
}

}  // namespace

extern "C" {

bgs_status bgs_frame_export_create(int cuda_device, size_t bytes, void** out_device_ptr, int* out_fd, size_t* out_alloc_bytes) {
    if (!out_device_ptr || !out_fd || bytes == 0) return BGS_EINVAL;
    *out_device_ptr = nullptr; *out_fd = -1;
    DrvApi& a = drv();
    if (!a.ok) return BGS_ECUDA;
    if (cudaSetDevice(cuda_device) != cudaSuccess || cudaFree(nullptr) != cudaSuccess) return BGS_ECUDA;   // (primary context up)
    const CUmemAllocationProp p = props_for(cuda_device);
    size_t gran = 0;
    if (a.MemGetAllocationGranularity(&gran, &p, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS || gran == 0) return BGS_ECUDA;
    const size_t size = (bytes + gran - 1) / gran * gran;
    CUmemGenericAllocationHandle h = 0;
    if (a.MemCreate(&h, size, &p, 0) != CUDA_SUCCESS) return BGS_ENOMEM;
    int fd = -1;
    if (a.MemExportToShareableHandle(&fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0) != CUDA_SUCCESS) { a.MemRelease(h); return BGS_ECUDA; }
    const bgs_status st = map_handle(cuda_device, h, size, gran, out_device_ptr);
    if (st != BGS_OK) { close(fd); a.MemRelease(h); return st; }
    *out_fd = fd;
    if (out_alloc_bytes) *out_alloc_bytes = size;
    return BGS_OK;
}

bgs_status bgs_frame_export_import(int cuda_device, int fd, size_t alloc_bytes, void** out_device_ptr) {
    if (!out_device_ptr || fd < 0 || alloc_bytes == 0) return BGS_EINVAL;
    *out_device_ptr = nullptr;
    DrvApi& a = drv();
    if (!a.ok) return BGS_ECUDA;
    if (cudaSetDevice(cuda_device) != cudaSuccess || cudaFree(nullptr) != cudaSuccess) return BGS_ECUDA;
    const CUmemAllocationProp p = props_for(cuda_device);
    size_t gran = 0;
    if (a.MemGetAllocationGranularity(&gran, &p, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS || gran == 0) return BGS_ECUDA;
    CUmemGenericAllocationHandle h = 0;
    if (a.MemImportFromShareableHandle(&h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR) != CUDA_SUCCESS) return BGS_ECUDA;
    const bgs_status st = map_handle(cuda_device, h, alloc_bytes, gran, out_device_ptr);
    if (st != BGS_OK) a.MemRelease(h);
    return st;
}

void bgs_frame_export_destroy(void* device_ptr) {
    if (!device_ptr) return;
    DrvApi& a = drv();
    if (!a.ok) return;
    Mapping m = {0, 0, 0};
    {
        std::lock_guard<std::mutex> lk(g_mu);
        for (size_t i = 0; i < g_maps.size(); ++i)
            if ((void*)g_maps[i].ptr == device_ptr) { m = g_maps[i]; g_maps.erase(g_maps.begin() + i); break; }
    }
    if (!m.ptr) return;
    a.MemUnmap(m.ptr, m.size);
    a.MemAddressFree(m.ptr, m.size);
    a.MemRelease(m.handle);
}

}  // extern "C"
