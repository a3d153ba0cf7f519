// device_memory_emul.h -- device memory as the CPU checker (tests/emul) tells it from host memory. TEST INFRASTRUCTURE.
//
// cuda_shim.h reports every pointer as page-locked, mapped host memory, which is what the scan_attach_host tests rely on. The
// device-pointer entry points (liinit_*_device) must tell device memory from host memory, so liinit_gpu.cu includes this header after
// the shim when it is compiled for the CPU (LI_SIMT_EMUL): it keeps a registry of the live cudaMalloc ranges, and
// cudaPointerGetAttributes reports cudaMemoryTypeDevice (device 0) inside them and defers to the shim everywhere else. cudaMallocHost /
// cudaHostAlloc memory and any other host buffer therefore stay "page-locked and mapped" as before.
#pragma once
#include <cstddef>
#include <map>
#include <mutex>

struct LiEmulDeviceRanges {
    std::mutex mu;
    std::map<const char*, size_t> r;   // start -> size of every live cudaMalloc allocation
};
inline LiEmulDeviceRanges& li_emul_device_ranges() {
    static LiEmulDeviceRanges R;
    return R;
}
inline bool li_emul_is_device(const void* p) {
    LiEmulDeviceRanges& R = li_emul_device_ranges();
    std::lock_guard<std::mutex> g(R.mu);
    const char* q = static_cast<const char*>(p);
    auto it = R.r.upper_bound(q);
    if (it == R.r.begin()) return false;
    --it;
    return q < it->first + it->second;
}

template <class T>
inline cudaError_t li_emul_cudaMalloc(T** p, size_t n) {
    const cudaError_t e = cudaMalloc(p, n);
    if (e == cudaSuccess) {
        LiEmulDeviceRanges& R = li_emul_device_ranges();
        std::lock_guard<std::mutex> g(R.mu);
        R.r[reinterpret_cast<const char*>(*p)] = n ? n : 1;
    }
    return e;
}
inline cudaError_t li_emul_cudaFree(void* p) {
    if (p) {
        LiEmulDeviceRanges& R = li_emul_device_ranges();
        std::lock_guard<std::mutex> g(R.mu);
        R.r.erase(static_cast<const char*>(p));
    }
    return cudaFree(p);
}

// the runtime's attribute struct has the device ordinal, the shim's does not
struct li_emul_PointerAttributes {
    cudaMemoryType type;
    int device;
    void* devicePointer;
    void* hostPointer;
};
inline cudaError_t li_emul_cudaPointerGetAttributes(li_emul_PointerAttributes* a, const void* p) {
    a->device = 0;
    if (li_emul_is_device(p)) {
        a->type = cudaMemoryTypeDevice;
        a->devicePointer = const_cast<void*>(p);
        a->hostPointer = nullptr;
        return cudaSuccess;
    }
    cudaPointerAttributes s;
    const cudaError_t e = cudaPointerGetAttributes(&s, p);
    a->type = s.type;
    a->devicePointer = s.devicePointer;
    a->hostPointer = s.hostPointer;
    return e;
}

#define cudaMalloc li_emul_cudaMalloc
#define cudaFree li_emul_cudaFree
#define cudaPointerAttributes li_emul_PointerAttributes
#define cudaPointerGetAttributes li_emul_cudaPointerGetAttributes
#define cudaMemoryTypeManaged (static_cast<cudaMemoryType>(3))

// For the tests: emulated device memory that the device-pointer entry points accept.
extern "C" void* liinit_emul_device_alloc(size_t bytes) {
    void* p = nullptr;
    return cudaMalloc(&p, bytes) == cudaSuccess ? p : nullptr;
}
extern "C" void liinit_emul_device_free(void* p) { cudaFree(p); }
