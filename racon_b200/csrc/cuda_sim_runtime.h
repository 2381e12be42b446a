/*
 * cuda_sim_runtime.h — TEST INFRASTRUCTURE ONLY.  A host stand-in for the handful of CUDA runtime calls rp_api.cu makes,
 * used when rp_api.cu is compiled with g++ -DRP_HOST_SIM=1 into racon_b200/lib/simapi/libracon_b200.so (build.py:
 * build_simapi).  "Device" memory is host memory, streams run synchronously, and a kernel launch runs the very same
 * device functions (poa_core.cuh, myers_core.cuh) as cooperative fibres (rp_warp.cuh), one window / overlap after the
 * other.  With it the whole C ABI — batch limits, escalation pass, band policy, read-back, the C++ host layer above it —
 * runs on a machine without a GPU, so that the tests marked `gpu` can be pre-verified here (RP_TEST_SIMAPI=1, see
 * tests/conftest.py).  Nothing in the product library includes this file: the product build sees <cuda_runtime.h>.
 */
#pragma once
#if !defined(RP_HOST_SIM)
#error "cuda_sim_runtime.h is for the host simulation build only"
#endif
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorNoDevice = 100, cudaErrorNotReady = 600 };
typedef struct rp_sim_stream* cudaStream_t;
enum { cudaStreamNonBlocking = 1, cudaHostAllocDefault = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };

struct cudaDeviceProp {
    char name[64];
    int multiProcessorCount;
    size_t sharedMemPerMultiprocessor, sharedMemPerBlockOptin, totalGlobalMem;
};

/* RP_SIM_DEVICES=0 plays a machine without a GPU */
inline int rp_sim_device_count() {
    const char* e = std::getenv("RP_SIM_DEVICES");
    return e ? std::atoi(e) : 1;
}
inline cudaError_t cudaGetDeviceCount(int* n) {
    *n = rp_sim_device_count();
    return *n > 0 ? cudaSuccess : cudaErrorNoDevice;
}
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
    std::memset(p, 0, sizeof(*p));
    std::strcpy(p->name, "host simulation");
    const char* e = std::getenv("RP_SIM_SMS");
    p->multiProcessorCount = e ? std::atoi(e) : 2;        // a small "GPU": a handful of workers, several waves per batch
    p->sharedMemPerMultiprocessor = 233472;                // sm_90: 228 KB
    p->sharedMemPerBlockOptin = 232448;                    // 227 KB
    p->totalGlobalMem = size_t(8) << 30;
    return cudaSuccess;
}
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int device) {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, device);
    *v = p.multiProcessorCount;
    return cudaSuccess;
}
inline cudaError_t cudaMemGetInfo(size_t* free_b, size_t* total_b) {
    const char* e = std::getenv("RP_SIM_FREE_MB");
    *total_b = size_t(8) << 30;
    *free_b = e ? size_t(std::atoll(e)) << 20 : size_t(4) << 30;
    return cudaSuccess;
}
inline const char* cudaGetErrorString(cudaError_t e) {
    return e == cudaSuccess ? "no error" : e == cudaErrorMemoryAllocation ? "out of memory" : "simulated CUDA error";
}
inline cudaError_t cudaGetLastError() { return cudaSuccess; }

inline cudaError_t cudaMalloc(void** p, size_t n) {
    *p = nullptr;
    if (posix_memalign(p, 256, n ? n : 1) != 0) return cudaErrorMemoryAllocation;
    std::memset(*p, 0xa5, n);   // uninitialised device memory is not zero
    return cudaSuccess;
}
template <typename T>
inline cudaError_t cudaMalloc(T** p, size_t n) {
    return cudaMalloc(reinterpret_cast<void**>(p), n);
}
inline cudaError_t cudaFree(void* p) {
    std::free(p);
    return cudaSuccess;
}
inline cudaError_t cudaHostAlloc(void** p, size_t n, unsigned) {
    *p = std::malloc(n ? n : 1);
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
inline cudaError_t cudaFreeHost(void* p) {
    std::free(p);
    return cudaSuccess;
}
inline cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t n, cudaMemcpyKind, cudaStream_t) {
    if (n) std::memmove(dst, src, n);
    return cudaSuccess;
}
inline cudaError_t cudaMemsetAsync(void* dst, int v, size_t n, cudaStream_t) {
    if (n) std::memset(dst, v, n);
    return cudaSuccess;
}
inline cudaError_t cudaStreamCreate(cudaStream_t* s) {
    *s = reinterpret_cast<cudaStream_t>(std::malloc(8));
    return cudaSuccess;
}
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { return cudaStreamCreate(s); }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) {
    std::free(s);
    return cudaSuccess;
}
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamQuery(cudaStream_t) { return cudaSuccess; }   // the work of a stream is done when queued
template <typename F>
inline cudaError_t cudaFuncSetAttribute(F, int, int) {
    return cudaSuccess;
}
template <typename F>
inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) {
    *n = 8;
    return cudaSuccess;
}
