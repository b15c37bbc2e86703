// TEST INFRASTRUCTURE ONLY -- minimal stand-in for the CUDA runtime used by tests/hostsim.
//
// The product library (pyctcdecode_b200/csrc, built by nvcc for sm_90a) has NO CPU path.
// To be able to exercise the kernel *logic* (hashing, merge, LM fusion, selection, backtrack)
// in the CPU-only CI container, tests/hostsim compiles the very same sources with g++ and
// -DB2C_HOSTSIM: kernel bodies run block by block on the host (see csrc/b2c_cta.h) and the
// handful of runtime calls below become malloc/memcpy.  Nothing under pyctcdecode_b200/
// loads this build; it exists for `pytest -m "not gpu"` only.
#pragma once
#include <cstdlib>
#include <cstring>

typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaDevAttrMultiProcessorCount = 16, cudaDevAttrMaxSharedMemoryPerBlockOptin = 97 };

inline const char* cudaGetErrorString(cudaError_t) { return "hostsim"; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaMalloc(void** p, size_t n) { *p = std::malloc(n ? n : 1); return *p ? cudaSuccess : 2; }
inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMallocHost(void** p, size_t n) { *p = std::malloc(n ? n : 1); return *p ? cudaSuccess : 2; }
inline cudaError_t cudaFreeHost(void* p) { std::free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { std::memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { std::memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dp, const void* s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t) {
    for (size_t r = 0; r < h; ++r) std::memcpy(static_cast<char*>(d) + r * dp, static_cast<const char*>(s) + r * sp, w);
    return cudaSuccess;
}
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) { std::memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = nullptr; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = nullptr; return cudaSuccess; }
enum { cudaEventDisableTiming = 2 };
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = nullptr; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, int attr, int) {
    *v = (attr == cudaDevAttrMultiProcessorCount) ? 4 : 227 * 1024;
    return cudaSuccess;
}
