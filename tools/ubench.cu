// micro-benchmarks of the instruction latencies the beam kernel's critical path is made of (H100, sm_90a)
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench tools/ubench.cu ; run: tools/ubench
#include <cstdio>
#include <cuda_runtime.h>
typedef unsigned long long u64; typedef unsigned int u32;
#define N 256
__global__ void k_dadd(double* out, double a, double b, long long* cyc) {
    double x = a; long long t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = x + b;
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_dfma(double* out, double a, double b, long long* cyc) {
    double x = a; long long t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = fma(x, b, a);
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_dsetp(double* out, double a, double b, long long* cyc) {
    double x = a; long long t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = (x > b) ? x + 1.0 : x - 1.0;   // DSETP + select + DADD
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_fadd(float* out, float a, float b, long long* cyc) {
    float x = a; long long t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = x + b;
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_imad64(u64* out, u64 a, u64 b, long long* cyc) {
    u64 x = a; long long t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = x * b + a;
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_lds(u32* out, long long* cyc) {
    __shared__ u32 s[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) s[i] = (i * 7 + 1) & 1023;
    __syncthreads();
    u32 x = threadIdx.x; long long t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = s[x];
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_lds64(u64* out, long long* cyc) {
    __shared__ u64 s[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) s[i] = (i * 7 + 1) & 1023;
    __syncthreads();
    u64 x = threadIdx.x; long long t0 = clock64();
#pragma unroll
    for (int i = 0; i < N; ++i) x = s[x];
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_atoms(u32* out, long long* cyc, int spread) {
    __shared__ u32 s[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) s[i] = 0;
    __syncthreads();
    u32 x = 0; long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) x += atomicAdd(&s[spread ? ((threadIdx.x + x) & 1023) : (x & 7)], 1u + (x & 1));
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_cas(u32* out, long long* cyc) {
    __shared__ u32 s[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) s[i] = 0xFFFFFFFFu;
    __syncthreads();
    u32 x = threadIdx.x; long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) x = (x + atomicCAS(&s[(x * 33 + i) & 1023], 0xFFFFFFFFu, x)) ;
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_bar(u32* out, long long* cyc) {
    u32 x = threadIdx.x; long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) { __syncthreads(); x += i; }
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_fence(u32* out, long long* cyc, const u32* g, int with_load) {
    __shared__ u32 s[1024];
    u32 x = threadIdx.x, acc = 0; long long t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < N; ++i) {
        u32 v = 0;
        if (with_load) v = g[(x * 4099u + i * 1000003u) & ((1u << 24) - 1)];   // L2/DRAM miss, NOT consumed before the fence
        s[(x + i) & 1023] = x;
        asm volatile("fence.acq_rel.cta;" ::: "memory");
        x += s[(x + i + 1) & 1023] & 1;
        acc += v;
    }
    long long t1 = clock64(); out[threadIdx.x] = x + acc; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_barload(u32* out, long long* cyc, const u32* g, int with_load) {
    u32 x = threadIdx.x, acc = 0; long long t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < N; ++i) {
        u32 v = 0;
        if (with_load) v = g[(x * 4099u + i * 1000003u) & ((1u << 24) - 1)];
        __syncthreads();
        x += i & 1;
        acc += v;        // consumed after the barrier; the sum is only needed at the very end
    }
    long long t1 = clock64(); out[threadIdx.x] = x + acc; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_ldg(u32* out, long long* cyc, const u32* g, u32 mask) {
    u32 x = threadIdx.x * 64; long long t0 = clock64();
#pragma unroll 4
    for (int i = 0; i < N; ++i) x = g[x & mask];
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_exp(double* out, double a, long long* cyc) {
    double x = a; long long t0 = clock64();
    for (int i = 0; i < 64; ++i) x = exp(x) - 1.0;
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_log(double* out, double a, long long* cyc) {
    double x = a; long long t0 = clock64();
    for (int i = 0; i < 64; ++i) x = log(x) + 3.0;
    long long t1 = clock64(); out[threadIdx.x] = x; if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
int main() {
    void* out; long long* cyc; u32* g;
    cudaMalloc(&out, 8 * 1024); cudaMalloc(&cyc, 8); cudaMalloc(&g, 64u << 20);
    // pointer-chase table: g[i] = random-ish next index
    { u32* h = new u32[16u << 20]; for (u32 i = 0; i < (16u << 20); ++i) h[i] = (i * 2654435761u + 12345u) & ((16u << 20) - 1); cudaMemcpy(g, h, 64u << 20, cudaMemcpyHostToDevice); delete[] h; }
    long long h;
#define RUN(name, threads, per, ...) do { for (int r = 0; r < 3; ++r) { __VA_ARGS__; cudaDeviceSynchronize(); } cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost); printf("%-34s threads=%4d  %.1f cycles/op\n", name, threads, double(h) / (per)); } while (0)
    for (int th : {32, 128}) {
        RUN("DADD dependent", th, N, (k_dadd<<<1, th>>>((double*)out, 1.0, 1e-3, cyc)));
        RUN("DFMA dependent", th, N, (k_dfma<<<1, th>>>((double*)out, 1.0, 0.999, cyc)));
        RUN("DSETP+SEL+DADD dependent", th, N, (k_dsetp<<<1, th>>>((double*)out, 1.0, 0.5, cyc)));
        RUN("FADD dependent", th, N, (k_fadd<<<1, th>>>((float*)out, 1.0f, 1e-3f, cyc)));
        RUN("IMAD64 (x*b+a) dependent", th, N, (k_imad64<<<1, th>>>((u64*)out, 3, 5, cyc)));
        RUN("LDS.32 dependent", th, N, (k_lds<<<1, th>>>((u32*)out, cyc)));
        RUN("LDS.64 dependent", th, N, (k_lds64<<<1, th>>>((u64*)out, cyc)));
        RUN("ATOMS.ADD few addresses", th, N, (k_atoms<<<1, th>>>((u32*)out, cyc, 0)));
        RUN("ATOMS.ADD spread addresses", th, N, (k_atoms<<<1, th>>>((u32*)out, cyc, 1)));
        RUN("ATOMS.CAS spread", th, N, (k_cas<<<1, th>>>((u32*)out, cyc)));
        RUN("BAR.SYNC", th, N, (k_bar<<<1, th>>>((u32*)out, cyc)));
        RUN("STS+fence.cta+LDS", th, N, (k_fence<<<1, th>>>((u32*)out, cyc, g, 0)));
        RUN("STS+fence.cta+LDS, LDG in flight", th, N, (k_fence<<<1, th>>>((u32*)out, cyc, g, 1)));
        RUN("BAR.SYNC, no load", th, N, (k_barload<<<1, th>>>((u32*)out, cyc, g, 0)));
        RUN("BAR.SYNC, LDG in flight", th, N, (k_barload<<<1, th>>>((u32*)out, cyc, g, 1)));
        RUN("exp(double) dependent", th, 64, (k_exp<<<1, th>>>((double*)out, 0.5, cyc)));
        RUN("log(double) dependent", th, 64, (k_log<<<1, th>>>((double*)out, 5.0, cyc)));
    }
    RUN("LDG chase, 4 KB footprint (L1)", 32, N, (k_ldg<<<1, 32>>>((u32*)out, cyc, g, 1023)));
    RUN("LDG chase, 4 MB footprint (L2)", 32, N, (k_ldg<<<1, 32>>>((u32*)out, cyc, g, (1u << 20) - 1)));
    RUN("LDG chase, 64 MB footprint", 32, N, (k_ldg<<<1, 32>>>((u32*)out, cyc, g, (16u << 20) - 1)));
    return 0;
}
