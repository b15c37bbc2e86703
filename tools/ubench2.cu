// does a CTA-scope fence / block barrier wait for outstanding global loads and stores?  (H100, sm_90a)
#include <cstdio>
#include <cuda_runtime.h>
typedef unsigned long long u64; typedef unsigned int u32;
// mode bits: 1 = LDG in flight (consumed at the very end), 2 = STG issued just before, 4 = use BAR.SYNC instead of fence, 8 = neither fence nor barrier
__global__ void k(u32* out, long long* cyc, const u32* g, u32* gs, int mode, u32 salt) {
    __shared__ u32 s[256];
    u32 x = threadIdx.x;
    s[x] = x;
    __syncthreads();
    u32 v = 0;
    long long t0 = clock64();
    if (mode & 1) v = g[(x * 4099u + salt * 1000003u) & ((1u << 24) - 1)];
    if (mode & 2) gs[(x * 64 + salt * 977u) & ((1u << 22) - 1)] = x;
    s[(x + 1) & 255] = x + salt;
    if (mode & 4) __syncthreads();
    else if (!(mode & 8)) asm volatile("fence.acq_rel.cta;" ::: "memory");
    u32 y = s[(x + 2) & 255];
    long long t1 = clock64();
    // consume late
    out[threadIdx.x] = y + v;
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}
__global__ void k_clock(long long* cyc) { long long t0 = clock64(); long long t1 = clock64(); long long t2 = clock64(); if (threadIdx.x == 0) { cyc[0] = t1 - t0; cyc[1] = t2 - t1; } }
int main() {
    u32 *out, *g, *gs; long long* cyc;
    cudaMalloc(&out, 4096); cudaMalloc(&cyc, 16); cudaMalloc(&g, 64u << 20); cudaMalloc(&gs, 16u << 20);
    cudaMemset(g, 0, 64u << 20);
    const char* names[] = {"fence", "fence, LDG in flight", "fence, STG before", "fence, LDG+STG", "BAR", "BAR, LDG in flight", "BAR, STG before", "BAR, LDG+STG",
                           "none", "none, LDG in flight", "none, STG before", "none, LDG+STG"};
    for (int mode = 0; mode < 12; ++mode) {
        long long best = 1 << 30, sum = 0;
        for (int r = 0; r < 20; ++r) {
            k<<<1, 128>>>(out, cyc, g, gs, mode, r + 1);
            cudaDeviceSynchronize();
            long long h; cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
            if (r >= 2) { sum += h; if (h < best) best = h; }
        }
        printf("%-26s STS -> sync -> LDS: min %lld  mean %.0f cycles\n", names[mode], best, sum / 18.0);
    }
    k_clock<<<1, 32>>>(cyc); cudaDeviceSynchronize();
    long long h[2]; cudaMemcpy(h, cyc, 16, cudaMemcpyDeviceToHost);
    printf("back-to-back clock64: %lld %lld cycles\n", h[0], h[1]);
    return 0;
}
