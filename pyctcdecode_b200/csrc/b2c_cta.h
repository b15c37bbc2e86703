// b200ctc -- the tiny execution-model layer the kernel bodies are written against.
//
// Kernel bodies are written as a sequence of phases separated by block barriers:
//
//     B2C_FOR(i, n) { ... work item i ... }      // items strided over the CTA's threads
//     B2C_SYNC();
//     B2C_LEADER { ... one thread ... }
//
// Compiled by nvcc for sm_90a these are the obvious CUDA constructs.  Compiled by g++ with
// B2C_HOSTSIM (tests/hostsim only -- NOT a product fallback, the product library contains no
// CPU path) a phase is a plain loop over all items and a barrier is a no-op, i.e. one legal
// interleaving of the CUDA execution.  Code outside B2C_FOR / B2C_LEADER between barriers
// must be block-uniform (it reads only kernel arguments and shared scalars).
#pragma once
#include "b2c_common.h"
#if !defined(__CUDACC__)
#include <cstdlib>
#endif

#if defined(__CUDACC__)
#define B2C_NOINLINE __noinline__
#else
#define B2C_NOINLINE __attribute__((noinline))
#endif

#if defined(__CUDA_ARCH__)
#define B2C_FOR(i, n) for (int i = static_cast<int>(threadIdx.x); i < static_cast<int>(n); i += static_cast<int>(blockDim.x))
#define B2C_SYNC() __syncthreads()
#define B2C_LEADER if (threadIdx.x == 0)
#define B2C_FOR_WARP(w, nw) for (int w = static_cast<int>(threadIdx.x >> 5), _once = 1; _once; _once = 0)
#define B2C_NWARPS() (static_cast<int>(blockDim.x >> 5))
#else
// hostsim runs the work items of a phase one after another.  Any order is a legal interleaving of the CUDA
// execution, so the results must not depend on it: B200CTC_HOSTSIM_ORDER=1 (reverse) / 2 (stride 7) / 3 (odd items
// first) make tests/ replay every phase in another order -- a cheap detector for missing barriers and for code that
// silently relies on thread order.
inline int b2c_hostsim_order() {
    static const int mode = [] { const char* e = std::getenv("B200CTC_HOSTSIM_ORDER"); return e ? std::atoi(e) : 0; }();
    return mode;
}
inline int b2c_hostsim_item(int k, int n) {
    switch (b2c_hostsim_order()) {
        case 1: return n - 1 - k;
        case 2: return n % 7 == 0 ? (n - 1 - k) : static_cast<int>((static_cast<long long>(k) * 7) % n);   // bijection iff gcd(7, n) == 1
        case 3: { const int odd = n / 2; return k < odd ? 2 * k + 1 : 2 * (k - odd); }
        default: return k;
    }
}
#define B2C_FOR(i, n) for (int _k##i = 0, _n##i = static_cast<int>(n), i = 0; _k##i < _n##i && ((i = b2c_hostsim_item(_k##i, _n##i)), true); ++_k##i)
#define B2C_SYNC() ((void)0)
#define B2C_LEADER if (true)
#define B2C_FOR_WARP(w, nw) for (int w = 0; w < static_cast<int>(nw); ++w)
#define B2C_NWARPS() (8)
#endif

// block-scope atomics on shared or global memory
B2C_HD u32 b2c_atomic_cas_u32(u32* p, u32 cmp, u32 val) {
#if defined(__CUDA_ARCH__)
    return atomicCAS(p, cmp, val);
#else
    u32 old = *p;
    if (old == cmp) *p = val;
    return old;
#endif
}
B2C_HD u32 b2c_atomic_add_u32(u32* p, u32 v) {
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, v);
#else
    u32 old = *p;
    *p = old + v;
    return old;
#endif
}
// one item from a bump counter per calling thread: the threads of a warp that arrive together share ONE atomic
// (hundreds of beams allocating a backtrack node each would otherwise serialise on one shared-memory word)
B2C_HD u32 b2c_alloc_one(u32* counter) {
#if defined(__CUDA_ARCH__)
    const unsigned m = __activemask();
    const unsigned lane = threadIdx.x & 31u;
    const int first = __ffs(static_cast<int>(m)) - 1;
    u32 base = 0;
    if (static_cast<int>(lane) == first) base = atomicAdd(counter, static_cast<u32>(__popc(m)));
    base = __shfl_sync(m, base, first);
    return base + static_cast<u32>(__popc(m & ((1u << lane) - 1u)));
#else
    return b2c_atomic_add_u32(counter, 1u);
#endif
}
B2C_HD void b2c_atomic_min_u32(u32* p, u32 v) {
#if defined(__CUDA_ARCH__)
    atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
B2C_HD void b2c_atomic_max_u32(u32* p, u32 v) {
#if defined(__CUDA_ARCH__)
    atomicMax(p, v);
#else
    if (v > *p) *p = v;
#endif
}
B2C_HD void b2c_atomic_max_u64(u64* p, u64 v) {
#if defined(__CUDA_ARCH__)
    atomicMax(p, v);
#else
    if (v > *p) *p = v;
#endif
}
B2C_HD void b2c_atomic_or_u32(u32* p, u32 v) {
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}

// _sum_log_scores (reference decoder.py:170-177), float64, symmetric in its arguments
B2C_HD double b2c_sum_log_scores(double s1, double s2) {
    if (s1 >= s2) return s1 + log(1 + exp(s2 - s1));
    return s2 + log(1 + exp(s1 - s2));
}
