// common.cuh — shared helpers for the sm_90a kernels behind include/elliot_b200.h
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/elliot_b200.h"

namespace eb {

extern thread_local char g_err[512];
int set_err(int code, const char *fmt, ...);

#define EB_CUDA(call)                                                                              \
    do {                                                                                           \
        cudaError_t _e = (call);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return eb::set_err(EB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call,           \
                               cudaGetErrorString(_e));                                            \
    } while (0)

#define EB_ARG(cond, ...)                                                                          \
    do {                                                                                           \
        if (!(cond)) return eb::set_err(EB_ERR_ARG, __VA_ARGS__);                                  \
    } while (0)

int sm_count();

// Philox4x32-10 (Salmon et al. 2011).  key = seed, counter = (triple index, attempt).
struct Philox {
    static constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    __host__ __device__ static inline void round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#ifdef __CUDA_ARCH__
        uint32_t hi0 = __umulhi(M0, c[0]), hi1 = __umulhi(M1, c[2]);
#else
        uint32_t hi0 = (uint32_t)(((uint64_t)M0 * c[0]) >> 32), hi1 = (uint32_t)(((uint64_t)M1 * c[2]) >> 32);
#endif
        uint32_t lo0 = M0 * c[0], lo1 = M1 * c[2];
        uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
        c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    }
    __host__ __device__ static inline void gen(uint64_t seed, uint64_t ctr, uint32_t attempt, uint32_t (&out)[4]) {
        uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
        out[0] = (uint32_t)ctr; out[1] = (uint32_t)(ctr >> 32); out[2] = attempt; out[3] = 0x454c4c49u;
#pragma unroll
        for (int r = 0; r < 10; r++) {
            round(out, k0, k1);
            k0 += W0; k1 += W1;
        }
    }
};

// uniform integer in [0, n) from a 32-bit word (multiply-high; bias < n / 2^32)
__host__ __device__ static inline uint32_t bounded(uint32_t r, uint32_t n) {
#ifdef __CUDA_ARCH__
    return __umulhi(r, n);
#else
    return (uint32_t)(((uint64_t)r * n) >> 32);
#endif
}

// binary search for `key` in sorted a[0..len)
__device__ static inline bool contains_sorted(const int32_t *__restrict__ a, int len, int32_t key) {
    int lo = 0, hi = len;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        int32_t v = __ldg(a + mid);
        if (v < key) lo = mid + 1; else hi = mid;
    }
    return lo < len && __ldg(a + lo) == key;
}

// Per-user membership signature (a Bloom filter of 32*words bits, 2 hashes) over the user's train items: the sampler's
// rejection test `j in ui` (custom_sampler.py:40-41) is a MISS for all but ~len/n_items of the candidates, and a miss is
// proven by one or two word loads here instead of a dependent binary search over the CSR row.  words is a power of two.
__host__ __device__ static inline void bloom_bits(uint32_t x, int log2bits, uint32_t &a, uint32_t &b) {
    a = (x * 0x9E3779B1u) >> (32 - log2bits);
    b = ((x ^ 0x5bd1e995u) * 0x85EBCA6Bu) >> (32 - log2bits);
}
__device__ static inline bool bloom_maybe(const uint32_t *__restrict__ f, int log2bits, uint32_t x) {
    uint32_t a, b;
    bloom_bits(x, log2bits, a, b);
    return ((__ldg(f + (a >> 5)) >> (a & 31)) & (__ldg(f + (b >> 5)) >> (b & 31)) & 1u) != 0;
}
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// 128-bit / 32-bit fire-and-forget float adds (vector / scalar RED instructions)
__device__ __forceinline__ void red_add_v4(float *p, float4 v) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void red_add_f32(float *p, float v) {
    asm volatile("red.relaxed.gpu.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
// the same with system scope, for rows that may live in a PEER GPU's memory (NVLink atomics; REDG...STRONG.SYS)
__device__ __forceinline__ void red_add_v4_sys(float *p, float4 v) {
    asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void red_add_f32_sys(float *p, float v) {
    asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
// 128-bit load that must observe other GPUs' writes (no stale L1 line): LDG.E.128.STRONG.SYS
__device__ __forceinline__ float4 ld_sys_v4(const float4 *p) {
    float4 r;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
    return r;
}
}  // namespace eb
