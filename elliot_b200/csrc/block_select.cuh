// block_select.cuh — the block-wide top-k select of the kNN, EASE^R and RP3beta kernels.
//
// One CTA of NT threads holds n candidates, read through get(i, key) -> bool (false: i is not a candidate), and keeps the
// k with the largest keys, ties to the lowest index:
//   radix_threshold : the key T of the k-th best and how many candidates with key == T to take, by a radix select on
//                     BITS-bit digits from the top (the last digit narrower): u32 keys at 11 bits are 11 + 11 + 10,
//                     u64 keys at 8 bits are 8 x 8;
//   collect         : emit(slot, i, key) for the selected candidates, slots 0, 1, ... in index order;
//   sort_desc       : a bitonic sort of 64-bit keys, largest first;
//   write_topk      : the first k sorted pair keys out as (index, value).
// Ranking by (value desc, index asc) is ranking by pair_key desc: its high half is the order-preserving key of the value
// and its low half the complemented index, so every (value, index) has its own key.  Candidate keys must not be 0: the
// select uses T = 0 for "take every candidate" and sort_desc pads with 0.
#pragma once
#include <stdint.h>

namespace eb {

constexpr int SELECT_KMAX = 1024;            // largest k of the sorted selects (keys buffered in shared memory)

// order-preserving map of a float onto uint32 (larger value -> larger key) and back
__device__ __forceinline__ uint32_t fkey(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unfkey(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// (value desc, index asc) as one 64-bit key: larger key first
__device__ __forceinline__ uint64_t pair_key(float v, uint32_t i) { return ((uint64_t)fkey(v) << 32) | (0xffffffffu - i); }
__device__ __forceinline__ int32_t pair_index(uint64_t key) { return (int32_t)(0xffffffffu - (uint32_t)key); }
__device__ __forceinline__ float pair_value(uint64_t key) { return unfkey((uint32_t)(key >> 32)); }

template <int NT, int BITS>
struct SelectShared {
    uint32_t hist[1 << BITS];
    int warp_sum[NT / 32];
    int bin, above, total;
};

// exclusive prefix of x over the block in thread order; every thread gets the block total
template <int NT, int BITS>
__device__ __forceinline__ int block_excl_scan(int x, SelectShared<NT, BITS> &sh, int &total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int v = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += y;
    }
    if (lane == 31) sh.warp_sum[warp] = v;
    __syncthreads();
    int before_w = 0, t = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; w++) {
        const int s = sh.warp_sum[w];
        if (w < warp) before_w += s;
        t += s;
    }
    __syncthreads();
    total = t;
    return before_w + v - x;
}

// Histogram done: the bin (counted from the top) where the running count of candidates reaches `need`.  Sets sh.bin,
// sh.above (candidates in higher bins) and sh.total (all candidates in the histogram).  Thread t owns PER bins from the
// top down; with fewer bins than threads, the threads past the last bin own none.
template <int NT, int BITS>
__device__ __forceinline__ void find_bin(SelectShared<NT, BITS> &sh, int need) {
    constexpr int BINS = 1 << BITS, PER = BINS >= NT ? BINS / NT : 1;
    const bool owns = BINS >= NT || (int)threadIdx.x < BINS;
    const int top = BINS - 1 - PER * (int)threadIdx.x;                      // this thread's bins: top, top-1, ...
    int s = 0;
    if (owns) {
#pragma unroll
        for (int j = 0; j < PER; j++) s += (int)sh.hist[top - j];
    }
    int total;
    const int pre = block_excl_scan(s, sh, total);
    if (threadIdx.x == 0) sh.total = total;
    if (owns && pre < need && need <= pre + s) {
        int c = pre;
#pragma unroll
        for (int j = 0; j < PER; j++) {
            const int h = (int)sh.hist[top - j];
            if (c + h >= need) { sh.bin = top - j; sh.above = c; break; }
            c += h;
        }
    }
    __syncthreads();
}

// Key T of the k-th largest candidate key and the number of candidates with key == T to take (the first ones by index).
// At most k candidates: T = 0, need_eq = 0, every candidate is taken, and the first pass is the only one.
template <int NT, int BITS, class Key, class Get>
__device__ void radix_threshold(const Get &get, int n, int k, SelectShared<NT, BITS> &sh, Key &T, int &need_eq) {
    constexpr int KEY_BITS = 8 * sizeof(Key), PASSES = (KEY_BITS + BITS - 1) / BITS;
    Key prefix = 0, hi_mask = 0;
    int need = k;
    for (int pass = 0; pass < PASSES; pass++) {
        const int sft = KEY_BITS - BITS * (pass + 1) > 0 ? KEY_BITS - BITS * (pass + 1) : 0;
        const Key dmask = ((Key)1 << (KEY_BITS - BITS * pass - sft)) - 1;
        for (int b = threadIdx.x; b < (1 << BITS); b += NT) sh.hist[b] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += NT) {
            Key key;
            if (get(i, key) && (key & hi_mask) == prefix) atomicAdd(&sh.hist[(uint32_t)((key >> sft) & dmask)], 1u);
        }
        __syncthreads();
        find_bin(sh, need);
        if (pass == 0 && sh.total <= k) { prefix = 0; need = 0; break; }   // uniform
        prefix |= (Key)sh.bin << sft;
        hi_mask |= dmask << sft;
        need -= sh.above;
    }
    T = prefix;
    need_eq = need;
}

// Calls emit(slot, i, key) for the selected candidates (key > T, then the first need_eq with key == T) with slots
// 0, 1, ... in index order, and returns how many were selected.  One block scan per chunk of NT candidates counts both
// kinds at once: ties in the high 16 bits, keys above T in the low 16 (each count is at most NT <= 65 535).
template <int NT, int BITS, class Key, class Get, class Emit>
__device__ int collect(const Get &get, int n, Key T, int need_eq, SelectShared<NT, BITS> &sh, const Emit &emit) {
    static_assert(NT < 65536, "packed counts");
    int base = 0, eq_seen = 0;
    for (int i0 = 0; i0 < n; i0 += NT) {
        const int i = i0 + (int)threadIdx.x;
        Key key = 0;
        const bool c = i < n && get(i, key);
        const bool gt = c && key > T, eq = c && key == T;
        int total;
        const int pre = block_excl_scan((eq ? 0x10000 : 0) | (gt ? 1 : 0), sh, total);
        const int quota = max(0, need_eq - eq_seen);                         // ties still to take
        const int eq_before = pre >> 16;
        if (gt || (eq && eq_before < quota)) emit(base + (pre & 0xffff) + min(eq_before, quota), i, key);
        base += (total & 0xffff) + min(total >> 16, quota);
        eq_seen += total >> 16;
    }
    return base;
}

// bitonic sort of keys[0..m) into descending order; slots [m, pow2) are padded with 0, which sorts last
template <int NT>
__device__ void sort_desc(uint64_t *keys, int m) {
    int P = 1;
    while (P < m) P <<= 1;
    for (int i = m + (int)threadIdx.x; i < P; i += NT) keys[i] = 0;
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < P / 2; t += NT) {
                const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const uint64_t a = keys[lo], b = keys[hi];
                if ((b > a) == up) { keys[lo] = b; keys[hi] = a; }
            }
            __syncthreads();
        }
    }
}

// idx[j], val[j] for j < k from the sorted pair keys[0..m); the slots past m get -1 and `pad`
template <int NT>
__device__ void write_topk(const uint64_t *keys, int m, int k, int32_t *idx, float *val, float pad) {
    for (int j = threadIdx.x; j < k; j += NT) {
        idx[j] = j < m ? pair_index(keys[j]) : -1;
        val[j] = j < m ? pair_value(keys[j]) : pad;
    }
}

}  // namespace eb
