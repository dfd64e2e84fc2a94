// slope_one.cu — SlopeOne (algebric/slope_one/slope_one_model.py:19-64) on the GPU, its fp64 scores reproduced bit for bit.
//   slope_one_dev_kernel   : E[i][j] = ((double)(M1 - M2)[i][j] * 2^-s) / F[i][j] for a row slab of the exact fp32
//                            products F = B^T B, M1 = X^T B, M2 = B^T X (X: ratings * 2^s, B: the entry pattern), NaN where
//                            F = 0.  D = (M1 - M2) 2^-s is the reference's exact sum of r_ui - r_uj, so E[i][j] is its
//                            dev[i][j] for i < j and -dev[j][i] for i > j, rounded once;
//   slope_one_score_kernel : one CTA per user: its mean (an exact fp64 sum of its ratings, one division), then for every
//                            candidate c of a column tile sum_j -E[j][c] over the user's train items j in the given order
//                            (plain sequential __dadd_rn, NaN terms skipped and counted out), one __ddiv_rn by the count
//                            and the mean added: the reference's `mean + sum(dev[c, j] for j in Ri) / len(Ri)`.  Train items
//                            are excluded; the k best by (score desc, item asc) come from block_select.cuh on 64-bit
//                            order-preserving keys of the fp64 scores, and a bitonic sort of (key, item) pairs.
// Reading row j of E at the tile's columns keeps every warp's loads coalesced.
#include <math_constants.h>

#include "block_select.cuh"
#include "common.cuh"

namespace eb {

constexpr int SO_NT = 256;                   // threads per CTA of the scorer
constexpr int SO_COLS = 4;                   // candidate columns per thread in flight
constexpr int SO_BITS = 8;                   // radix digit: 8 x 8 bits of the 64-bit keys
constexpr int SO_TILE = 4096;                // fp64 score keys per column tile (32 KB of shared memory: 4 CTAs per SM)

using SoSel = SelectShared<SO_NT, SO_BITS>;

// order-preserving map of a double onto uint64 (larger value -> larger key); 0 only for one NaN pattern, which no score has
__device__ __forceinline__ uint64_t dkey(double v) {
    const uint64_t u = (uint64_t)__double_as_longlong(v);
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double undkey(uint64_t k) {
    return __longlong_as_double((long long)((k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k));
}

// ---------------------------------------------------------------- deviations
__global__ void slope_one_dev_kernel(const float *__restrict__ F, const float *__restrict__ M1, const float *__restrict__ M2,
                                     int64_t ld_in, int32_t n_rows, int32_t n, double unscale, double *__restrict__ E,
                                     int64_t lde) {
    const int64_t total = (int64_t)n_rows * n;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / n, c = t - r * n;
        const int64_t a = r * ld_in + c;
        const float f = F[a];
        // every product is an fp32 integer below 2^24, so the difference and the scaling are exact in fp64
        E[r * lde + c] = f == 0.f ? CUDART_NAN : __ddiv_rn(((double)M1[a] - (double)M2[a]) * unscale, (double)f);
    }
}

// ---------------------------------------------------------------- scores and top-k
struct SlopeOneParams {
    const double *E;
    int64_t lde;
    int32_t n_items;
    const int64_t *indptr; const int32_t *items; const float *ratings;      // train items per user in the summation order
    const int64_t *mask_indptr; const int32_t *mask_indices;               // excluded items per user (any order)
    const int32_t *users;
    int32_t user_begin;
    int64_t n_sel;
    int k, tile, kbuf;          // kbuf: a power of two >= 2k, the length of the pair buffers
    int32_t *out_idx;
    double *out_val;
};

// (key desc, item asc) as the order of pairs: a ranks before b
__device__ __forceinline__ bool pair_before(uint64_t ka, uint32_t ia, uint64_t kb, uint32_t ib) {
    return ka > kb || (ka == kb && ia < ib);
}

// bitonic sort of (keys, idx)[0..m) into rank order; slots [m, pow2) are padded with (0, UINT32_MAX), which rank last
__device__ __forceinline__ void sort_pairs(uint64_t *keys, uint32_t *idx, int m) {
    int P = 1;
    while (P < m) P <<= 1;
    for (int i = m + (int)threadIdx.x; i < P; i += SO_NT) { keys[i] = 0; idx[i] = 0xffffffffu; }
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < P / 2; t += SO_NT) {
                const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const uint64_t ka = keys[lo], kb = keys[hi];
                const uint32_t ia = idx[lo], ib = idx[hi];
                if (pair_before(kb, ib, ka, ia) == up) { keys[lo] = kb; keys[hi] = ka; idx[lo] = ib; idx[hi] = ia; }
            }
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(SO_NT, 4) slope_one_score_kernel(const SlopeOneParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t *sk = reinterpret_cast<uint64_t *>(smem_raw);                  // [tile] score keys, 0 = not a candidate
    uint64_t *bk = sk + p.tile;                                              // [kbuf] best keys so far + this tile's
    uint32_t *bi = reinterpret_cast<uint32_t *>(bk + p.kbuf);                // [kbuf] their items
    __shared__ SoSel sh;
    __shared__ double mean_sh;
    const int lane = threadIdx.x & 31;
    for (int64_t q = blockIdx.x; q < p.n_sel; q += gridDim.x) {
        const int u = p.users ? p.users[q] : p.user_begin + (int)q;
        const int64_t a0 = p.indptr[u], a1 = p.indptr[u + 1];
        if (threadIdx.x < 32) {
            // ratings * 2^s are integers, so the fp64 sum is exact in any order (np.mean's pairwise sum gives the same)
            double s = 0.0;
            for (int64_t e = a0 + lane; e < a1; e += 32) s += (double)__ldg(p.ratings + e);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) mean_sh = __ddiv_rn(s, (double)(a1 - a0));
        }
        __syncthreads();
        const double mean = mean_sh;
        int cur = 0;
        for (int c0 = 0; c0 < p.n_items; c0 += p.tile) {
            const int tn = min(p.tile, p.n_items - c0);
            for (int i0 = threadIdx.x; i0 < tn; i0 += SO_NT * SO_COLS) {
                double s[SO_COLS];
                int cnt[SO_COLS];
#pragma unroll
                for (int r = 0; r < SO_COLS; r++) { s[r] = 0.0; cnt[r] = 0; }
                for (int64_t e = a0; e < a1; e++) {
                    const double *row = p.E + (int64_t)__ldg(p.items + e) * p.lde + c0;
#pragma unroll
                    for (int r = 0; r < SO_COLS; r++) {
                        const int i = i0 + r * SO_NT;
                        if (i < tn) {
                            const double x = __ldg(row + i);
                            if (x == x) { s[r] = __dadd_rn(s[r], -x); cnt[r]++; }
                        }
                    }
                }
#pragma unroll
                for (int r = 0; r < SO_COLS; r++) {
                    const int i = i0 + r * SO_NT;
                    if (i < tn) sk[i] = dkey(cnt[r] ? __dadd_rn(mean, __ddiv_rn(s[r], (double)cnt[r])) : mean);
                }
            }
            __syncthreads();
            if (p.mask_indptr) {
                const int64_t m0 = p.mask_indptr[u], m1 = p.mask_indptr[u + 1];
                for (int64_t m = m0 + threadIdx.x; m < m1; m += SO_NT) {
                    const int c = __ldg(p.mask_indices + m) - c0;
                    if (c >= 0 && c < tn) sk[c] = 0;
                }
            }
            __syncthreads();
            auto get = [sk](int i, uint64_t &key) {
                key = sk[i];
                return key != 0;
            };
            uint64_t T;
            int need_eq;
            radix_threshold(get, tn, p.k, sh, T, need_eq);
            const int m = collect(get, tn, T, need_eq, sh, [bk, bi, cur, c0](int slot, int i, uint64_t key) {
                bk[cur + slot] = key;
                bi[cur + slot] = (uint32_t)(i + c0);
            });
            sort_pairs(bk, bi, cur + m);
            cur = min(cur + m, p.k);
        }
        for (int j = threadIdx.x; j < p.k; j += SO_NT) {
            p.out_idx[q * p.k + j] = j < cur ? (int32_t)bi[j] : -1;
            p.out_val[q * p.k + j] = j < cur ? undkey(bk[j]) : -CUDART_INF;
        }
        __syncthreads();
    }
}

static int so_tile(int32_t n_items) {
    const int t = (n_items + 255) / 256 * 256;
    return t < SO_TILE ? t : SO_TILE;
}

static int so_kbuf(int k) {
    int b = 2;
    while (b < 2 * k) b <<= 1;
    return b;
}

}  // namespace eb

using namespace eb;

extern "C" int eb_slope_one_dev_f64(const float *F, const float *M1, const float *M2, int64_t ld_in, int32_t n_rows, int32_t n,
                                    int s, double *E, int64_t lde, void *stream) {
    EB_ARG(F && M1 && M2 && E, "null pointer");
    EB_ARG(n >= 1 && n_rows >= 0 && ld_in >= n && lde >= n, "bad shape n=%d n_rows=%d ld_in=%lld lde=%lld", n, n_rows,
           (long long)ld_in, (long long)lde);
    EB_ARG(s >= 0 && s <= 30, "s=%d outside [0, 30]", s);
    if (n_rows == 0) return EB_OK;
    int64_t grid = ((int64_t)n_rows * n + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    slope_one_dev_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(F, M1, M2, ld_in, n_rows, n, ldexp(1.0, -s), E, lde);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_slope_one_score_topk_f64(const double *E, int64_t lde, int32_t n_items, const int64_t *indptr,
                                           const int32_t *items, const float *ratings, const int64_t *mask_indptr,
                                           const int32_t *mask_indices, const int32_t *users, int32_t user_begin,
                                           int64_t n_sel, int k, int32_t *out_idx, double *out_val, void *stream) {
    EB_ARG(E && indptr && items && ratings && out_idx && out_val, "null pointer");
    EB_ARG(n_items >= 1 && lde >= n_items && n_sel >= 0 && user_begin >= 0, "bad shape n_items=%d lde=%lld n_sel=%lld",
           n_items, (long long)lde, (long long)n_sel);
    EB_ARG(k >= 1 && k <= SELECT_KMAX, "k=%d outside [1, %d]", k, SELECT_KMAX);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel == 0) return EB_OK;
    SlopeOneParams p{E, lde, n_items, indptr, items, ratings, mask_indptr, mask_indices, users, user_begin, n_sel, k,
                     so_tile(n_items), so_kbuf(k), out_idx, out_val};
    const size_t smem = (size_t)p.tile * 8 + (size_t)p.kbuf * 12;
    EB_CUDA(cudaFuncSetAttribute(slope_one_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    EB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, slope_one_score_kernel, SO_NT, smem));
    if (per_sm < 1) per_sm = 1;
    int64_t grid = (int64_t)sm_count() * per_sm;
    if (grid > n_sel) grid = n_sel;
    slope_one_score_kernel<<<(unsigned)grid, SO_NT, smem, (cudaStream_t)stream>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
