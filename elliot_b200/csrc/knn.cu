// knn.cu — ItemKNN / UserKNN (knn/item_knn/item_knn_similarity.py, knn/user_knn/user_knn_similarity.py, standard
// implementation) on the GPU.  Three kernels:
//   eb_csr_to_dense_bf16    : a row range of the rating CSR, times 2^s, into a zero-filled bf16 matrix (the Gram operand,
//                             which eb_gemm_bf16 multiplies exactly when every scaled rating is an integer <= 256 and every
//                             diagonal entry of the scaled Gram is < 2^24), plus the exact squared row / column norms;
//   eb_knn_neighbors_f32    : per row of a Gram slab, cosine (or dot) values and the k largest nonzero ones
//                             (value desc, column asc) by a three-pass radix select;
//   eb_knn_score_topk_f32   : pred[p, :] = sum_q A[p, q] B[q, :] (Gustavson, int64 fixed-point accumulators in shared
//                             memory, order independent), masked, and its top k; the dense score row never reaches HBM;
//   eb_dense_score_topk_f32 : the same kernel with a dense fp32 B (EASE^R's weights): one thread per column of a tile
//                             sums that column's terms in a register, so the output equals the sparse path's bit for bit.
#include <cuda_bf16.h>
#include <math_constants.h>

#include "common.cuh"

namespace eb {

constexpr int KNN_NT = 512;                  // threads per CTA, both selection kernels
constexpr int KNN_BINS = 2048;               // radix digit: 11 + 11 + 10 bits
constexpr int KNN_KMAX = 1024;
constexpr int KNN_TILE = 24576;              // int64 accumulators per score tile (192 KB of shared memory)
constexpr long long KNN_MASKED = (long long)0x8000000000000000ull;

// order-preserving map of a float onto uint32 (larger value -> larger key)
__device__ __forceinline__ uint32_t fkey(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ bool before(float va, int ia, float vb, int ib) {   // (value desc, index asc)
    return va > vb || (va == vb && ia < ib);
}

struct SelShared {
    uint32_t hist[KNN_BINS];
    int warp_sum[KNN_NT / 32];
    int bin, above, total, base, placed;
};

// exclusive prefix of `flag` over the block in thread order; every thread gets the block total in `total`
__device__ __forceinline__ int block_excl_scan(int x, SelShared &sh, int &total) {
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
    for (int w = 0; w < KNN_NT / 32; w++) {
        const int s = sh.warp_sum[w];
        if (w < warp) before_w += s;
        t += s;
    }
    __syncthreads();
    total = t;
    return before_w + v - x;
}

// Histogram done: find the bin (counted from the top) where the running count of candidates reaches `need`.
// Sets sh.bin and sh.above (candidates in higher bins) and sh.total (all candidates in the histogram).
__device__ void find_bin(SelShared &sh, int need) {
    constexpr int PER = KNN_BINS / KNN_NT;
    const int top = KNN_BINS - 1 - PER * (int)threadIdx.x;                  // this thread's bins: top, top-1, ...
    int s = 0;
#pragma unroll
    for (int j = 0; j < PER; j++) s += (int)sh.hist[top - j];
    int total;
    const int pre = block_excl_scan(s, sh, total);
    if (threadIdx.x == 0) sh.total = total;
    if (pre < need && need <= pre + s) {
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

// Top-k threshold of the candidates get(i, v) (i in [0, n)): returns the key T of the k-th best and the number of
// candidates with key == T to take (the first ones by index).  When there are at most k candidates, T = 0 and every
// candidate is taken (no float has key 0 except a NaN pattern, which never occurs here).
template <class Get>
__device__ void radix_threshold(const Get &get, int n, int k, SelShared &sh, uint32_t &T, int &need_eq) {
    uint32_t prefix = 0, hi_mask = 0;
    int need = k;
    const int shifts[3] = {21, 10, 0}, widths[3] = {11, 11, 10};
    for (int pass = 0; pass < 3; pass++) {
        for (int b = threadIdx.x; b < KNN_BINS; b += KNN_NT) sh.hist[b] = 0;
        __syncthreads();
        const int sft = shifts[pass];
        const uint32_t dmask = (1u << widths[pass]) - 1u;
        for (int i = threadIdx.x; i < n; i += KNN_NT) {
            float v;
            if (!get(i, v)) continue;
            const uint32_t key = fkey(v);
            if ((key & hi_mask) == prefix) atomicAdd(&sh.hist[(key >> sft) & dmask], 1u);
        }
        __syncthreads();
        find_bin(sh, need);
        if (pass == 0 && sh.total <= k) { T = 0; need_eq = 0; return; }   // uniform: every candidate is taken
        prefix |= (uint32_t)sh.bin << sft;
        hi_mask |= dmask << sft;
        need -= sh.above;
        __syncthreads();
    }
    T = prefix;
    need_eq = need;
}

// Appends the selected candidates (key > T, then the first need_eq with key == T in index order) to (bv, bi)[base..).
// Returns how many were appended (placement order is arbitrary; the caller sorts).
template <class Get>
__device__ int collect(const Get &get, int n, uint32_t T, int need_eq, float *bv, int *bi, int base, int idx_offset,
                       SelShared &sh) {
    if (threadIdx.x == 0) sh.placed = 0;
    int eq_seen = 0;
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += KNN_NT) {
        const int i = i0 + (int)threadIdx.x;
        float v = 0.f;
        const bool c = i < n && get(i, v);
        const uint32_t key = c ? fkey(v) : 0u;
        const bool eq = c && key == T && need_eq > 0;
        int eq_total;
        const int r = block_excl_scan(eq ? 1 : 0, sh, eq_total);             // uniform call
        const bool take = (c && key > T) || (eq && eq_seen + r < need_eq);
        if (take) {
            const int slot = atomicAdd(&sh.placed, 1);
            bv[base + slot] = v;
            bi[base + slot] = i + idx_offset;
        }
        eq_seen += eq_total;
    }
    __syncthreads();
    return sh.placed;
}

// bitonic sort of (bv, bi)[0..m) by (value desc, index asc); slots [m, pow2) are padded with sentinels
__device__ void sort_pairs(float *bv, int *bi, int m) {
    int P = 1;
    while (P < m) P <<= 1;
    for (int i = m + (int)threadIdx.x; i < P; i += KNN_NT) { bv[i] = -CUDART_INF_F; bi[i] = 0x7fffffff; }
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < P / 2; t += KNN_NT) {
                const int lo = 2 * t - (t & (stride - 1));
                const int hi = lo + stride;
                const bool up = (lo & size) == 0;                             // ascending in (before) order
                const float va = bv[lo], vb = bv[hi];
                const int ia = bi[lo], ib = bi[hi];
                if (before(vb, ib, va, ia) == up) { bv[lo] = vb; bi[lo] = ib; bv[hi] = va; bi[hi] = ia; }
            }
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------- densify
__global__ void csr_to_dense_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                    const float *__restrict__ values, int32_t row0, int32_t n_rows, float scale,
                                    __nv_bfloat16 *__restrict__ dst, int64_t ld, float *row_sq, float *col_sq) {
    const int lane = threadIdx.x & 31;
    const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = wid; r < n_rows; r += nw) {
        float acc = 0.f;
        for (int64_t e = indptr[row0 + r] + lane; e < indptr[row0 + r + 1]; e += 32) {
            const float x = (values ? values[e] : 1.f) * scale;
            const int c = indices[e];
            dst[r * ld + c] = __float2bfloat16_rn(x);
            // scaled integers with squares < 2^24 summed below 2^24: exact in any order
            if (col_sq) atomicAdd(col_sq + c, x * x);
            acc += x * x;
        }
        if (row_sq) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0) row_sq[r] = acc;
        }
    }
}

// ---------------------------------------------------------------- neighbour selection
struct NbrParams {
    float *slab;                // [n_rows][ld]: Gram rows row0.. (overwritten with the similarity values)
    int64_t ld;
    int32_t n_rows, n, row0;
    const float *diag;          // [>= row0 + n_rows, n] Gram diagonal
    int cosine;
    float dot_scale;
    int k;
    int32_t *out_idx;
    float *out_val;
    int32_t *out_cnt;
};

__global__ void __launch_bounds__(KNN_NT) knn_neighbors_kernel(const NbrParams p) {
    __shared__ SelShared sh;
    __shared__ float bv[KNN_KMAX];
    __shared__ int bi[KNN_KMAX];
    for (int s = blockIdx.x; s < p.n_rows; s += gridDim.x) {
        float *row = p.slab + (int64_t)s * p.ld;
        const double grr = (double)p.diag[p.row0 + s];
        for (int c = threadIdx.x; c < p.n; c += KNN_NT) {
            const float g = row[c];
            float v;
            if (p.cosine) {
                const double gcc = (double)p.diag[c];
                v = (grr == 0.0 || gcc == 0.0) ? 0.f : (float)((double)g / sqrt(grr * gcc));
            } else {
                v = g * p.dot_scale;
            }
            row[c] = v;
        }
        __syncthreads();
        auto get = [row](int i, float &v) { v = row[i]; return v != 0.f; };
        uint32_t T;
        int need_eq;
        radix_threshold(get, p.n, p.k, sh, T, need_eq);
        const int m = collect(get, p.n, T, need_eq, bv, bi, 0, 0, sh);
        sort_pairs(bv, bi, m);
        for (int j = threadIdx.x; j < p.k; j += KNN_NT) {
            p.out_idx[(int64_t)s * p.k + j] = j < m ? bi[j] : -1;
            p.out_val[(int64_t)s * p.k + j] = j < m ? bv[j] : 0.f;
        }
        if (threadIdx.x == 0) p.out_cnt[s] = m;
        __syncthreads();
    }
}

// ---------------------------------------------------------------- fused sparse product + masked top-k
struct ScoreKnnParams {
    const int64_t *a_indptr; const int32_t *a_indices; const float *a_values;
    const int64_t *b_indptr; const int32_t *b_indices; const float *b_values;
    int32_t n_cols;
    const int64_t *mask_indptr; const int32_t *mask_indices;
    const int32_t *users;
    int32_t user_begin;
    int64_t n_sel;
    int k, frac_bits, tile;
    int32_t *out_idx;
    float *out_val;
    const float *b_dense;       // DENSE: B as a row-major [>= n_mid][ldb] matrix (b_indptr / b_indices / b_values unused)
    int64_t ldb;
};

__device__ __forceinline__ int64_t lower_bound64(const int32_t *__restrict__ a, int64_t lo, int64_t hi, int32_t key) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

template <bool DENSE>
__global__ void __launch_bounds__(KNN_NT) knn_score_topk_kernel(const ScoreKnnParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    long long *acc = reinterpret_cast<long long *>(smem_raw);                       // [tile]
    float *bv = reinterpret_cast<float *>(acc + p.tile);                             // [2 * KNN_KMAX]
    int *bi = reinterpret_cast<int *>(bv + 2 * KNN_KMAX);                            // [2 * KNN_KMAX]
    __shared__ SelShared sh;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double up = ldexp(1.0, p.frac_bits), down = ldexp(1.0, -p.frac_bits);
    for (int64_t q = blockIdx.x; q < p.n_sel; q += gridDim.x) {
        const int u = p.users ? p.users[q] : p.user_begin + (int)q;
        const int64_t a0 = p.a_indptr[u], a1 = p.a_indptr[u + 1];
        const int64_t m0 = p.mask_indptr ? p.mask_indptr[u] : 0, m1 = p.mask_indptr ? p.mask_indptr[u + 1] : 0;
        int cur = 0;
        for (int c0 = 0; c0 < p.n_cols; c0 += p.tile) {
            const int tn = min(p.tile, p.n_cols - c0);
            if (DENSE) {
                // one thread per column: the same fixed-point terms as below, summed in a register (B rows coalesced)
                for (int i = threadIdx.x; i < tn; i += KNN_NT) {
                    unsigned long long s = 0;
                    const float *bc = p.b_dense + c0 + i;
#pragma unroll 4
                    for (int64_t e = a0; e < a1; e++) {
                        const double a = (double)__ldg(p.a_values + e) * up;
                        s += (unsigned long long)__double2ll_rn(a * (double)__ldg(bc + (int64_t)__ldg(p.a_indices + e) * p.ldb));
                    }
                    acc[i] = (long long)s;
                }
            } else {
                for (int i = threadIdx.x; i < tn; i += KNN_NT) acc[i] = 0;
                __syncthreads();
                // Gustavson: one warp per A entry walks the B row's part inside this tile
                for (int64_t e = a0 + warp; e < a1; e += KNN_NT / 32) {
                    const int32_t qq = __ldg(p.a_indices + e);
                    const double a = (double)__ldg(p.a_values + e) * up;
                    const int64_t b0 = p.b_indptr[qq], b1 = p.b_indptr[qq + 1];
                    const int64_t j0 = c0 == 0 ? b0 : lower_bound64(p.b_indices, b0, b1, c0);
                    for (int64_t j = j0 + lane; j < b1; j += 32) {
                        const int32_t c = __ldg(p.b_indices + j);
                        if (c >= c0 + tn) break;                                  // rows are sorted
                        // a * b is exact in double; one rounding to the fixed-point grid per term, then exact int64 sums
                        const long long t = __double2ll_rn(a * (double)__ldg(p.b_values + j));
                        atomicAdd(reinterpret_cast<unsigned long long *>(acc + (c - c0)), (unsigned long long)t);
                    }
                }
            }
            __syncthreads();
            if (p.mask_indptr) {
                const int64_t s0 = lower_bound64(p.mask_indices, m0, m1, c0);
                for (int64_t m = s0 + threadIdx.x; m < m1; m += KNN_NT) {
                    const int32_t c = __ldg(p.mask_indices + m);
                    if (c >= c0 + tn) break;
                    acc[c - c0] = KNN_MASKED;
                }
            }
            __syncthreads();
            auto get = [acc, down](int i, float &v) {
                const long long x = acc[i];
                v = (float)((double)x * down);
                return x != KNN_MASKED;
            };
            uint32_t T;
            int need_eq;
            radix_threshold(get, tn, p.k, sh, T, need_eq);
            const int m = collect(get, tn, T, need_eq, bv, bi, cur, c0, sh);
            sort_pairs(bv, bi, cur + m);
            cur = min(cur + m, p.k);
        }
        for (int j = threadIdx.x; j < p.k; j += KNN_NT) {
            p.out_idx[q * p.k + j] = j < cur ? bi[j] : -1;
            p.out_val[q * p.k + j] = j < cur ? bv[j] : -CUDART_INF_F;
        }
        __syncthreads();
    }
}

static int knn_tile(int32_t n_cols) {
    const int t = (n_cols + 255) / 256 * 256;
    return t < KNN_TILE ? t : KNN_TILE;
}

template <bool DENSE>
static int launch_score_topk(const ScoreKnnParams &p, void *stream) {
    const size_t smem = (size_t)p.tile * 8 + (size_t)2 * KNN_KMAX * 8;
    EB_CUDA(cudaFuncSetAttribute(knn_score_topk_kernel<DENSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    EB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, knn_score_topk_kernel<DENSE>, KNN_NT, smem));
    if (per_sm < 1) per_sm = 1;
    int64_t grid = (int64_t)sm_count() * per_sm;
    if (grid > p.n_sel) grid = p.n_sel;
    knn_score_topk_kernel<DENSE><<<(unsigned)grid, KNN_NT, smem, (cudaStream_t)stream>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

}  // namespace eb

using namespace eb;

extern "C" int eb_csr_to_dense_bf16(const int64_t *indptr, const int32_t *indices, const float *values, int32_t row0,
                                    int32_t n_rows, int32_t n_cols, float scale, void *dst_bf16, int64_t ld, float *row_sq,
                                    float *col_sq, void *stream) {
    EB_ARG(indptr && indices && dst_bf16, "null pointer");
    EB_ARG(row0 >= 0 && n_rows >= 0 && n_cols >= 1 && ld >= n_cols, "bad shape row0=%d n_rows=%d n_cols=%d ld=%lld", row0,
           n_rows, n_cols, (long long)ld);
    if (n_rows == 0) return EB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    EB_CUDA(cudaMemsetAsync(dst_bf16, 0, (size_t)n_rows * (size_t)ld * 2, st));
    if (row_sq) EB_CUDA(cudaMemsetAsync(row_sq, 0, (size_t)n_rows * 4, st));
    if (col_sq) EB_CUDA(cudaMemsetAsync(col_sq, 0, (size_t)n_cols * 4, st));
    int64_t grid = ((int64_t)n_rows + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    csr_to_dense_kernel<<<(unsigned)grid, 256, 0, st>>>(indptr, indices, values, row0, n_rows, scale,
                                                         (__nv_bfloat16 *)dst_bf16, ld, row_sq, col_sq);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_knn_neighbors_f32(float *slab, int64_t ld, int32_t n_rows, int32_t n, int32_t row0, const float *diag,
                                    int cosine, float dot_scale, int k, int32_t *out_idx, float *out_val, int32_t *out_cnt,
                                    void *stream) {
    EB_ARG(slab && diag && out_idx && out_val && out_cnt, "null pointer");
    EB_ARG(n >= 1 && ld >= n && n_rows >= 0 && row0 >= 0, "bad shape n=%d ld=%lld n_rows=%d", n, (long long)ld, n_rows);
    EB_ARG(k >= 1 && k <= KNN_KMAX, "k=%d outside [1, %d]", k, KNN_KMAX);
    if (n_rows == 0) return EB_OK;
    NbrParams p{slab, ld, n_rows, n, row0, diag, cosine ? 1 : 0, dot_scale, k, out_idx, out_val, out_cnt};
    int64_t grid = (int64_t)sm_count() * 4;
    if (grid > n_rows) grid = n_rows;
    knn_neighbors_kernel<<<(unsigned)grid, KNN_NT, 0, (cudaStream_t)stream>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_knn_score_tile_cols(void) { return KNN_TILE; }

extern "C" int eb_knn_score_topk_f32(const int64_t *a_indptr, const int32_t *a_indices, const float *a_values,
                                     const int64_t *b_indptr, const int32_t *b_indices, const float *b_values, int32_t n_cols,
                                     const int64_t *mask_indptr, const int32_t *mask_indices, const int32_t *users,
                                     int32_t user_begin, int64_t n_sel, int k, int frac_bits, int32_t *out_idx,
                                     float *out_val, void *stream) {
    EB_ARG(a_indptr && a_indices && a_values && b_indptr && b_indices && b_values && out_idx && out_val, "null pointer");
    EB_ARG(n_cols >= 1 && n_sel >= 0 && user_begin >= 0, "bad shape n_cols=%d n_sel=%lld", n_cols, (long long)n_sel);
    EB_ARG(k >= 1 && k <= KNN_KMAX, "k=%d outside [1, %d]", k, KNN_KMAX);
    EB_ARG(frac_bits >= -1000 && frac_bits <= 1000, "frac_bits=%d out of range", frac_bits);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel == 0) return EB_OK;
    ScoreKnnParams p{a_indptr, a_indices, a_values, b_indptr, b_indices, b_values, n_cols, mask_indptr, mask_indices, users,
                     user_begin, n_sel, k, frac_bits, knn_tile(n_cols), out_idx, out_val, nullptr, 0};
    return launch_score_topk<false>(p, stream);
}

extern "C" int eb_dense_score_topk_f32(const int64_t *a_indptr, const int32_t *a_indices, const float *a_values,
                                       const float *b, int64_t ldb, int32_t n_cols, const int64_t *mask_indptr,
                                       const int32_t *mask_indices, const int32_t *users, int32_t user_begin, int64_t n_sel,
                                       int k, int frac_bits, int32_t *out_idx, float *out_val, void *stream) {
    EB_ARG(a_indptr && a_indices && a_values && b && out_idx && out_val, "null pointer");
    EB_ARG(n_cols >= 1 && ldb >= n_cols && n_sel >= 0 && user_begin >= 0, "bad shape n_cols=%d ldb=%lld n_sel=%lld", n_cols,
           (long long)ldb, (long long)n_sel);
    EB_ARG(k >= 1 && k <= KNN_KMAX, "k=%d outside [1, %d]", k, KNN_KMAX);
    EB_ARG(frac_bits >= -1000 && frac_bits <= 1000, "frac_bits=%d out of range", frac_bits);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel == 0) return EB_OK;
    ScoreKnnParams p{a_indptr, a_indices, a_values, nullptr, nullptr, nullptr, n_cols, mask_indptr, mask_indices, users,
                     user_begin, n_sel, k, frac_bits, knn_tile(n_cols), out_idx, out_val, b, ldb};
    return launch_score_topk<true>(p, stream);
}
