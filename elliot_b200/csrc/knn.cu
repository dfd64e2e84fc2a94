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
// Both selects run block_select.cuh on 32-bit float keys with 11-bit digits and sort 64-bit (value, column) pair keys.
#include <cuda_bf16.h>
#include <math_constants.h>

#include "block_select.cuh"
#include "common.cuh"

namespace eb {

constexpr int KNN_NT = 512;                  // threads per CTA, both selection kernels
constexpr int KNN_BITS = 11;                 // radix digit: 11 + 11 + 10 bits of the float keys
constexpr int KNN_TILE = 24576;              // int64 accumulators per score tile (192 KB of shared memory)
constexpr long long KNN_MASKED = (long long)0x8000000000000000ull;

// Both kernels key a candidate value v by fkey(v) for the select and by pair_key(v, column) for the sort.  pair_key order
// is (v desc, column asc) under the order of the float bits, which differs from the order of the values only for -0.0 vs
// +0.0 and for NaN.  Neither is ever a candidate: the neighbour rows drop v == 0 and hold cosine or dot values of an exact
// Gram, which are finite; a score is fp32((double)x * 2^-f) of an int64 x, never -0.0 or NaN.
using KnnShared = SelectShared<KNN_NT, KNN_BITS>;

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
    __shared__ KnnShared sh;
    __shared__ uint64_t keys[SELECT_KMAX];
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
        auto get = [row](int i, uint32_t &key) {
            const float v = row[i];
            key = fkey(v);
            return v != 0.f;
        };
        uint32_t T;
        int need_eq;
        radix_threshold(get, p.n, p.k, sh, T, need_eq);
        const int m = collect(get, p.n, T, need_eq, sh,
                              [](int slot, int i, uint32_t key) { keys[slot] = pair_key(unfkey(key), (uint32_t)i); });
        sort_desc<KNN_NT>(keys, m);
        write_topk<KNN_NT>(keys, m, p.k, p.out_idx + (int64_t)s * p.k, p.out_val + (int64_t)s * p.k, 0.f);
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
    uint64_t *keys = reinterpret_cast<uint64_t *>(acc + p.tile);                    // [2 * SELECT_KMAX]
    __shared__ KnnShared sh;
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
            auto get = [acc, down](int i, uint32_t &key) {
                const long long x = acc[i];
                key = fkey((float)((double)x * down));
                return x != KNN_MASKED;
            };
            uint32_t T;
            int need_eq;
            radix_threshold(get, tn, p.k, sh, T, need_eq);
            const int m = collect(get, tn, T, need_eq, sh, [keys, cur, c0](int slot, int i, uint32_t key) {
                keys[cur + slot] = pair_key(unfkey(key), (uint32_t)(i + c0));
            });
            sort_desc<KNN_NT>(keys, cur + m);
            cur = min(cur + m, p.k);
        }
        write_topk<KNN_NT>(keys, cur, p.k, p.out_idx + q * p.k, p.out_val + q * p.k, -CUDART_INF_F);
        __syncthreads();
    }
}

static int knn_tile(int32_t n_cols) {
    const int t = (n_cols + 255) / 256 * 256;
    return t < KNN_TILE ? t : KNN_TILE;
}

template <bool DENSE>
static int launch_score_topk(const ScoreKnnParams &p, void *stream) {
    const size_t smem = (size_t)p.tile * 8 + (size_t)2 * SELECT_KMAX * 8;
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
    EB_ARG(k >= 1 && k <= SELECT_KMAX, "k=%d outside [1, %d]", k, SELECT_KMAX);
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
    EB_ARG(k >= 1 && k <= SELECT_KMAX, "k=%d outside [1, %d]", k, SELECT_KMAX);
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
    EB_ARG(k >= 1 && k <= SELECT_KMAX, "k=%d outside [1, %d]", k, SELECT_KMAX);
    EB_ARG(frac_bits >= -1000 && frac_bits <= 1000, "frac_bits=%d out of range", frac_bits);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel == 0) return EB_OK;
    ScoreKnnParams p{a_indptr, a_indices, a_values, nullptr, nullptr, nullptr, n_cols, mask_indptr, mask_indices, users,
                     user_begin, n_sel, k, frac_bits, knn_tile(n_cols), out_idx, out_val, b, ldb};
    return launch_score_topk<true>(p, stream);
}
