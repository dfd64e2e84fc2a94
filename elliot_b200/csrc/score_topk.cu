// score_topk.cu — exact full-catalogue scoring + train mask + per-user top-k on CUDA cores.
//
// Replaces MFModel.get_user_predictions (BPRMF_model.py:70-85) and
// BPRMF_batch_model.predict/get_top_k (BPRMF_batch_model.py:82-88) in the table's own
// precision (fp32 or fp64).  It is the exact path for small catalogues and the
// re-check path for users the tensor-core kernel (score_topk_tc.cu) cannot certify.
// One CTA per user at a time: warps stream item rows (coalesced), the score row lives in
// an L2-resident scratch line, masking is a CSR scatter of -inf, selection is k rounds of
// a block-wide (value desc, index asc) arg-max.
#include <math_constants.h>

#include "common.cuh"

namespace eb {

template <typename T>
struct ScoreParams {
    const T *U, *V, *bias;
    int32_t n_items;
    int d, ld;
    const int64_t *mask_indptr;
    const int32_t *mask_indices;
    const int32_t *users;
    const int32_t *positions;  // optional: row q works on user_begin+positions[q] and writes output row positions[q]
    const int32_t *n_rows_dev; // optional: number of rows actually present (device side), <= n_sel
    int32_t user_begin;
    int64_t n_sel;
    int k;
    int32_t *out_idx;
    T *out_val;
    T *scratch;  // gridDim.x rows of n_items
};

template <typename T> __device__ __forceinline__ T neg_inf();
template <> __device__ __forceinline__ float neg_inf<float>() { return -CUDART_INF_F; }
template <> __device__ __forceinline__ double neg_inf<double>() { return -CUDART_INF; }

template <typename T>
__device__ __forceinline__ bool better(T v, int i, T bv, int bi) {
    return v > bv || (v == bv && v > neg_inf<T>() && i < bi);
}

// Score of item row vr for the user row su, as every exact scoring path computes it (score_topk_exact_kernel and
// score_rank_kernel call this; the re-check filter below repeats the order for four items at once): lane-strided fma
// from 0, the xor-shuffle tree, then bias + acc.  Called by a whole warp; every lane returns the score.
template <typename T>
__device__ __forceinline__ T warp_score(const T *su, const T *vr, const T *bias, int it, int d, int lane) {
    T acc = 0;
    for (int k = lane; k < d; k += 32) acc = fma(su[k], vr[k], acc);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    return (bias ? bias[it] : (T)0) + acc;
}

template <typename T>
__global__ void __launch_bounds__(256) score_topk_exact_kernel(const ScoreParams<T> p) {
    extern __shared__ unsigned char smem_raw[];
    T *su = reinterpret_cast<T *>(smem_raw);  // user row, d entries
    __shared__ T red_v[8];
    __shared__ int red_i[8];
    __shared__ int win_i;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T *s = p.scratch + (int64_t)blockIdx.x * p.n_items;
    const int64_t n_rows = p.n_rows_dev ? min((int64_t)*p.n_rows_dev, p.n_sel) : p.n_sel;
    for (int64_t q = blockIdx.x; q < n_rows; q += gridDim.x) {
        const int64_t qo = p.positions ? (int64_t)p.positions[q] : q;
        const int u = p.users ? p.users[q] : p.user_begin + (int)qo;
        __syncthreads();
        for (int k = threadIdx.x; k < p.d; k += blockDim.x) su[k] = p.U[(int64_t)u * p.ld + k];
        __syncthreads();
        // phase 1: scores
        for (int it = warp; it < p.n_items; it += 8) {
            const T v = warp_score(su, p.V + (int64_t)it * p.ld, p.bias, it, p.d, lane);   // score_topk_tc.cu re-rank mirrors this order
            if (lane == 0) s[it] = v;
        }
        __syncthreads();
        // phase 2: train items -> -inf  (BPRMF_model.py:73-74, BPRMF_batch_model.py:88)
        if (p.mask_indptr) {
            const int64_t beg = p.mask_indptr[u], end = p.mask_indptr[u + 1];
            for (int64_t m = beg + threadIdx.x; m < end; m += blockDim.x) s[p.mask_indices[m]] = neg_inf<T>();
        }
        __syncthreads();
        // phase 3: k rounds of arg-max, ties -> lower index
        for (int r = 0; r < p.k; r++) {
            T bv = neg_inf<T>();
            int bi = 0x7fffffff;
            for (int it = threadIdx.x; it < p.n_items; it += blockDim.x) {
                const T v = s[it];
                if (better<T>(v, it, bv, bi)) { bv = v; bi = it; }
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const T ov = __shfl_xor_sync(0xffffffffu, bv, off);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
                if (better<T>(ov, oi, bv, bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) { red_v[warp] = bv; red_i[warp] = bi; }
            __syncthreads();
            if (warp == 0) {
                bv = lane < 8 ? red_v[lane] : neg_inf<T>();
                bi = lane < 8 ? red_i[lane] : 0x7fffffff;
#pragma unroll
                for (int off = 4; off > 0; off >>= 1) {
                    const T ov = __shfl_xor_sync(0xffffffffu, bv, off);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
                    if (better<T>(ov, oi, bv, bi)) { bv = ov; bi = oi; }
                }
                if (lane == 0) {
                    const bool ok = bv > neg_inf<T>();
                    p.out_idx[qo * p.k + r] = ok ? bi : -1;
                    p.out_val[qo * p.k + r] = bv;
                    win_i = ok ? bi : -1;
                    if (ok) s[bi] = neg_inf<T>();
                }
            }
            __syncthreads();
            if (win_i < 0) {  // nothing finite left: pad the tail
                for (int rr = r + 1 + threadIdx.x; rr < p.k; rr += blockDim.x) {
                    p.out_idx[qo * p.k + rr] = -1;
                    p.out_val[qo * p.k + rr] = neg_inf<T>();
                }
                break;
            }
        }
    }
}

// ---------------------------------------------------------------- re-check of the tensor-core kernel's uncertified users
// The list is short in practice (the certificate fails for a handful of users per call) while the catalogue may be huge, so
// a row-per-CTA scan is the wrong shape (2 M x 128 floats through ONE CTA: ~200 ms).  Instead:
//   filter : the ITEMS are spread over the whole grid; a warp holds four item rows in registers and runs the loop over the
//            flagged users inside, so V is read once whatever their number.  The k-th score of the user's (uncertified)
//            candidate list is a lower bound of the true k-th score, so only items scoring >= it can be in the answer: those
//            (minus train items) are appended to a short per-user list.  Per (user, item) the operations and their order are
//            those of score_topk_exact_kernel's phase 1, so the scores are bit-identical.
//   select : one warp per flagged user picks the k best of its list (score desc, index asc).
// Users beyond RC_ROWS, users whose list overflows RC_CAP and users without a finite lower bound are passed on to the
// row-per-CTA kernel through a second device-side list (normally empty).
constexpr int RC_ROWS = 1024;     // flagged users the filter handles
constexpr int RC_CAP = 1024;      // list entries per flagged user

struct RecheckParams {
    const float *U, *V, *bias;
    int32_t n_items;
    int d, ld;
    const int64_t *mask_indptr;
    const int32_t *mask_indices;
    const int32_t *positions;   // flagged rows (positions in the selected user range)
    const int32_t *n_rows_dev;  // their number
    int32_t user_begin;
    int64_t n_sel;
    int k;
    int32_t *out_idx;
    float *out_val;
    int32_t *cnt;               // [RC_ROWS] list lengths (zeroed by the caller)
    float2 *lists;              // [RC_ROWS][RC_CAP] (score, item id as int bits)
    int32_t *ovf_count;         // rows handed to the row-per-CTA kernel (zeroed by the caller)
    int32_t *ovf_list;
};

__global__ void __launch_bounds__(256) recheck_filter_kernel(const RecheckParams p) {
    __shared__ float thr[RC_ROWS];
    const int lane = threadIdx.x & 31;
    const int n_rows = (int)min(min((int64_t)*p.n_rows_dev, p.n_sel), (int64_t)RC_ROWS);
    if (n_rows <= 0) return;
    for (int q = threadIdx.x; q < n_rows; q += blockDim.x) thr[q] = p.out_val[(int64_t)p.positions[q] * p.k + p.k - 1];
    __syncthreads();
    const int wid = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), nw = (int)((gridDim.x * blockDim.x) >> 5);
    for (int64_t it0 = (int64_t)wid * 4; it0 < p.n_items; it0 += (int64_t)nw * 4) {
        float v[4][8];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const float *vr = p.V + min(it0 + j, (int64_t)p.n_items - 1) * p.ld;
#pragma unroll
            for (int c = 0; c < 8; c++) v[j][c] = lane + 32 * c < p.d ? vr[lane + 32 * c] : 0.f;
        }
        const float my_bias = (lane < 4 && it0 + lane < p.n_items && p.bias) ? p.bias[it0 + lane] : 0.f;
        for (int q = 0; q < n_rows; q++) {
            const int u = p.user_begin + p.positions[q];
            const float *ur = p.U + (int64_t)u * p.ld;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int c = 0; c < 8; c++) {
                if (32 * c < p.d) {                                   // warp-uniform
                    const bool in = lane + 32 * c < p.d;
                    const float uk = in ? __ldg(ur + lane + 32 * c) : 0.f;
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        if (in) acc[j] = fmaf(uk, v[j][c], acc[j]);
                }
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], off);
            const float t = thr[q];
            if (lane < 4 && it0 + lane < p.n_items && t > -CUDART_INF_F) {
                const float a = lane == 0 ? acc[0] : (lane == 1 ? acc[1] : (lane == 2 ? acc[2] : acc[3]));
                const float sc = my_bias + a;
                if (sc >= t) {
                    const int32_t it = (int32_t)(it0 + lane);
                    bool masked = false;
                    if (p.mask_indptr) {
                        const int64_t beg = p.mask_indptr[u];
                        masked = contains_sorted(p.mask_indices + beg, (int)(p.mask_indptr[u + 1] - beg), it);
                    }
                    if (!masked) {
                        const int slot = atomicAdd(p.cnt + q, 1);
                        if (slot < RC_CAP) p.lists[(int64_t)q * RC_CAP + slot] = make_float2(sc, __int_as_float(it));
                    }
                }
            }
        }
    }
}

__global__ void __launch_bounds__(256) recheck_select_kernel(const RecheckParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t n_rows = min((int64_t)*p.n_rows_dev, p.n_sel);
    const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t q = wid; q < n_rows; q += nw) {
        const int32_t pos = p.positions[q];
        const int c = q < RC_ROWS ? p.cnt[q] : 0;
        const bool usable = q < RC_ROWS && c <= RC_CAP && p.out_val[(int64_t)pos * p.k + p.k - 1] > -CUDART_INF_F;
        if (!usable) {                                                // warp-uniform
            if (lane == 0) p.ovf_list[atomicAdd(p.ovf_count, 1)] = pos;
            continue;
        }
        __syncwarp();
        // the k candidates that set the bound are in the list themselves (same arithmetic), so c >= k
        const float2 *L = p.lists + q * RC_CAP;
        float pv = CUDART_INF_F; int pi = -1;                          // previous winner: later rounds take strictly worse entries
        for (int r = 0; r < p.k; r++) {
            float bv = -CUDART_INF_F; int bi = 0x7fffffff;
            for (int e = lane; e < c; e += 32) {
                const float2 x = L[e];
                const float xv = x.x; const int xi = __float_as_int(x.y);
                const bool after_prev = xv < pv || (xv == pv && xi > pi);
                if (after_prev && (xv > bv || (xv == bv && xi < bi))) { bv = xv; bi = xi; }
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            const bool ok = bi != 0x7fffffff;
            if (lane == 0) {
                p.out_idx[(int64_t)pos * p.k + r] = ok ? bi : -1;
                p.out_val[(int64_t)pos * p.k + r] = ok ? bv : -CUDART_INF_F;
            }
            pv = bv; pi = bi;
            if (!ok) { pv = -CUDART_INF_F; pi = 0x7fffffff; }
        }
        __syncwarp();
    }
}

static int64_t score_ctas(int64_t n_sel) {
    int64_t c = (int64_t)sm_count() * 4;
    return n_sel < c ? (n_sel < 1 ? 1 : n_sel) : c;
}

template <typename T>
static int score_topk_exact(const T *U, const T *V, const T *bias, int32_t n_items, int d, int ld,
                            const int64_t *mask_indptr, const int32_t *mask_indices, const int32_t *users,
                            int32_t user_begin, int64_t n_sel, int k, int32_t *out_idx, T *out_val, void *workspace,
                            size_t workspace_bytes, void *stream, const int32_t *positions = nullptr,
                            const int32_t *n_rows_dev = nullptr) {
    EB_ARG(U && V && out_idx && out_val, "null pointer");
    EB_ARG(d >= 1 && ld >= d && n_items >= 1 && k >= 1, "bad shape d=%d ld=%d n_items=%d k=%d", d, ld, n_items, k);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel <= 0) return EB_OK;
    int64_t ctas = score_ctas(n_sel);
    const size_t row = sizeof(T) * (size_t)n_items;
    if (workspace_bytes < row || !workspace)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < one score row %zu", workspace_bytes, row);
    if ((size_t)ctas * row > workspace_bytes) ctas = (int64_t)(workspace_bytes / row);
    ScoreParams<T> p{U, V, bias, n_items, d, ld, mask_indptr, mask_indices, users, positions, n_rows_dev, user_begin, n_sel, k, out_idx,
                     out_val, (T *)workspace};
    score_topk_exact_kernel<T><<<(unsigned)ctas, 256, sizeof(T) * (size_t)d, (cudaStream_t)stream>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

// ---------------------------------------------------------------- rank of every relevant item in the full list
// For one user the full list is what score_topk_exact_kernel lists with k = n_items: every item outside the train mask
// whose score is neither -inf nor NaN, by (score desc, item asc).  For each relevant item in that list (a positive) the
// kernel counts the non-relevant entries ahead of it (c_i, the reference's r_i - i in auc.py / gauc.py).  One CTA per
// row, RANK_CHUNK relevant-CSR entries per pass:
//   score   : a warp per entry scores the chunk's positives (warp_score: the list's own scores, bit for bit);
//   sort    : each positive's place in (score desc, item asc) order is the number of positives better than it;
//   stream  : each warp scores 32 catalogue items, then every lane takes one: an item that is finite, not relevant and
//             not a train item adds 1 to hist[p], p = the number of positives ahead of it (binary search);
//   finish  : c of the j-th positive is hist[0] + .. + hist[j], so sum c = sum_p hist[p] * (n - p).
// Only integer atomics, so the counts do not depend on the order the warps run in.  No score row, no bitmap: any
// catalogue the scorer takes, and any number of positives (one pass over the catalogue per chunk).
constexpr int RANK_CHUNK = 1024;

template <typename T>
struct RankParams {
    const T *U, *V, *bias;
    int32_t n_items;
    int d, ld;
    const int64_t *mask_indptr;
    const int32_t *mask_indices;
    const int64_t *rel_indptr;
    const int32_t *rel_items;    // item-sorted per row, -1 (never listed) first
    const int32_t *users;
    int32_t user_begin;
    int64_t n_sel;
    int64_t *n_pos, *sum_c;
    int64_t *c_out;              // optional, per relevant-CSR entry: c of a positive, -1 otherwise
};

template <typename T>
static size_t rank_smem_bytes(int d) {
    return ((sizeof(T) * (size_t)d + 15) / 16 * 16) + (size_t)RANK_CHUNK * (2 * sizeof(T) + 3 * sizeof(int32_t)) +
           sizeof(uint32_t) * (RANK_CHUNK + 1);
}

template <typename T>
__global__ void __launch_bounds__(256) score_rank_kernel(const RankParams<T> p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T *su = reinterpret_cast<T *>(smem_raw);
    T *cv = reinterpret_cast<T *>(smem_raw + (sizeof(T) * (size_t)p.d + 15) / 16 * 16);   // chunk scores, entry order
    T *sv = cv + RANK_CHUNK;                                                              // positives, list order
    int32_t *ci = reinterpret_cast<int32_t *>(sv + RANK_CHUNK);                           // chunk items, -1: not listed
    int32_t *si = ci + RANK_CHUNK;                                                        // positives' items
    int32_t *se = si + RANK_CHUNK;                                                        // their CSR entries
    uint32_t *hist = reinterpret_cast<uint32_t *>(se + RANK_CHUNK);
    __shared__ unsigned long long s_sum;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t q = blockIdx.x; q < p.n_sel; q += gridDim.x) {
        const int u = p.users ? p.users[q] : p.user_begin + (int)q;
        const int64_t rb = p.rel_indptr[u], re = p.rel_indptr[u + 1];
        const int64_t mb = p.mask_indptr ? p.mask_indptr[u] : 0;
        const int mn = p.mask_indptr ? (int)(p.mask_indptr[u + 1] - mb) : 0;
        const int32_t *mrow = p.mask_indptr ? p.mask_indices + mb : nullptr;
        __syncthreads();
        for (int k = threadIdx.x; k < p.d; k += blockDim.x) su[k] = p.U[(int64_t)u * p.ld + k];
        if (threadIdx.x == 0) s_sum = 0;
        int64_t n_pos = 0;
        for (int64_t cb = rb; cb < re; cb += RANK_CHUNK) {
            const int ne = (int)min((int64_t)RANK_CHUNK, re - cb);
            __syncthreads();
            for (int j = warp; j < ne; j += 8) {                                          // score
                const int32_t it = p.rel_items[cb + j];
                const bool listed = it >= 0 && it < p.n_items && !contains_sorted(mrow, mn, it);             // warp-uniform
                const T v = listed ? warp_score(su, p.V + (int64_t)it * p.ld, p.bias, it, p.d, lane) : neg_inf<T>();
                if (lane == 0) { cv[j] = v; ci[j] = v > neg_inf<T>() ? it : -1; }       // NaN and -inf are not listed
            }
            __syncthreads();
            for (int j = threadIdx.x; j < ne; j += blockDim.x) {                          // sort
                const T v = cv[j];
                const int32_t it = ci[j];
                if (it < 0) {
                    if (p.c_out) p.c_out[cb + j] = -1;
                    continue;
                }
                int r = 0;
                for (int o = 0; o < ne; o++) r += ci[o] >= 0 && better<T>(cv[o], ci[o], v, it);
                sv[r] = v; si[r] = it; se[r] = (int32_t)j;
            }
            int n = 0;                                                                    // positives in the chunk
            for (int j0 = 0; j0 < RANK_CHUNK; j0 += 256) n += __syncthreads_count(j0 + (int)threadIdx.x < ne && ci[j0 + threadIdx.x] >= 0);
            if (n == 0) continue;
            for (int j = threadIdx.x; j <= n; j += blockDim.x) hist[j] = 0;
            __syncthreads();
            for (int64_t base = (int64_t)warp * 32; base < p.n_items; base += 8 * 32) {  // stream
                T mine = neg_inf<T>();
                const int m = (int)min((int64_t)32, p.n_items - base);
                for (int l = 0; l < m; l++) {
                    const int32_t it = (int32_t)(base + l);
                    const T v = warp_score(su, p.V + (int64_t)it * p.ld, p.bias, it, p.d, lane);
                    if (lane == l) mine = v;
                }
                const int32_t it = (int32_t)(base + lane);
                if (lane < m && mine > neg_inf<T>() && !contains_sorted(p.rel_items + rb, (int)(re - rb), it) &&
                    !contains_sorted(mrow, mn, it)) {
                    int lo = 0, hi = n;
                    while (lo < hi) {
                        const int mid = (lo + hi) >> 1;
                        if (better<T>(sv[mid], si[mid], mine, it)) lo = mid + 1; else hi = mid;
                    }
                    atomicAdd(hist + lo, 1u);
                }
            }
            __syncthreads();
            unsigned long long part = 0;                                                  // finish
            for (int j = threadIdx.x; j <= n; j += blockDim.x) part += (unsigned long long)hist[j] * (unsigned)(n - j);
            if (part) atomicAdd(&s_sum, part);
            if (p.c_out && threadIdx.x == 0) {
                int64_t c = 0;
                for (int j = 0; j < n; j++) { c += hist[j]; p.c_out[cb + se[j]] = c; }
            }
            n_pos += n;
        }
        __syncthreads();
        if (threadIdx.x == 0) { p.n_pos[q] = n_pos; p.sum_c[q] = (int64_t)s_sum; }
    }
}

template <typename T>
static int score_rank(const T *U, const T *V, const T *bias, int32_t n_items, int d, int ld, const int64_t *mask_indptr,
                      const int32_t *mask_indices, const int64_t *rel_indptr, const int32_t *rel_items, const int32_t *users,
                      int32_t user_begin, int64_t n_sel, int64_t *n_pos, int64_t *sum_c, int64_t *c_out, void *stream) {
    EB_ARG(U && V && rel_indptr && rel_items && n_pos && sum_c, "null pointer");
    EB_ARG(d >= 1 && ld >= d && n_items >= 1, "bad shape d=%d ld=%d n_items=%d", d, ld, n_items);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel <= 0) return EB_OK;
    const size_t smem = rank_smem_bytes<T>(d);
    if (smem > 48 * 1024) EB_CUDA(cudaFuncSetAttribute(score_rank_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    RankParams<T> p{U, V, bias, n_items, d, ld, mask_indptr, mask_indices, rel_indptr, rel_items, users, user_begin, n_sel,
                    n_pos, sum_c, c_out};
    score_rank_kernel<T><<<(unsigned)score_ctas(n_sel), 256, smem, (cudaStream_t)stream>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

}  // namespace eb

extern "C" size_t eb_score_topk_workspace_bytes(int64_t n_sel, int32_t n_items, int elem_size) {
    return (size_t)eb::score_ctas(n_sel) * (size_t)n_items * (size_t)elem_size;
}

extern "C" int eb_score_topk_f32(const float *U, const float *V, const float *item_bias, int32_t n_items, int d, int ld,
                                 const int64_t *mask_indptr, const int32_t *mask_indices, const int32_t *users,
                                 int32_t user_begin, int64_t n_sel, int k, int32_t *out_idx, float *out_val,
                                 void *workspace, size_t workspace_bytes, void *stream) {
    return eb::score_topk_exact<float>(U, V, item_bias, n_items, d, ld, mask_indptr, mask_indices, users, user_begin,
                                       n_sel, k, out_idx, out_val, workspace, workspace_bytes, stream);
}

extern "C" int eb_score_topk_f64(const double *U, const double *V, const double *item_bias, int32_t n_items, int d,
                                 int ld, const int64_t *mask_indptr, const int32_t *mask_indices, const int32_t *users,
                                 int32_t user_begin, int64_t n_sel, int k, int32_t *out_idx, double *out_val,
                                 void *workspace, size_t workspace_bytes, void *stream) {
    return eb::score_topk_exact<double>(U, V, item_bias, n_items, d, ld, mask_indptr, mask_indices, users, user_begin,
                                        n_sel, k, out_idx, out_val, workspace, workspace_bytes, stream);
}

// re-check entry used by score_topk_tc.cu: row q scores user user_begin+positions[q] and writes output row positions[q]
extern "C" int eb_score_topk_f32_mapped(const float *U, const float *V, const float *item_bias, int32_t n_items, int d,
                                        int ld, const int64_t *mask_indptr, const int32_t *mask_indices,
                                        const int32_t *positions, int32_t user_begin, int64_t n_sel, int k,
                                        int32_t *out_idx, float *out_val, void *workspace, size_t workspace_bytes,
                                        void *stream) {
    return eb::score_topk_exact<float>(U, V, item_bias, n_items, d, ld, mask_indptr, mask_indices, nullptr, user_begin,
                                       n_sel, k, out_idx, out_val, workspace, workspace_bytes, stream, positions);
}

// workspace of eb_score_topk_f32_mapped_dev: the filter's lists and counters + scratch rows for the row-per-CTA fallback
static inline size_t rc_al(size_t x) { return (x + 255) / 256 * 256; }
static const int RC_FALLBACK_ROWS = 16;
extern "C" size_t eb_score_recheck_workspace_bytes(int64_t n_sel_max, int32_t n_items) {
    if (n_sel_max < 1) n_sel_max = 1;
    const int64_t rows = n_sel_max < RC_FALLBACK_ROWS ? n_sel_max : RC_FALLBACK_ROWS;
    return rc_al((size_t)eb::RC_ROWS * 4 + 256) + rc_al((size_t)n_sel_max * 4) + rc_al((size_t)eb::RC_ROWS * eb::RC_CAP * 8) +
           rc_al((size_t)rows * (size_t)n_items * 4);
}

extern "C" int eb_score_topk_f32_mapped_dev(const float *U, const float *V, const float *item_bias, int32_t n_items, int d,
                                            int ld, const int64_t *mask_indptr, const int32_t *mask_indices,
                                            const int32_t *positions, const int32_t *n_rows_dev, int32_t user_begin,
                                            int64_t n_sel_max, int k, int32_t *out_idx, float *out_val, void *workspace,
                                            size_t workspace_bytes, void *stream) {
    EB_ARG(positions && n_rows_dev && U && V && out_idx && out_val && workspace, "null pointer");
    EB_ARG(d >= 1 && d <= 256 && ld >= d && n_items >= 1 && k >= 1, "bad shape d=%d ld=%d n_items=%d k=%d", d, ld, n_items, k);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel_max <= 0) return EB_OK;
    if (workspace_bytes < eb_score_recheck_workspace_bytes(n_sel_max, n_items))
        return eb::set_err(EB_ERR_WORKSPACE, "re-check workspace %zu < required %zu", workspace_bytes,
                           eb_score_recheck_workspace_bytes(n_sel_max, n_items));
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    size_t off = 0;
    int32_t *cnt = (int32_t *)(ws + off); int32_t *ovf_count = cnt + eb::RC_ROWS; off += rc_al((size_t)eb::RC_ROWS * 4 + 256);
    int32_t *ovf_list = (int32_t *)(ws + off); off += rc_al((size_t)n_sel_max * 4);
    float2 *lists = (float2 *)(ws + off); off += rc_al((size_t)eb::RC_ROWS * eb::RC_CAP * 8);
    EB_CUDA(cudaMemsetAsync(cnt, 0, (size_t)eb::RC_ROWS * 4 + 256, st));
    eb::RecheckParams p{U, V, item_bias, n_items, d, ld, mask_indptr, mask_indices, positions, n_rows_dev, user_begin, n_sel_max, k,
                        out_idx, out_val, cnt, lists, ovf_count, ovf_list};
    const int sms = eb::sm_count();
    eb::recheck_filter_kernel<<<sms * 4, 256, 0, st>>>(p);
    eb::recheck_select_kernel<<<sms, 256, 0, st>>>(p);
    EB_CUDA(cudaGetLastError());
    // whatever the filter could not take (normally nothing): one CTA per row, as eb_score_topk_f32
    return eb::score_topk_exact<float>(U, V, item_bias, n_items, d, ld, mask_indptr, mask_indices, nullptr, user_begin, n_sel_max, k,
                                       out_idx, out_val, ws + off, workspace_bytes - off, stream, ovf_list, ovf_count);
}

extern "C" int eb_score_rank_f32(const float *U, const float *V, const float *item_bias, int32_t n_items, int d, int ld,
                                 const int64_t *mask_indptr, const int32_t *mask_indices, const int64_t *rel_indptr,
                                 const int32_t *rel_items, const int32_t *users, int32_t user_begin, int64_t n_sel,
                                 int64_t *out_n_pos, int64_t *out_sum_c, int64_t *out_c, void *stream) {
    return eb::score_rank<float>(U, V, item_bias, n_items, d, ld, mask_indptr, mask_indices, rel_indptr, rel_items, users,
                                 user_begin, n_sel, out_n_pos, out_sum_c, out_c, stream);
}

extern "C" int eb_score_rank_f64(const double *U, const double *V, const double *item_bias, int32_t n_items, int d, int ld,
                                 const int64_t *mask_indptr, const int32_t *mask_indices, const int64_t *rel_indptr,
                                 const int32_t *rel_items, const int32_t *users, int32_t user_begin, int64_t n_sel,
                                 int64_t *out_n_pos, int64_t *out_sum_c, int64_t *out_c, void *stream) {
    return eb::score_rank<double>(U, V, item_bias, n_items, d, ld, mask_indptr, mask_indices, rel_indptr, rel_items, users,
                                  user_begin, n_sel, out_n_pos, out_sum_c, out_c, stream);
}
