// pure_svd.cu — the pieces of a randomized truncated SVD (latent_factor_models/PureSVD/pure_svd_model.py:36-43, which
// calls sklearn's randomized_svd), in fp64:
//   eb_csr_spmm_f64         : Y = A X for a CSR A (fp32 values) and a row-major fp64 X, one warp per output row, every
//                             element summed over the row's entries in stored order (no atomics: bit-reproducible);
//   eb_chol_pivoted_f64     : one CTA factors P^T G P = L L^T with diagonal pivoting (G = X^T X from eb_gram_f64) and
//                             writes M = P L^-T, so that X M has orthonormal columns (pivoted CholeskyQR);
//   eb_tall_times_small_f64 : Y = X M for a tall X and a small M, rows staged in shared memory (in place when Y == X);
//   eb_sym_eig_f64          : one CTA, cyclic Jacobi in the parallel (round-robin) order, eigenvalues descending;
//   eb_svd_finish_f64       : singular values, the transposed orientation's column scaling, and sklearn's svd_flip on the
//                             user-side vectors.
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace eb {

constexpr int SVD_WMAX = 200;
constexpr int SPMM_NT = 256;
constexpr int CHOL_NT = 512;
constexpr int CHOL_WARPS = CHOL_NT / 32;
constexpr int TTS_ROWS = 32;
constexpr int EIG_NT = 1024;
constexpr int EIG_MAX_SWEEPS = 60;
constexpr int FIN_NT = 256;

__device__ int32_t g_eig_sweeps;             // sweeps the last eb_sym_eig_f64 took (-1: it did not converge)

__device__ __forceinline__ int pk(int i, int j) { return i >= j ? i * (i + 1) / 2 + j : j * (j + 1) / 2 + i; }

// Output row r (one warp): Y[r][c] = sum over entries e of row r, in stored order, of fma(a_e, X[col_e][c], .) for the
// columns c = lane + 32 j.  The warp loads 32 entries at a time and broadcasts them.
template <int J>
__global__ void __launch_bounds__(SPMM_NT) spmm_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                       const float *__restrict__ data, int64_t n_rows, const double *__restrict__ X,
                                                       int w, int64_t ldx, double *__restrict__ Y, int64_t ldy) {
    const int lane = threadIdx.x & 31;
    const int64_t r = (int64_t)blockIdx.x * (SPMM_NT / 32) + (threadIdx.x >> 5);
    if (r >= n_rows) return;
    double acc[J];
#pragma unroll
    for (int j = 0; j < J; j++) acc[j] = 0.0;
    const int64_t b = indptr[r], e = indptr[r + 1];
    for (int64_t e0 = b; e0 < e; e0 += 32) {
        const int n = (int)min((int64_t)32, e - e0);
        int32_t my_c = 0;
        double my_v = 0.0;
        if (lane < n) {
            my_c = __ldg(indices + e0 + lane);
            my_v = (double)__ldg(data + e0 + lane);
        }
        for (int t = 0; t < n; t++) {
            const int64_t c = __shfl_sync(0xffffffffu, my_c, t);
            const double v = __shfl_sync(0xffffffffu, my_v, t);
            const double *xr = X + c * ldx;
#pragma unroll
            for (int j = 0; j < J; j++) {
                const int col = lane + 32 * j;
                if (col < w) acc[j] = fma(v, __ldg(xr + col), acc[j]);
            }
        }
    }
#pragma unroll
    for (int j = 0; j < J; j++) {
        const int col = lane + 32 * j;
        if (col < w) Y[r * ldy + col] = acc[j];
    }
}

// One CTA.  Right-looking Cholesky with diagonal pivoting on the packed lower triangle of G, without moving data: the
// Schur complement stays at the original indices, column k of L is stored at the pivot's row/column of S.  The pivot is
// the largest remaining diagonal entry (ties: the lowest index); the factorisation stops at the first pivot <= tol.
// Then every warp inverts columns of L by forward substitution and writes M[piv[j]][k] = (L^-1)[k][j].  M must be zero.
__global__ void __launch_bounds__(CHOL_NT) chol_pivoted_kernel(const double *__restrict__ G, int w, double *__restrict__ M,
                                                               int32_t *rank_out) {
    extern __shared__ double sm[];
    double *S = sm;                                        // packed lower triangle, w (w + 1) / 2
    double *xs = S + w * (w + 1) / 2;                      // CHOL_WARPS rows of w
    int *rem = (int *)(xs + CHOL_WARPS * w);               // remaining indices, ascending
    int *piv = rem + w;
    __shared__ int s_m, s_r, s_p;
    __shared__ double s_tol;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = warp; i < w; i += CHOL_WARPS)
        for (int j = lane; j <= i; j += 32) S[pk(i, j)] = G[(int64_t)i * w + j];
    for (int i = tid; i < w; i += CHOL_NT) rem[i] = i;
    __syncthreads();
    if (tid == 0) {
        double tr = 0.0;
        for (int i = 0; i < w; i++) tr += S[pk(i, i)];
        s_tol = (double)w * DBL_EPSILON * tr;
        s_m = w;
        s_r = 0;
    }
    __syncthreads();
    for (int k = 0; k < w; k++) {
        const int m = s_m;
        if (warp == 0) {
            double best = -INFINITY;
            int at = -1;
            for (int t = lane; t < m; t += 32) {
                const double v = S[pk(rem[t], rem[t])];
                if (v > best) { best = v; at = t; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int oa = __shfl_xor_sync(0xffffffffu, at, o);
                if (oa >= 0 && (at < 0 || ob > best || (ob == best && oa < at))) { best = ob; at = oa; }
            }
            if (lane == 0) {
                if (at >= 0 && best > s_tol) {
                    s_p = rem[at];
                    piv[k] = s_p;
                    for (int t = at; t < m - 1; t++) rem[t] = rem[t + 1];
                    s_m = m - 1;
                    s_r = k + 1;
                } else {
                    s_p = -1;
                }
            }
        }
        __syncthreads();
        const int p = s_p, mm = s_m;
        if (p < 0) break;
        const double l = sqrt(S[pk(p, p)]);
        for (int t = tid; t < mm; t += CHOL_NT) S[pk(rem[t], p)] /= l;
        __syncthreads();
        if (tid == 0) S[pk(p, p)] = l;
        for (int a = warp; a < mm; a += CHOL_WARPS) {
            const int qa = rem[a];
            const double la = S[pk(qa, p)];
            for (int b = lane; b <= a; b += 32) {
                const int qb = rem[b];
                S[pk(qa, qb)] = fma(-la, S[pk(qb, p)], S[pk(qa, qb)]);
            }
        }
        __syncthreads();
    }
    const int r = s_r;
    if (tid == 0 && rank_out) *rank_out = r;
    double *x = xs + warp * w;
    for (int j = warp; j < r; j += CHOL_WARPS) {
        for (int i = j + lane; i < r; i += 32) x[i] = i == j ? 1.0 : 0.0;
        __syncwarp();
        for (int k = j; k < r; k++) {
            const int pk_ = piv[k];
            const double xk = x[k] / S[pk(pk_, pk_)];
            __syncwarp();
            if (lane == 0) x[k] = xk;
            for (int i = k + 1 + lane; i < r; i += 32) x[i] = fma(-S[pk(piv[i], pk_)], xk, x[i]);
            __syncwarp();
        }
        double *row = M + (int64_t)piv[j] * w;
        for (int k = j + lane; k < r; k += 32) row[k] = x[k];
        __syncwarp();
    }
}

// Rows [32 b, 32 b + 32) of Y = X M: the rows of X are staged in shared memory first, so Y may be X itself when d == w.
// Thread c computes column c of every staged row, summing over k in order.
__global__ void tts_kernel(const double *X, int64_t n, int w, int64_t ldx, const double *__restrict__ M, int d, double *Y,
                           int64_t ldy) {
    extern __shared__ double xs[];
    const int64_t r0 = (int64_t)blockIdx.x * TTS_ROWS;
    const int rows = (int)min((int64_t)TTS_ROWS, n - r0);
    for (int x = threadIdx.x; x < TTS_ROWS * w; x += blockDim.x) {
        const int r = x / w, k = x - r * w;
        xs[x] = r < rows ? X[(r0 + r) * ldx + k] : 0.0;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < d; c += blockDim.x) {
        double acc[TTS_ROWS];
#pragma unroll
        for (int r = 0; r < TTS_ROWS; r++) acc[r] = 0.0;
        for (int k = 0; k < w; k++) {
            const double m = __ldg(M + (int64_t)k * d + c);
#pragma unroll
            for (int r = 0; r < TTS_ROWS; r++) acc[r] = fma(xs[r * w + k], m, acc[r]);
        }
#pragma unroll
        for (int r = 0; r < TTS_ROWS; r++)
            if (r < rows) Y[(r0 + r) * ldy + c] = acc[r];
    }
}

// One CTA.  A (w x w, symmetric, a working copy) and V live in global memory (they stay in L2).  One sweep visits every
// pair once in n' - 1 steps of n' / 2 disjoint pairs (round-robin order, n' = w rounded up to even); a pair is rotated
// when |a_pq| > eps sqrt(|a_pp a_qq|) and |a_pq| > w eps sum_i |a_ii|.  The absolute floor, the rank tolerance of
// eb_chol_pivoted_f64, ends the sweeps on rank-deficient matrices, whose null block otherwise keeps trading rounding
// noise with the other rows.  The sweeps stop after one without a rotation.
__global__ void __launch_bounds__(EIG_NT) sym_eig_kernel(double *A, double *V, int w, double *evals, double *evecs) {
    __shared__ double cs[SVD_WMAX / 2 + 1], sn[SVD_WMAX / 2 + 1];
    __shared__ int pp[SVD_WMAX / 2 + 1], qq[SVD_WMAX / 2 + 1];
    __shared__ int s_rot;
    __shared__ double s_floor;
    const int tid = threadIdx.x;
    const int np = (w + 1) & ~1, half = np / 2;
    for (int x = tid; x < w * w; x += EIG_NT) V[x] = (x / w == x % w) ? 1.0 : 0.0;
    if (tid == 0) {
        double tr = 0.0;
        for (int i = 0; i < w; i++) tr += fabs(A[i * w + i]);
        s_floor = (double)w * DBL_EPSILON * tr;
    }
    __syncthreads();
    const double floor_abs = s_floor;
    int sweeps = -1;
    for (int sweep = 0; sweep < EIG_MAX_SWEEPS && w > 1; sweep++) {
        if (tid == 0) s_rot = 0;
        __syncthreads();
        for (int step = 0; step < np - 1; step++) {
            if (tid < half) {
                int a, b;
                if (tid == 0) { a = np - 1; b = step; }
                else { a = (step + tid) % (np - 1); b = (step - tid + np - 1) % (np - 1); }
                const int p = min(a, b), q = max(a, b);
                double c = 1.0, s = 0.0;
                bool act = false;
                if (q < w) {
                    const double apq = A[p * w + q], app = A[p * w + p], aqq = A[q * w + q];
                    if (fabs(apq) > floor_abs && fabs(apq) > DBL_EPSILON * sqrt(fabs(app * aqq))) {
                        const double tau = (aqq - app) / (2.0 * apq);
                        const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + hypot(1.0, tau));
                        c = 1.0 / sqrt(1.0 + t * t);
                        s = t * c;
                        act = true;
                        s_rot = 1;
                    }
                }
                pp[tid] = act ? p : -1;
                qq[tid] = q;
                cs[tid] = c;
                sn[tid] = s;
            }
            __syncthreads();
            for (int x = tid; x < half * w; x += EIG_NT) {            // rows p, q <- J^T A
                const int i = x / w, j = x - i * w, p = pp[i];
                if (p < 0) continue;
                const int q = qq[i];
                const double c = cs[i], s = sn[i], ap = A[p * w + j], aq = A[q * w + j];
                A[p * w + j] = c * ap - s * aq;
                A[q * w + j] = s * ap + c * aq;
            }
            __syncthreads();
            for (int x = tid; x < half * w; x += EIG_NT) {            // columns p, q <- A J, V J
                const int i = x / w, j = x - i * w, p = pp[i];
                if (p < 0) continue;
                const int q = qq[i];
                const double c = cs[i], s = sn[i];
                const double ap = A[j * w + p], aq = A[j * w + q];
                A[j * w + p] = c * ap - s * aq;
                A[j * w + q] = s * ap + c * aq;
                const double vp = V[j * w + p], vq = V[j * w + q];
                V[j * w + p] = c * vp - s * vq;
                V[j * w + q] = s * vp + c * vq;
            }
            __syncthreads();
        }
        if (!s_rot) { sweeps = sweep + 1; break; }
        __syncthreads();
    }
    if (w == 1) sweeps = 0;
    if (tid == 0) g_eig_sweeps = sweeps;
    // descending order, ties by the lower index
    for (int i = tid; i < w; i += EIG_NT) {
        const double di = A[i * w + i];
        int rank = 0;
        for (int j = 0; j < w; j++) {
            const double dj = A[j * w + j];
            rank += (dj > di || (dj == di && j < i)) ? 1 : 0;
        }
        evals[rank] = di;
        for (int row = 0; row < w; row++) evecs[row * w + rank] = V[row * w + i];
    }
}

// One CTA per kept column k: s_k = sqrt(max(lambda_k, 0)); with scale_user_by_inv_s (the transposed orientation), the
// user column is multiplied by 1 / s_k (0 when lambda_k <= w eps sum_j max(lambda_j, 0)) and the item column by s_k.
// Then both columns are multiplied by the sign of the user column's first largest-|.| entry (+1 for a zero column).
__global__ void __launch_bounds__(FIN_NT) finish_kernel(const double *evals, int w, double *user, int64_t n_user, int64_t ld_user,
                                                        double *item, int64_t n_item, int64_t ld_item, int scale_user_by_inv_s,
                                                        double *s_out) {
    __shared__ double s_abs[FIN_NT], s_val[FIN_NT];
    __shared__ int64_t s_row[FIN_NT];
    __shared__ double s_us, s_is;
    const int k = blockIdx.x, tid = threadIdx.x;
    if (tid == 0) {
        double tr = 0.0;
        for (int j = 0; j < w; j++) tr += fmax(evals[j], 0.0);
        const double lam = fmax(evals[k], 0.0), s = sqrt(lam);
        s_out[k] = s;
        s_us = scale_user_by_inv_s ? (lam > (double)w * DBL_EPSILON * tr ? 1.0 / s : 0.0) : 1.0;
        s_is = scale_user_by_inv_s ? s : 1.0;
    }
    __syncthreads();
    const double us = s_us, is = s_is;
    double best = -1.0, bval = 0.0;
    int64_t brow = INT64_MAX;
    for (int64_t r = tid; r < n_user; r += FIN_NT) {
        const double v = user[r * ld_user + k] * us;
        if (fabs(v) > best) { best = fabs(v); bval = v; brow = r; }
    }
    s_abs[tid] = best; s_val[tid] = bval; s_row[tid] = brow;
    __syncthreads();
    for (int o = FIN_NT / 2; o > 0; o >>= 1) {
        if (tid < o) {
            const double ob = s_abs[tid + o];
            const int64_t orow = s_row[tid + o];
            if (ob > s_abs[tid] || (ob == s_abs[tid] && orow < s_row[tid])) {
                s_abs[tid] = ob; s_val[tid] = s_val[tid + o]; s_row[tid] = orow;
            }
        }
        __syncthreads();
    }
    const double sign = s_val[0] < 0.0 ? -1.0 : 1.0;
    for (int64_t r = tid; r < n_user; r += FIN_NT) user[r * ld_user + k] = user[r * ld_user + k] * us * sign;
    for (int64_t r = tid; r < n_item; r += FIN_NT) item[r * ld_item + k] = item[r * ld_item + k] * is * sign;
}

static bool aligned8(const void *p) { return ((uintptr_t)p % 8) == 0; }

static int optin_smem() {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return 227 * 1024;
    return v;
}

}  // namespace eb

using namespace eb;

extern "C" int eb_svd_max_width(void) { return SVD_WMAX; }

extern "C" int eb_csr_spmm_f64(const int64_t *indptr, const int32_t *indices, const float *data, int64_t n_rows,
                               const double *X, int w, int64_t ldx, double *Y, int64_t ldy, void *stream) {
    EB_ARG(indptr && X && Y, "null pointer");
    EB_ARG(w >= 1 && w <= SVD_WMAX, "w=%d outside [1, %d]", w, SVD_WMAX);
    EB_ARG(n_rows >= 0 && ldx >= w && ldy >= w, "bad shape n_rows=%lld w=%d ldx=%lld ldy=%lld", (long long)n_rows, w,
           (long long)ldx, (long long)ldy);
    EB_ARG(aligned8(indptr) && aligned8(X) && aligned8(Y), "misaligned pointer (fp64 and int64 arrays need 8 bytes)");
    EB_ARG((const void *)X != (const void *)Y, "Y must not be X");
    if (n_rows == 0) return EB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t grid = (n_rows + SPMM_NT / 32 - 1) / (SPMM_NT / 32);
    EB_ARG(grid <= INT32_MAX, "n_rows=%lld too large", (long long)n_rows);
    if (w <= 32) spmm_kernel<1><<<(unsigned)grid, SPMM_NT, 0, st>>>(indptr, indices, data, n_rows, X, w, ldx, Y, ldy);
    else if (w <= 64) spmm_kernel<2><<<(unsigned)grid, SPMM_NT, 0, st>>>(indptr, indices, data, n_rows, X, w, ldx, Y, ldy);
    else if (w <= 128) spmm_kernel<4><<<(unsigned)grid, SPMM_NT, 0, st>>>(indptr, indices, data, n_rows, X, w, ldx, Y, ldy);
    else spmm_kernel<7><<<(unsigned)grid, SPMM_NT, 0, st>>>(indptr, indices, data, n_rows, X, w, ldx, Y, ldy);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_chol_pivoted_f64(const double *G, int w, double *M, int32_t *rank, void *stream) {
    EB_ARG(G && M, "null pointer");
    EB_ARG(w >= 1 && w <= SVD_WMAX, "w=%d outside [1, %d]", w, SVD_WMAX);
    EB_ARG(aligned8(G) && aligned8(M), "misaligned pointer (fp64 arrays need 8 bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = ((size_t)w * (w + 1) / 2 + (size_t)CHOL_WARPS * w) * sizeof(double) + 2 * (size_t)w * sizeof(int);
    EB_ARG(smem <= (size_t)optin_smem(), "w=%d needs %zu bytes of shared memory", w, smem);
    EB_CUDA(cudaMemsetAsync(M, 0, (size_t)w * w * sizeof(double), st));
    EB_CUDA(cudaFuncSetAttribute(chol_pivoted_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    chol_pivoted_kernel<<<1, CHOL_NT, smem, st>>>(G, w, M, rank);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_tall_times_small_f64(const double *X, int64_t n, int w, int64_t ldx, const double *M, int d, double *Y,
                                       int64_t ldy, void *stream) {
    EB_ARG(X && M && Y, "null pointer");
    EB_ARG(w >= 1 && w <= SVD_WMAX && d >= 1 && d <= SVD_WMAX, "w=%d or d=%d outside [1, %d]", w, d, SVD_WMAX);
    EB_ARG(n >= 0 && ldx >= w && ldy >= d, "bad shape n=%lld w=%d ldx=%lld d=%d ldy=%lld", (long long)n, w, (long long)ldx, d,
           (long long)ldy);
    EB_ARG(aligned8(X) && aligned8(M) && aligned8(Y), "misaligned pointer (fp64 arrays need 8 bytes)");
    EB_ARG((const void *)X != (const void *)Y || (d == w && ldx == ldy), "in place needs d == w and ldy == ldx");
    if (n == 0) return EB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t grid = (n + TTS_ROWS - 1) / TTS_ROWS;
    EB_ARG(grid <= INT32_MAX, "n=%lld too large", (long long)n);
    const int nt = (d + 31) / 32 * 32;
    const size_t smem = (size_t)TTS_ROWS * w * sizeof(double);
    EB_CUDA(cudaFuncSetAttribute(tts_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    tts_kernel<<<(unsigned)grid, nt, smem, st>>>(X, n, w, ldx, M, d, Y, ldy);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" size_t eb_sym_eig_f64_workspace_bytes(int w) {
    if (w < 1 || w > SVD_WMAX) return 0;
    return 2 * (size_t)w * w * sizeof(double);
}

extern "C" int eb_sym_eig_f64(const double *A, int w, double *evals, double *evecs, void *workspace, size_t workspace_bytes,
                              void *stream) {
    EB_ARG(A && evals && evecs, "null pointer");
    EB_ARG(w >= 1 && w <= SVD_WMAX, "w=%d outside [1, %d]", w, SVD_WMAX);
    EB_ARG(aligned8(A) && aligned8(evals) && aligned8(evecs) && aligned8(workspace), "misaligned pointer (fp64 arrays need 8 bytes)");
    const size_t need = eb_sym_eig_f64_workspace_bytes(w);
    if (!workspace || workspace_bytes < need)
        return set_err(EB_ERR_WORKSPACE, "eb_sym_eig_f64: workspace %zu bytes < %zu", workspace_bytes, need);
    cudaStream_t st = (cudaStream_t)stream;
    double *Aw = (double *)workspace, *V = Aw + (size_t)w * w;
    EB_CUDA(cudaMemcpyAsync(Aw, A, (size_t)w * w * sizeof(double), cudaMemcpyDeviceToDevice, st));
    sym_eig_kernel<<<1, EIG_NT, 0, st>>>(Aw, V, w, evals, evecs);
    EB_CUDA(cudaGetLastError());
    int32_t sweeps = 0;
    EB_CUDA(cudaMemcpyFromSymbolAsync(&sweeps, g_eig_sweeps, sizeof(sweeps), 0, cudaMemcpyDeviceToHost, st));
    EB_CUDA(cudaStreamSynchronize(st));
    if (sweeps < 0)
        return set_err(EB_ERR_DATA, "eb_sym_eig_f64: no convergence in %d sweeps (is the matrix finite?)", EIG_MAX_SWEEPS);
    return EB_OK;
}

extern "C" int eb_svd_finish_f64(const double *evals, int w, int d, double *user, int64_t n_user, int64_t ld_user, double *item,
                                 int64_t n_item, int64_t ld_item, int scale_user_by_inv_s, double *s_out, void *stream) {
    EB_ARG(evals && user && item && s_out, "null pointer");
    EB_ARG(w >= 1 && w <= SVD_WMAX && d >= 1 && d <= w, "w=%d, d=%d: need 1 <= d <= w <= %d", w, d, SVD_WMAX);
    EB_ARG(n_user >= 0 && n_item >= 0 && ld_user >= d && ld_item >= d, "bad shape");
    EB_ARG(aligned8(evals) && aligned8(user) && aligned8(item) && aligned8(s_out), "misaligned pointer (fp64 arrays need 8 bytes)");
    cudaStream_t st = (cudaStream_t)stream;
    finish_kernel<<<d, FIN_NT, 0, st>>>(evals, w, user, n_user, ld_user, item, n_item, ld_item, scale_user_by_inv_s, s_out);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
