// ease.cu — EASE^R (autoencoders/EASE_R/ease_r.py:69-91) on the GPU, in fp64.  Entry points:
//   eb_ease_normal_f64  : rows of the normal matrix from an exact fp32 Gram slab (times 4^-s, the exactness scale), with
//                         the diagonal set to fp32(count + l2_norm) as the reference stores it;
//   eb_inverse_f64      : in-place inverse of a general n x n matrix by blocked Gauss-Jordan elimination with partial
//                         pivoting (the normal matrix of explicit ratings is indefinite, so Cholesky is not an option);
//   eb_ease_weights_f32 : B = fp32(-P / diag(P)) column by column, B_jj = 0.
//
// The inverse, per panel of INV_NB columns [k0, k0 + b):
//   1. inv_panel_kernel (ONE cooperative launch): Gauss-Jordan on the n x b panel, column by column.  Per column: the
//      pivot is the largest |a| among rows >= column (lowest row on a tie, as idamax; NaN counts as the largest, so a
//      non-finite pivot is reported), then every row of the panel is updated.  Each CTA owns a contiguous block of rows;
//      one grid barrier per column separates publishing the CTAs' pivot candidates from reading them.  The panel ends up
//      holding the panel columns of the accumulated elimination matrix T.
//   2. inv_swap_kernel: the panel's row interchanges applied to every other column, and the b pivot rows copied to W.
//   3. inv_update_kernel: every other column, A <- T A, i.e. A[i][j] = (i a pivot row ? 0 : A[i][j]) + sum_c T[i][c]
//      W[c][j], an n x n x b fp64 GEMM on the tensor cores (mma.sync m16n8k16 f64, DMMA).  This is the O(n^3) work.
// After the last panel the column interchanges are applied in reverse order (inv_permute_kernel).
// Every element sees a fixed sequence of operations and no arithmetic uses atomics, so reruns are bit-identical and the
// result does not depend on the grid.
#include <cooperative_groups.h>
#include <limits.h>
#include <math_constants.h>

#include <vector>

#include "common.cuh"
#include "dmma.cuh"

namespace eb {

namespace cg = cooperative_groups;

constexpr int INV_NB = 64;                   // panel width (the GEMM's K)
constexpr int INV_NT = 256;
constexpr int INV_WARPS = INV_NT / 32;
constexpr int INV_GMAX = 1024;               // most CTAs in a panel launch
constexpr int INV_STAGE_ROWS = 256;          // rows staged at once by the final column permutation
constexpr int UPD_TILE = 64;                 // GEMM output tile (UPD_TILE x UPD_TILE)
constexpr int UPD_LDT = INV_NB + 4;          // smem row stride of the T tile: conflict-free a-fragment loads
constexpr int UPD_LDW = UPD_TILE + 8;        // smem row stride of the W tile: conflict-free b-fragment loads

__device__ int64_t g_inv_bad_col;            // smallest column with a zero or non-finite pivot (INT64_MAX: none)
__device__ int64_t g_ease_bad_col;           // smallest column j with P[j][j] zero (INT64_MAX: none)

// total order of pivot candidates: larger key first, then lower row
__device__ __forceinline__ bool piv_better(double ka, int64_t ra, double kb, int64_t rb) {
    return ka > kb || (ka == kb && ra < rb);
}
__device__ __forceinline__ double piv_key(double v) { return isnan(v) ? CUDART_INF : fabs(v); }

struct PanelParams {
    double *A;
    int64_t ld, n, k0;
    int b;
    int64_t rows;                // rows per CTA
    int32_t *piv;                // [n]
    double *cand;                // [2][INV_GMAX][INV_NB]: each CTA's best candidate row (panel columns)
    double *cand_key;            // [2][INV_GMAX]
    int64_t *cand_row;           // [2][INV_GMAX]
    double *rowc;                // [2][INV_NB]: row k0 + c before its step
};

// Reduces the warps' candidates for panel column `c` (rows >= k0 + c) and publishes the CTA's best row and, if this CTA
// owns it, row k0 + c, into buffer `par`.
__device__ void publish(const PanelParams &p, int c, int par, double bk, int64_t br, double *wkey, int64_t *wrow,
                        int64_t r0, int64_t r1) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { wkey[warp] = bk; wrow[warp] = br; }
    __syncthreads();                                          // also orders this CTA's panel writes before the copies
    double k = wkey[0];
    int64_t r = wrow[0];
#pragma unroll
    for (int w = 1; w < INV_WARPS; w++)
        if (piv_better(wkey[w], wrow[w], k, r)) { k = wkey[w]; r = wrow[w]; }
    const double *P = p.A + p.k0;
    if (threadIdx.x == 0) {
        p.cand_key[par * INV_GMAX + blockIdx.x] = k;
        p.cand_row[par * INV_GMAX + blockIdx.x] = r;
    }
    for (int j = threadIdx.x; j < p.b; j += INV_NT) {
        if (r >= 0) p.cand[((int64_t)par * INV_GMAX + blockIdx.x) * INV_NB + j] = P[r * p.ld + j];
        const int64_t kc = p.k0 + c;
        if (kc >= r0 && kc < r1) p.rowc[par * INV_NB + j] = P[kc * p.ld + j];
    }
    __syncthreads();
}

__global__ void __launch_bounds__(INV_NT) inv_panel_kernel(const PanelParams p) {
    if (g_inv_bad_col != INT64_MAX) return;                  // an earlier panel failed (uniform over the grid)
    cg::grid_group grid = cg::this_grid();
    __shared__ double prow[INV_NB], crow[INV_NB], wkey[INV_WARPS];
    __shared__ int64_t wrow[INV_WARPS];
    __shared__ int s_gbest;
    __shared__ int64_t s_rbest;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, b = p.b;
    const int64_t r0 = (int64_t)blockIdx.x * p.rows, r1 = min(p.n, r0 + p.rows);
    double *P = p.A + p.k0;
    const bool l0 = lane < b, l1 = lane + 32 < b;

    double bk = -1.0;
    int64_t br = -1;
    for (int64_t i = max(r0, p.k0) + warp; i < r1; i += INV_WARPS) {
        const double kv = piv_key(P[i * p.ld]);
        if (piv_better(kv, i, bk, br) || br < 0) { bk = kv; br = i; }
    }
    publish(p, 0, 0, bk, br, wkey, wrow, r0, r1);

    for (int c = 0; c < b; c++) {
        const int par = c & 1;
        const int64_t kc = p.k0 + c;
        grid.sync();
        if (warp == 0) {                                      // the grid's best candidate, in a fixed order
            double k = -1.0;
            int64_t r = -1;
            int gb = -1;
            for (int g = lane; g < (int)gridDim.x; g += 32) {
                const double kg = p.cand_key[par * INV_GMAX + g];
                const int64_t rg = p.cand_row[par * INV_GMAX + g];
                if (rg >= 0 && (r < 0 || piv_better(kg, rg, k, r))) { k = kg; r = rg; gb = g; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const double ko = __shfl_xor_sync(0xffffffffu, k, o);
                const int64_t ro = __shfl_xor_sync(0xffffffffu, r, o);
                const int go = __shfl_xor_sync(0xffffffffu, gb, o);
                if (ro >= 0 && (r < 0 || piv_better(ko, ro, k, r))) { k = ko; r = ro; gb = go; }
            }
            if (lane == 0) { s_gbest = gb; s_rbest = r; }
        }
        __syncthreads();
        const int gb = s_gbest;
        const int64_t pr = s_rbest;
        const double *cr = p.cand + ((int64_t)par * INV_GMAX + gb) * INV_NB;
        const double v = cr[c];
        if (!(v != 0.0 && isfinite(v))) {                     // the same v in every CTA: the whole grid stops here
            if (blockIdx.x == 0 && threadIdx.x == 0) g_inv_bad_col = kc;
            return;
        }
        for (int j = threadIdx.x; j < INV_NB; j += INV_NT) {
            prow[j] = j < b ? (j == c ? 1.0 / v : cr[j] / v) : 0.0;
            crow[j] = j < b ? p.rowc[par * INV_NB + j] : 0.0;
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) p.piv[kc] = (int32_t)pr;
        __syncthreads();
        // every row of the panel, one warp per row, two columns per lane: row kc takes the scaled pivot row, row pr
        // (the one swapped with kc) starts from the old row kc
        const bool next = c + 1 < b;
        bk = -1.0;
        br = -1;
        for (int64_t i = r0 + warp; i < r1; i += INV_WARPS) {
            double x0, x1;
            if (i == kc) {
                x0 = prow[lane];
                x1 = prow[lane + 32];
            } else {
                double a0, a1;
                if (i == pr) {
                    a0 = crow[lane];
                    a1 = crow[lane + 32];
                } else {
                    a0 = l0 ? P[i * p.ld + lane] : 0.0;
                    a1 = l1 ? P[i * p.ld + lane + 32] : 0.0;
                }
                const double t = __shfl_sync(0xffffffffu, c < 32 ? a0 : a1, c & 31);
                x0 = lane == c ? -t * prow[c] : fma(-t, prow[lane], a0);
                x1 = lane + 32 == c ? -t * prow[c] : fma(-t, prow[lane + 32], a1);
            }
            if (l0) P[i * p.ld + lane] = x0;
            if (l1) P[i * p.ld + lane + 32] = x1;
            if (next && i > kc) {
                const double kv = piv_key(__shfl_sync(0xffffffffu, c + 1 < 32 ? x0 : x1, (c + 1) & 31));
                if (br < 0 || piv_better(kv, i, bk, br)) { bk = kv; br = i; }
            }
        }
        if (next) publish(p, c + 1, par ^ 1, bk, br, wkey, wrow, r0, r1);
    }
}

// The panel's row interchanges on every column outside it, then W[c][j] = A[k0 + c][j] (rows c >= b are zero).
__global__ void inv_swap_kernel(double *A, int64_t ld, int64_t n, int64_t k0, int b, const int32_t *piv, double *W) {
    if (g_inv_bad_col != INT64_MAX) return;
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
        if (j >= k0 && j < k0 + b) continue;
        for (int c = 0; c < b; c++) {
            const int64_t kc = k0 + c, pr = piv[kc];
            if (pr != kc) {
                const double x = A[kc * ld + j];
                A[kc * ld + j] = A[pr * ld + j];
                A[pr * ld + j] = x;
            }
            W[(int64_t)c * n + j] = A[kc * ld + j];
        }
        for (int c = b; c < INV_NB; c++) W[(int64_t)c * n + j] = 0.0;
    }
}

// A[i][j] <- (k0 <= i < k0 + b ? 0 : A[i][j]) + sum_c T[i][c] W[c][j] for every column j outside the panel, where
// T[i][c] = A[i][k0 + c] (the panel).  64 x 64 output tile per CTA; 8 warps of 32 x 16, each 2 x 2 DMMA tiles.
__global__ void __launch_bounds__(INV_NT) inv_update_kernel(double *A, int64_t ld, int64_t n, int64_t k0, int b,
                                                             const double *W) {
    if (g_inv_bad_col != INT64_MAX) return;
    const int64_t col0 = (int64_t)blockIdx.x * UPD_TILE, row0 = (int64_t)blockIdx.y * UPD_TILE;
    if (col0 == k0) return;                                   // the panel's own columns (k0 is a multiple of the tile)
    extern __shared__ __align__(16) double usm[];
    double *Ts = usm, *Ws = usm + UPD_TILE * UPD_LDT;
    for (int x = threadIdx.x; x < UPD_TILE * INV_NB; x += INV_NT) {
        const int r = x / INV_NB, k = x % INV_NB;
        Ts[r * UPD_LDT + k] = (row0 + r < n && k < b) ? A[(row0 + r) * ld + k0 + k] : 0.0;
        const int kk = x / UPD_TILE, cc = x % UPD_TILE;
        Ws[kk * UPD_LDW + cc] = col0 + cc < n ? W[(int64_t)kk * n + col0 + cc] : 0.0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, q = lane & 3;
    const int wm = (warp & 1) * 32, wn = (warp >> 1) * 16;
    double acc[2][2][4];
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
        for (int ni = 0; ni < 2; ni++)
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int64_t i = row0 + wm + 16 * mi + g + 8 * (e >> 1), j = col0 + wn + 8 * ni + 2 * q + (e & 1);
                acc[mi][ni][e] = (i < n && j < n && !(i >= k0 && i < k0 + b)) ? A[i * ld + j] : 0.0;
            }
#pragma unroll
    for (int s = 0; s < INV_NB / 16; s++) {
        double a[2][8], bf[2][4];
#pragma unroll
        for (int mi = 0; mi < 2; mi++)
#pragma unroll
            for (int x = 0; x < 8; x++) a[mi][x] = Ts[(wm + 16 * mi + g + 8 * (x & 1)) * UPD_LDT + 16 * s + q + 4 * (x >> 1)];
#pragma unroll
        for (int ni = 0; ni < 2; ni++)
#pragma unroll
            for (int x = 0; x < 4; x++) bf[ni][x] = Ws[(16 * s + q + 4 * x) * UPD_LDW + wn + 8 * ni + g];
#pragma unroll
        for (int mi = 0; mi < 2; mi++)
#pragma unroll
            for (int ni = 0; ni < 2; ni++) dmma(acc[mi][ni], a[mi], bf[ni]);
    }
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
        for (int ni = 0; ni < 2; ni++)
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int64_t i = row0 + wm + 16 * mi + g + 8 * (e >> 1), j = col0 + wn + 8 * ni + 2 * q + (e & 1);
                if (i < n && j < n) A[i * ld + j] = acc[mi][ni][e];
            }
}

// A[i][j] <- A[i][perm[j]] for every row: rows are staged INV_STAGE_ROWS at a time, one CTA per row.
__global__ void inv_permute_kernel(double *A, int64_t ld, int64_t n, int64_t i0, int64_t rows, const int32_t *perm,
                                   double *stage) {
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        double *row = A + (i0 + r) * ld, *st = stage + r * n;
        for (int64_t j = threadIdx.x; j < n; j += blockDim.x) st[j] = row[j];
        __syncthreads();
        for (int64_t j = threadIdx.x; j < n; j += blockDim.x) row[j] = st[perm[j]];
        __syncthreads();
    }
}

// ---------------------------------------------------------------- normal matrix and weights
__global__ void ease_normal_kernel(const float *slab, int64_t lds, int32_t n_rows, int64_t n, int64_t row0,
                                   const int32_t *count, double l2_norm, double scale, double *A, int64_t lda) {
    for (int64_t r = blockIdx.y; r < n_rows; r += gridDim.y) {
        const int64_t i = row0 + r;
        for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x)
            A[i * lda + j] = j == i ? (double)(float)((double)count[j] + l2_norm) : (double)slab[r * lds + j] * scale;
    }
}

__global__ void ease_weights_kernel(const double *P, int64_t ldp, int64_t n, float *B, int64_t ldb) {
    for (int64_t i = blockIdx.y; i < n; i += gridDim.y) {
        for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
            const double d = P[j * ldp + j];
            if (i == j) {
                B[i * ldb + j] = 0.f;
                if (d == 0.0) atomicMin((unsigned long long *)&g_ease_bad_col, (unsigned long long)j);
            } else {
                B[i * ldb + j] = (float)(-P[i * ldp + j] / d);
            }
        }
    }
}

static size_t align256(size_t x) { return (x + 255) / 256 * 256; }

struct InvWorkspace {
    double *W, *cand, *cand_key, *rowc;
    int64_t *cand_row;
    int32_t *piv, *perm;
};

static size_t inv_layout(int64_t n, char *base, InvWorkspace *w) {
    const int64_t wrows = INV_STAGE_ROWS > INV_NB ? INV_STAGE_ROWS : INV_NB;
    const size_t sizes[7] = {(size_t)wrows * n * 8, (size_t)2 * INV_GMAX * INV_NB * 8, (size_t)2 * INV_GMAX * 8,
                             (size_t)2 * INV_NB * 8, (size_t)2 * INV_GMAX * 8, (size_t)n * 4, (size_t)n * 4};
    size_t off[7], o = 0;
    for (int s = 0; s < 7; s++) { off[s] = o; o += align256(sizes[s]); }
    if (w) {
        w->W = (double *)(base + off[0]); w->cand = (double *)(base + off[1]); w->cand_key = (double *)(base + off[2]);
        w->rowc = (double *)(base + off[3]); w->cand_row = (int64_t *)(base + off[4]); w->piv = (int32_t *)(base + off[5]);
        w->perm = (int32_t *)(base + off[6]);
    }
    return o;
}

static bool aligned8(const void *p) { return ((uintptr_t)p % 8) == 0; }

}  // namespace eb

using namespace eb;

extern "C" size_t eb_inverse_f64_workspace_bytes(int64_t n) {
    if (n <= 0) return 0;
    return inv_layout(n, nullptr, nullptr);
}

extern "C" int eb_inverse_f64(double *A, int64_t n, int64_t ld, void *workspace, size_t workspace_bytes, void *stream) {
    EB_ARG(A, "null pointer");
    EB_ARG(n >= 1 && n <= (int64_t)65535 * UPD_TILE && n <= INT_MAX && ld >= n, "bad shape n=%lld ld=%lld", (long long)n,
           (long long)ld);
    EB_ARG(aligned8(A) && aligned8(workspace), "A and workspace must be 8-byte aligned");
    const size_t need = eb_inverse_f64_workspace_bytes(n);
    if (!workspace || workspace_bytes < need)
        return set_err(EB_ERR_WORKSPACE, "eb_inverse_f64: workspace %zu bytes < %zu", workspace_bytes, need);
    cudaStream_t st = (cudaStream_t)stream;
    InvWorkspace w;
    inv_layout(n, (char *)workspace, &w);
    static const int64_t none = INT64_MAX;
    EB_CUDA(cudaMemcpyToSymbolAsync(g_inv_bad_col, &none, sizeof(none), 0, cudaMemcpyHostToDevice, st));

    int per_sm = 0;
    EB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, inv_panel_kernel, INV_NT, 0));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 2) per_sm = 2;                               // more CTAs only make the per-column grid barrier slower
    int64_t grid = (int64_t)sm_count() * per_sm;
    if (grid > INV_GMAX) grid = INV_GMAX;
    const int64_t by_rows = (n + INV_WARPS - 1) / INV_WARPS;  // at least one row per warp
    if (grid > by_rows) grid = by_rows;
    const int64_t rows = (n + grid - 1) / grid;
    grid = (n + rows - 1) / rows;
    const size_t usmem = (size_t)(UPD_TILE * UPD_LDT + INV_NB * UPD_LDW) * sizeof(double);
    EB_CUDA(cudaFuncSetAttribute(inv_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)usmem));
    const int64_t tiles = (n + UPD_TILE - 1) / UPD_TILE;
    const unsigned swap_grid = (unsigned)((n + 255) / 256);

    for (int64_t k0 = 0; k0 < n; k0 += INV_NB) {
        PanelParams p{A, ld, n, k0, (int)(n - k0 < INV_NB ? n - k0 : INV_NB), rows, w.piv, w.cand, w.cand_key,
                      w.cand_row, w.rowc};
        void *args[] = {&p};
        EB_CUDA(cudaLaunchCooperativeKernel((void *)inv_panel_kernel, dim3((unsigned)grid), dim3(INV_NT), args, 0, st));
        if (n > p.b) {
            inv_swap_kernel<<<swap_grid, 256, 0, st>>>(A, ld, n, k0, p.b, w.piv, w.W);
            EB_CUDA(cudaGetLastError());
            inv_update_kernel<<<dim3((unsigned)tiles, (unsigned)tiles), INV_NT, usmem, st>>>(A, ld, n, k0, p.b, w.W);
            EB_CUDA(cudaGetLastError());
        }
    }
    int64_t bad = INT64_MAX;
    std::vector<int32_t> piv((size_t)n);
    EB_CUDA(cudaMemcpyFromSymbolAsync(&bad, g_inv_bad_col, sizeof(bad), 0, cudaMemcpyDeviceToHost, st));
    EB_CUDA(cudaMemcpyAsync(piv.data(), w.piv, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    EB_CUDA(cudaStreamSynchronize(st));
    if (bad != INT64_MAX)
        return set_err(EB_ERR_DATA, "eb_inverse_f64: column %lld: the pivot is zero or not finite (the matrix is singular "
                       "to working precision or holds a non-finite value)", (long long)bad);
    // A^-1 = X P for X = (P A)^-1 and P the product of the row interchanges: the columns are interchanged in reverse
    std::vector<int32_t> perm((size_t)n);
    for (int64_t j = 0; j < n; j++) perm[j] = (int32_t)j;
    bool identity = true;
    for (int64_t k = n - 1; k >= 0; k--) {
        const int32_t pk = piv[k];
        if (pk != k) {
            const int32_t t = perm[k]; perm[k] = perm[pk]; perm[pk] = t;
            identity = false;
        }
    }
    if (!identity) {
        EB_CUDA(cudaMemcpyAsync(w.perm, perm.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
        for (int64_t i0 = 0; i0 < n; i0 += INV_STAGE_ROWS) {
            const int64_t r = n - i0 < INV_STAGE_ROWS ? n - i0 : INV_STAGE_ROWS;
            inv_permute_kernel<<<(unsigned)r, 256, 0, st>>>(A, ld, n, i0, r, w.perm, w.W);
            EB_CUDA(cudaGetLastError());
        }
        EB_CUDA(cudaStreamSynchronize(st));                   // `perm` is host memory the copy reads
    }
    return EB_OK;
}

extern "C" int eb_ease_normal_f64(const float *slab, int64_t ld_slab, int32_t n_rows, int64_t n, int64_t row0,
                                  const int32_t *count, double l2_norm, double scale, double *A, int64_t ld, void *stream) {
    EB_ARG(slab && count && A, "null pointer");
    EB_ARG(n >= 1 && n_rows >= 0 && row0 >= 0 && row0 + n_rows <= n && ld_slab >= n && ld >= n,
           "bad shape n=%lld n_rows=%d row0=%lld ld_slab=%lld ld=%lld", (long long)n, n_rows, (long long)row0,
           (long long)ld_slab, (long long)ld);
    if (n_rows == 0) return EB_OK;
    const unsigned gx = (unsigned)((n + 255) / 256 < 64 ? (n + 255) / 256 : 64);
    const unsigned gy = (unsigned)(n_rows < 4096 ? n_rows : 4096);
    ease_normal_kernel<<<dim3(gx, gy), 256, 0, (cudaStream_t)stream>>>(slab, ld_slab, n_rows, n, row0, count, l2_norm, scale,
                                                                      A, ld);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_ease_weights_f32(const double *P, int64_t ld_p, int64_t n, float *B, int64_t ld_b, void *stream) {
    EB_ARG(P && B, "null pointer");
    EB_ARG(n >= 1 && ld_p >= n && ld_b >= n, "bad shape n=%lld ld_p=%lld ld_b=%lld", (long long)n, (long long)ld_p,
           (long long)ld_b);
    cudaStream_t st = (cudaStream_t)stream;
    static const int64_t none = INT64_MAX;
    EB_CUDA(cudaMemcpyToSymbolAsync(g_ease_bad_col, &none, sizeof(none), 0, cudaMemcpyHostToDevice, st));
    const unsigned gx = (unsigned)((n + 255) / 256 < 64 ? (n + 255) / 256 : 64);
    const unsigned gy = (unsigned)(n < 4096 ? n : 4096);
    ease_weights_kernel<<<dim3(gx, gy), 256, 0, st>>>(P, ld_p, n, B, ld_b);
    EB_CUDA(cudaGetLastError());
    int64_t bad = INT64_MAX;
    EB_CUDA(cudaMemcpyFromSymbolAsync(&bad, g_ease_bad_col, sizeof(bad), 0, cudaMemcpyDeviceToHost, st));
    EB_CUDA(cudaStreamSynchronize(st));
    if (bad != INT64_MAX)
        return set_err(EB_ERR_DATA, "eb_ease_weights_f32: column %lld: P[j][j] is zero", (long long)bad);
    return EB_OK;
}
