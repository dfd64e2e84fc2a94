// als.cu — iALS / WRMF normal equations (latent_factor_models/iALS/iALS_model.py:37-65,
// latent_factor_models/WRMF/wrmf_model.py:41-58) on the GPU, in fp64.  Two entry points:
//   eb_gram_f64      : G = Y^T Y, fixed-order partial sums per row part, fixed-order final sum (bit-reproducible);
//   eb_als_solve_f64 : per row r, A = G + sum_e w_e y_e y_e^T + reg I and b = sum_e c_e y_e, X[r] = A^-1 b by a
//                      Cholesky factorisation and two triangular solves in shared memory.
// The rank-k updates run on the fp64 tensor cores (mma.sync m16n8k16 f64, DMMA): the gathered rows y_e of a chunk are
// staged in shared memory, the A operand scaled by w_e as it is loaded, and only the 16x8 tiles that touch the lower
// triangle are accumulated.  A lives in shared memory as a packed lower triangle (row i at i(i+1)/2), so the DMMA
// accumulators are read from and written back to it around each chunk.
// Mappings: d <= ALS_SMALL_D gives one warp per row (8 rows per CTA); larger d gives one CTA per row.  Every element
// of A, b and x sees the same sequence of operations in both mappings and in any CTA, so results do not depend on the
// mapping, the grid or the order in which rows are visited.
#include <limits.h>

#include "common.cuh"
#include "dmma.cuh"

namespace eb {

constexpr int ALS_DMAX = 200;
constexpr int ALS_SMALL_D = 32;
constexpr int ALS_NT = 256;
constexpr int ALS_WARPS = ALS_NT / 32;
constexpr int ALS_SMALL_CH = 16;             // entries staged per chunk, small mapping
constexpr int GRAM_ROWS = 256;               // rows per Gram part (at most GRAM_PARTS parts)
constexpr int GRAM_PARTS = 128;

__device__ int32_t g_als_bad_row;            // smallest row whose factorisation met a pivot <= 0 (INT_MAX: none)

__device__ __forceinline__ int pk(int i, int j) { return i * (i + 1) / 2 + j; }

// row stride of a staged chunk: 16-column tiles plus 4, so the fragment loads of a half-warp hit 16 distinct banks
__host__ __device__ __forceinline__ int stage_ld(int d) { return (d + 15) / 16 * 16 + 4; }

// One warp: A (packed lower, d x d) += sum_k ws[k] ys[k] ys[k]^T over k < 16 * ksteps, for the lower 16x8 tiles
// t with t % tstride == t0.  Fragment layouts (PTX ISA, m16n8k16 .f64): g = lane / 4, q = lane % 4;
// a_i = A[g + 8 (i & 1)][q + 4 (i >> 1)], b_j = B[q + 4 j][g], c = {(g, 2q), (g, 2q + 1), (g + 8, 2q), (g + 8, 2q + 1)}.
__device__ void accum_lower(double *A, int d, const double *ys, int lds, const double *ws, int ksteps, int t0, int tstride) {
    const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
    const int mt = (d + 15) >> 4, nlast = (d - 1) >> 3;
    int t = 0;
    for (int mi = 0; mi < mt; mi++) {
        const int nmax = min(2 * mi + 1, nlast);
        for (int nj = 0; nj <= nmax; nj++, t++) {
            if (t % tstride != t0) continue;
            const int m0 = 16 * mi + g, m1 = m0 + 8, n0 = 8 * nj + 2 * q, n1 = n0 + 1, nb = 8 * nj + g;
            const bool k00 = m0 < d && n0 <= m0, k01 = m0 < d && n1 <= m0, k10 = m1 < d && n0 <= m1, k11 = m1 < d && n1 <= m1;
            double c[4] = {k00 ? A[pk(m0, n0)] : 0.0, k01 ? A[pk(m0, n1)] : 0.0, k10 ? A[pk(m1, n0)] : 0.0,
                           k11 ? A[pk(m1, n1)] : 0.0};
            for (int s = 0; s < ksteps; s++) {
                double a[8], b[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int k = 16 * s + q + 4 * j;
                    const double *row = ys + k * lds;
                    const double wk = ws[k];
                    a[2 * j] = row[m0] * wk;
                    a[2 * j + 1] = row[m1] * wk;
                    b[j] = row[nb];
                }
                dmma(c, a, b);
            }
            if (k00) A[pk(m0, n0)] = c[0];
            if (k01) A[pk(m0, n1)] = c[1];
            if (k10) A[pk(m1, n0)] = c[2];
            if (k11) A[pk(m1, n1)] = c[3];
        }
    }
}

// Group-wide helpers.  BLOCK: the whole CTA works on one system; otherwise one warp does.
template <bool BLOCK>
__device__ __forceinline__ void gsync() {
    if (BLOCK) __syncthreads(); else __syncwarp();
}
template <bool BLOCK>
__device__ __forceinline__ int grank() { return BLOCK ? (int)threadIdx.x : (int)(threadIdx.x & 31); }
template <bool BLOCK>
__device__ __forceinline__ int gsize() { return BLOCK ? ALS_NT : 32; }

// Stages entries [e0, e0 + n) (rows of Y, by `idx` or, when idx is NULL, the rows e0.. themselves) into ys[CH][lds],
// zero padded in both directions, with their weights (w NULL: 1) and right-hand-side weights (c may be NULL).
template <bool BLOCK>
__device__ void stage(const double *__restrict__ Y, int64_t ld_y, int d, const int32_t *__restrict__ idx,
                      const double *__restrict__ w, const double *__restrict__ c, int64_t e0, int n, int CH, int lds,
                      double *ys, double *ws, double *cs) {
    const int rk = grank<BLOCK>(), gs = gsize<BLOCK>();
    for (int x = rk; x < CH * lds; x += gs) {
        const int k = x / lds, m = x - k * lds;
        double v = 0.0;
        if (k < n && m < d) {
            const int64_t row = idx ? (int64_t)__ldg(idx + e0 + k) : e0 + k;
            v = __ldg(Y + row * ld_y + m);
        }
        ys[x] = v;
    }
    for (int k = rk; k < CH; k += gs) {
        ws[k] = k < n ? (w ? __ldg(w + e0 + k) : 1.0) : 0.0;
        if (cs) cs[k] = k < n ? __ldg(c + e0 + k) : 0.0;
    }
}

// In-place Cholesky factorisation A = L L^T of the packed lower triangle.  Returns false (uniformly over the group) if
// a pivot is not > 0.
template <bool BLOCK>
__device__ bool cholesky(double *A, int d) {
    const int rk = grank<BLOCK>(), gs = gsize<BLOCK>(), lane = threadIdx.x & 31;
    const int i0 = BLOCK ? (int)(threadIdx.x >> 5) : 0, istep = BLOCK ? ALS_WARPS : 1;
    for (int k = 0; k < d; k++) {
        const double piv = A[pk(k, k)];
        if (!(piv > 0.0)) return false;
        const double l = sqrt(piv);
        gsync<BLOCK>();
        if (rk == 0) A[pk(k, k)] = l;
        for (int i = k + 1 + rk; i < d; i += gs) A[pk(i, k)] /= l;
        gsync<BLOCK>();
        for (int i = k + 1 + i0; i < d; i += istep) {
            const double lik = A[pk(i, k)];
            for (int j = k + 1 + lane; j <= i; j += 32) A[pk(i, j)] = fma(-lik, A[pk(j, k)], A[pk(i, j)]);
        }
        gsync<BLOCK>();
    }
    return true;
}

// One warp: b <- (L L^T)^-1 b for the factor L of cholesky().
__device__ void chol_solve_warp(const double *L, int d, double *b) {
    const int lane = threadIdx.x & 31;
    for (int k = 0; k < d; k++) {
        const double zk = b[k] / L[pk(k, k)];
        __syncwarp();
        if (lane == 0) b[k] = zk;
        for (int i = k + 1 + lane; i < d; i += 32) b[i] = fma(-L[pk(i, k)], zk, b[i]);
        __syncwarp();
    }
    for (int k = d - 1; k >= 0; k--) {
        const double xk = b[k] / L[pk(k, k)];
        __syncwarp();
        if (lane == 0) b[k] = xk;
        for (int i = lane; i < k; i += 32) b[i] = fma(-L[pk(k, i)], xk, b[i]);
        __syncwarp();
    }
}

struct SolveParams {
    const double *G;
    const double *Y;
    int64_t ld_y;
    int d;
    const int64_t *indptr;
    const int32_t *indices;
    const double *w, *c;
    const int32_t *order;
    int64_t n_rows;
    double reg;
    double *X;
    int64_t ld_x;
    int ch;      // entries staged per chunk (multiple of 16)
};

// The whole solve of row r by one group (a CTA or a warp) over its shared-memory region.
template <bool BLOCK>
__device__ void solve_row(const SolveParams &p, int r, double *A, double *ys, double *ws, double *cs, double *bv) {
    const int d = p.d, lds = stage_ld(d), rk = grank<BLOCK>(), gs = gsize<BLOCK>(), lane = threadIdx.x & 31;
    const int i0 = BLOCK ? (int)(threadIdx.x >> 5) : 0, istep = BLOCK ? ALS_WARPS : 1;
    for (int i = i0; i < d; i += istep)
        for (int j = lane; j <= i; j += 32) A[pk(i, j)] = p.G[(int64_t)i * d + j] + (i == j ? p.reg : 0.0);
    for (int m = rk; m < d; m += gs) bv[m] = 0.0;
    const int64_t e_beg = p.indptr[r], e_end = p.indptr[r + 1];
    for (int64_t e0 = e_beg; e0 < e_end; e0 += p.ch) {
        const int n = (int)min((int64_t)p.ch, e_end - e0);
        gsync<BLOCK>();
        stage<BLOCK>(p.Y, p.ld_y, d, p.indices, p.w, p.c, e0, n, p.ch, lds, ys, ws, cs);
        gsync<BLOCK>();
        accum_lower(A, d, ys, lds, ws, p.ch / 16, BLOCK ? (int)(threadIdx.x >> 5) : 0, BLOCK ? ALS_WARPS : 1);
        for (int m = rk; m < d; m += gs) {
            double acc = bv[m];
            for (int k = 0; k < n; k++) acc = fma(cs[k], ys[k * lds + m], acc);
            bv[m] = acc;
        }
    }
    gsync<BLOCK>();
    if (!cholesky<BLOCK>(A, d)) {
        if (rk == 0) atomicMin(&g_als_bad_row, r);
        gsync<BLOCK>();
        return;
    }
    if (!BLOCK || threadIdx.x < 32) chol_solve_warp(A, d, bv);
    gsync<BLOCK>();
    for (int m = rk; m < d; m += gs) p.X[(int64_t)r * p.ld_x + m] = bv[m];
    gsync<BLOCK>();
}

// shared-memory doubles of one solve region: packed A, staged chunk, w and c of the chunk, b
__host__ __device__ __forceinline__ size_t region_doubles(int d, int ch) {
    return (size_t)d * (d + 1) / 2 + (size_t)ch * stage_ld(d) + 2 * (size_t)ch + stage_ld(d);
}

__global__ void __launch_bounds__(ALS_NT) als_solve_large_kernel(SolveParams p) {
    extern __shared__ double sm[];
    const int d = p.d;
    double *A = sm, *ys = A + d * (d + 1) / 2, *ws = ys + p.ch * stage_ld(d), *cs = ws + p.ch, *bv = cs + p.ch;
    for (int64_t s = blockIdx.x; s < p.n_rows; s += gridDim.x) solve_row<true>(p, p.order[s], A, ys, ws, cs, bv);
}

__global__ void __launch_bounds__(ALS_NT) als_solve_small_kernel(SolveParams p) {
    extern __shared__ double sm[];
    const int d = p.d, warp = threadIdx.x >> 5;
    double *A = sm + region_doubles(d, ALS_SMALL_CH) * warp;
    double *ys = A + d * (d + 1) / 2, *ws = ys + ALS_SMALL_CH * stage_ld(d), *cs = ws + ALS_SMALL_CH, *bv = cs + ALS_SMALL_CH;
    for (int64_t s = (int64_t)blockIdx.x * ALS_WARPS + warp; s < p.n_rows; s += (int64_t)gridDim.x * ALS_WARPS)
        solve_row<false>(p, p.order[s], A, ys, ws, cs, bv);
}

// Part p of the Gram matrix: sum over rows [p * rows, min(n, (p + 1) * rows)) in row order, packed lower triangle.
__global__ void __launch_bounds__(ALS_NT) gram_part_kernel(const double *Y, int64_t n, int d, int64_t ld, int64_t rows,
                                                           int ch, double *parts) {
    extern __shared__ double sm[];
    const int npk = d * (d + 1) / 2, lds = stage_ld(d);
    double *A = sm, *ys = A + npk, *ws = ys + ch * lds;
    for (int x = threadIdx.x; x < npk; x += ALS_NT) A[x] = 0.0;
    const int64_t r_beg = (int64_t)blockIdx.x * rows, r_end = min(n, r_beg + rows);
    for (int64_t e0 = r_beg; e0 < r_end; e0 += ch) {
        const int m = (int)min((int64_t)ch, r_end - e0);
        __syncthreads();
        stage<true>(Y, ld, d, nullptr, nullptr, nullptr, e0, m, ch, lds, ys, ws, nullptr);
        __syncthreads();
        accum_lower(A, d, ys, lds, ws, ch / 16, threadIdx.x >> 5, ALS_WARPS);
    }
    __syncthreads();
    double *out = parts + (int64_t)blockIdx.x * npk;
    for (int x = threadIdx.x; x < npk; x += ALS_NT) out[x] = A[x];
}

__global__ void gram_final_kernel(const double *parts, int n_parts, int d, double *G) {
    const int npk = d * (d + 1) / 2;
    for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < d * d; x += gridDim.x * blockDim.x) {
        const int i = x / d, j = x - i * d;
        const int o = i >= j ? pk(i, j) : pk(j, i);
        double s = 0.0;
        for (int q = 0; q < n_parts; q++) s += parts[(int64_t)q * npk + o];
        G[x] = s;
    }
}

static int gram_parts(int64_t n) {
    const int64_t p = (n + GRAM_ROWS - 1) / GRAM_ROWS;
    return (int)(p < GRAM_PARTS ? p : GRAM_PARTS);
}

static int max_smem_optin() {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return 227 * 1024;
    return v;
}

// largest chunk (64, 32 or 16 entries) whose region fits in one CTA's shared memory
static int large_chunk(int d) {
    const size_t cap = (size_t)max_smem_optin();
    for (int ch = 64; ch > 16; ch /= 2)
        if (region_doubles(d, ch) * 8 <= cap) return ch;
    return 16;
}

static bool aligned(const void *p, size_t a) { return ((uintptr_t)p % a) == 0; }

}  // namespace eb

using namespace eb;

extern "C" size_t eb_gram_f64_workspace_bytes(int64_t n, int d) {
    if (n <= 0 || d < 1 || d > ALS_DMAX) return 0;
    return (size_t)gram_parts(n) * ((size_t)d * (d + 1) / 2) * sizeof(double);
}

extern "C" int eb_gram_f64(const double *Y, int64_t n, int d, int64_t ld, double *G, void *workspace, size_t workspace_bytes,
                           void *stream) {
    EB_ARG(Y && G, "null pointer");
    EB_ARG(d >= 1 && d <= ALS_DMAX, "d=%d outside [1, %d]", d, ALS_DMAX);
    EB_ARG(n >= 0 && ld >= d, "bad shape n=%lld d=%d ld=%lld", (long long)n, d, (long long)ld);
    EB_ARG(aligned(Y, 8) && aligned(G, 8) && aligned(workspace, 8), "Y, G and workspace must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        EB_CUDA(cudaMemsetAsync(G, 0, (size_t)d * d * sizeof(double), st));
        return EB_OK;
    }
    const size_t need = eb_gram_f64_workspace_bytes(n, d);
    if (!workspace || workspace_bytes < need)
        return set_err(EB_ERR_WORKSPACE, "eb_gram_f64: workspace %zu bytes < %zu", workspace_bytes, need);
    const int parts = gram_parts(n);
    const int64_t rows = (n + parts - 1) / parts;
    const int ch = large_chunk(d);
    const size_t smem = ((size_t)d * (d + 1) / 2 + (size_t)ch * stage_ld(d) + ch) * sizeof(double);
    EB_CUDA(cudaFuncSetAttribute(gram_part_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gram_part_kernel<<<parts, ALS_NT, smem, st>>>(Y, n, d, ld, rows, ch, (double *)workspace);
    EB_CUDA(cudaGetLastError());
    const int blocks = (d * d + 255) / 256;
    gram_final_kernel<<<blocks, 256, 0, st>>>((const double *)workspace, parts, d, G);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_als_small_d_max(void) { return ALS_SMALL_D; }

extern "C" int eb_als_solve_f64(const double *G, const double *Y, int64_t ld_y, int d, const int64_t *indptr,
                                const int32_t *indices, const double *w, const double *c, const int32_t *order, int64_t n_rows,
                                double reg, double *X, int64_t ld_x, void *stream) {
    EB_ARG(G && Y && indptr && indices && w && c && order && X, "null pointer");
    EB_ARG(d >= 1 && d <= ALS_DMAX, "d=%d outside [1, %d]", d, ALS_DMAX);
    EB_ARG(ld_y >= d && ld_x >= d && n_rows >= 0, "bad shape d=%d ld_y=%lld ld_x=%lld n_rows=%lld", d, (long long)ld_y,
           (long long)ld_x, (long long)n_rows);
    EB_ARG(aligned(G, 8) && aligned(Y, 8) && aligned(w, 8) && aligned(c, 8) && aligned(X, 8) && aligned(indptr, 8) &&
               aligned(indices, 4) && aligned(order, 4),
           "misaligned pointer (fp64 and int64 arrays need 8 bytes, int32 arrays 4)");
    if (n_rows == 0) return EB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    static const int32_t none = INT_MAX;
    EB_CUDA(cudaMemcpyToSymbolAsync(g_als_bad_row, &none, sizeof(none), 0, cudaMemcpyHostToDevice, st));
    const bool small = d <= ALS_SMALL_D;
    SolveParams p{G, Y, ld_y, d, indptr, indices, w, c, order, n_rows, reg, X, ld_x, small ? ALS_SMALL_CH : large_chunk(d)};
    const size_t smem = region_doubles(d, p.ch) * sizeof(double) * (small ? ALS_WARPS : 1);
    auto kern = small ? als_solve_small_kernel : als_solve_large_kernel;
    EB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    EB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, ALS_NT, smem));
    if (per_sm < 1) per_sm = 1;
    const int64_t per_block = small ? ALS_WARPS : 1;
    int64_t grid = (int64_t)sm_count() * per_sm;
    const int64_t need = (n_rows + per_block - 1) / per_block;
    if (grid > need) grid = need;
    kern<<<(unsigned)grid, ALS_NT, smem, st>>>(p);
    EB_CUDA(cudaGetLastError());
    int32_t bad = INT_MAX;
    EB_CUDA(cudaMemcpyFromSymbolAsync(&bad, g_als_bad_row, sizeof(bad), 0, cudaMemcpyDeviceToHost, st));
    EB_CUDA(cudaStreamSynchronize(st));
    if (bad != INT_MAX)
        return set_err(EB_ERR_DATA, "eb_als_solve_f64: row %d: the normal matrix has a pivot <= 0 (not positive definite)",
                       bad);
    return EB_OK;
}
