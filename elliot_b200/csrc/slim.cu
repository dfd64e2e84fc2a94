// slim.cu — SLIM (latent_factor_models/Slim/slim_model.py:44-113): one positive elastic net per item, fitted by
// sklearn's sparse coordinate descent (_cd_fast.pyx: sparse_enet_coordinate_descent, gap_enet_sparse), batched.
//
// One warp (one CTA) per item problem p.  Every problem reads the same CSC of X [users][items]; problem p treats user
// row p as zero (the reference zeroes the CSR row it indexes with the item id) and regresses y = X[:, p] (taken before
// the zeroing) on every column, its own included.  Per problem:
//   residual   R [n_users] fp32, in shared memory when it fits, otherwise in a per-problem global row;
//   norms      the shared column norms, recomputed for the columns user p rates;
//   w, XtA     [n_items] fp32, the active set [n_items] and the excluded flags [n_items], in per-problem global rows.
// Per coordinate: j = active[xorshift() % n_active] (the stream is the same for every problem, as every fit starts from
// the same seed); tmp = sum R[u] * x_uj in fp32, users ascending, one rounded product and one rounded add each (the
// warp forms 32 products at a time and adds them in order); tmp += w_j * norm_j; w_j = 0 if tmp < 0, else
// fp32((fp64(|tmp|) - l1) / fp64(norm_j + l2)) (the soft threshold runs in double in the reference: Cython binds the
// fused fmax of a double argument to its double version); then R[u] += x_uj * (w_old - w_new) in fp32.
// After an epoch whose largest update is small (d_w_max / w_max <= tol, fp32) or the last one, the duality gap: XtA is
// the reference's ordered fp32 loop, the BLAS reductions (R.R, R.y, w.w, sum |w|, y.y) run in fp64 with the warp's
// butterfly order.  gap <= tol * y.y stops; otherwise gap-safe screening rebuilds the active set in column order and
// removes the screened columns' contributions from R in column order, as the reference does.
// Epilogue: nnz of w and the entry the reference's min(nnz - 1, neighborhood) rule drops when nnz <= neighborhood (the
// smallest value, ties: the highest column), and w written to W's dense layout coef_t[i][p].
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>

#include "block_select.cuh"
#include "common.cuh"

namespace eb {

constexpr unsigned FULL = 0xffffffffu;

struct SlimParams {
    const int64_t *colptr;          // CSC of X
    const int32_t *rows;
    const float *vals;
    const int64_t *rowptr;          // CSR pattern of X (user p's columns)
    const int32_t *cols;
    const float *norm_base;         // column norms of X
    int32_t n_users, n_items, item_begin, n_problems;
    float l1, l2, tol;
    uint32_t seed;
    int max_iter, neighborhood;
    int shared_residual;
    // per-slot rows (slot = blockIdx.x)
    float *w, *norm, *xta, *resid;
    uint32_t *active;
    uint8_t *excl;
    // outputs, by item
    float *coef_t;                  // [n_items][n_items], coef_t[i * n_items + p]
    int32_t *n_iter, *nnz, *drop;
    float *gap;
};

__device__ __forceinline__ uint32_t xorshift(uint32_t &s) {
    if (s == 0) s = 1;
    s ^= s << 13;
    s ^= s >> 17;
    s ^= s << 5;
    return s % 2147483648u;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// sum over column j of x_uj * R[u] in fp32 in stored (user) order, x_pj read as 0; every lane gets the sum
__device__ __forceinline__ float col_dot(const SlimParams &q, int j, int p, const float *R, int lane) {
    const int64_t s = q.colptr[j], e = q.colptr[j + 1];
    float acc = 0.f;
    for (int64_t b = s; b < e; b += 32) {
        const int64_t i = b + lane;
        float prod = 0.f;
        if (i < e) {
            const int u = q.rows[i];
            prod = __fmul_rn(R[u], u == p ? 0.f : q.vals[i]);
        }
        const int cnt = (int)min((int64_t)32, e - b);
#pragma unroll
        for (int k = 0; k < 32; k++) {
            const float t = __shfl_sync(FULL, prod, k);
            if (k < cnt) acc = __fadd_rn(acc, t);
        }
    }
    return acc;
}

// R[u] += x_uj * a over column j (user p skipped: its x is 0)
__device__ __forceinline__ void col_axpy(const SlimParams &q, int j, int p, float a, float *R, int lane) {
    const int64_t s = q.colptr[j], e = q.colptr[j + 1];
    for (int64_t i = s + lane; i < e; i += 32) {
        const int u = q.rows[i];
        if (u != p) R[u] = __fadd_rn(R[u], __fmul_rn(q.vals[i], a));
    }
    __syncwarp();
}

// the duality gap (as fp32) and XtA; dual = max XtA
__device__ float gap_of(const SlimParams &q, int p, const float *R, const float *w, float *xta, float &dual, int lane) {
    const int U = q.n_users, n = q.n_items;
    double rr = 0, ry = 0, ww = 0, wl1 = 0;
    for (int u = lane; u < U; u += 32) rr += (double)R[u] * (double)R[u];
    for (int64_t i = q.colptr[p] + lane; i < q.colptr[p + 1]; i += 32) ry += (double)R[q.rows[i]] * (double)q.vals[i];
    float dmax = -CUDART_INF_F;
    for (int j = lane; j < n; j += 32) {
        const float wj = w[j];
        ww += (double)wj * (double)wj;
        wl1 += fabs((double)wj);
        float acc = 0.f;
        for (int64_t i = q.colptr[j]; i < q.colptr[j + 1]; i++) {
            const int u = q.rows[i];
            acc = __fadd_rn(acc, __fmul_rn(u == p ? 0.f : q.vals[i], R[u]));
        }
        acc = __fsub_rn(acc, __fmul_rn(q.l2, wj));
        xta[j] = acc;
        dmax = fmaxf(dmax, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dmax = fmaxf(dmax, __shfl_xor_sync(FULL, dmax, o));
    rr = warp_sum(rr); ry = warp_sum(ry); ww = warp_sum(ww); wl1 = warp_sum(wl1);
    __syncwarp();
    dual = dmax;
    const double a = q.l1, quad = rr + (double)q.l2 * ww;
    const double scale = (double)dmax > a ? a / (double)dmax : 1.0;
    const double primal = 0.5 * quad + a * wl1, dualv = -0.5 * scale * scale * quad + scale * ry;
    return (float)(primal - dualv);
}

// gap-safe screening over the columns not yet excluded (initial: also drops zero-norm columns); returns n_active
__device__ int screen(const SlimParams &q, int p, float *R, float *w, const float *norm, const float *xta, float dual,
                      float gap, uint32_t *active, uint8_t *excl, bool initial, int lane) {
    const int n = q.n_items;
    const float den = fmaxf(q.l1, dual);
    const double bound = sqrt(2.0 * (double)gap) / (double)q.l1;
    int n_active = 0;
    for (int j0 = 0; j0 < n; j0 += 32) {
        const int j = j0 + lane;
        bool consider = false, keep = false;
        if (j < n) {
            consider = initial || !excl[j];
            if (consider) {
                if (initial && norm[j] == 0.f) {
                    keep = false;
                } else {
                    const float xj = __fdiv_rn(xta[j], den);
                    const float dj = (float)((1.0 - fabs((double)xj)) / sqrt((double)__fadd_rn(norm[j], q.l2)));
                    keep = (double)dj <= bound;
                }
            }
        }
        const unsigned kb = __ballot_sync(FULL, keep);
        if (keep) { active[n_active + __popc(kb & ((1u << lane) - 1u))] = (uint32_t)j; excl[j] = 0; }
        n_active += __popc(kb);
        unsigned db = __ballot_sync(FULL, consider && !keep);
        if (consider && !keep) excl[j] = 1;
        // remove each screened column's contribution in column order
        while (db) {
            const int l = __ffs(db) - 1;
            db &= db - 1;
            const int jj = j0 + l;
            const float wj = w[jj];
            if (wj != 0.f) {
                col_axpy(q, jj, p, wj, R, lane);
                if (lane == 0) w[jj] = 0.f;
            }
        }
        __syncwarp();
    }
    return n_active;
}

__global__ void __launch_bounds__(32) slim_cd_kernel(const SlimParams q) {
    extern __shared__ float smem_r[];
    const int lane = threadIdx.x;
    const int U = q.n_users, n = q.n_items;
    const int64_t slot = blockIdx.x;
    float *w = q.w + slot * n, *norm = q.norm + slot * n, *xta = q.xta + slot * n;
    uint32_t *active = q.active + slot * n;
    uint8_t *excl = q.excl + slot * n;
    float *R = q.shared_residual ? smem_r : q.resid + slot * U;

    for (int t = blockIdx.x; t < q.n_problems; t += gridDim.x) {
        const int p = q.item_begin + t;
        // y into R, w = 0, the norms with user p's entries taken out
        for (int u = lane; u < U; u += 32) R[u] = 0.f;
        for (int j = lane; j < n; j += 32) { w[j] = 0.f; norm[j] = q.norm_base[j]; excl[j] = 0; }
        __syncwarp();
        for (int64_t i = q.colptr[p] + lane; i < q.colptr[p + 1]; i += 32) R[q.rows[i]] = q.vals[i];
        if (p < U)
            for (int64_t e = q.rowptr[p] + lane; e < q.rowptr[p + 1]; e += 32) {
                const int j = q.cols[e];
                float s = 0.f;
                for (int64_t i = q.colptr[j]; i < q.colptr[j + 1]; i++) {
                    const float x = q.rows[i] == p ? 0.f : q.vals[i];
                    s = __fadd_rn(s, __fmul_rn(x, x));
                }
                norm[j] = s;
            }
        __syncwarp();
        double yy = 0;
        for (int64_t i = q.colptr[p] + lane; i < q.colptr[p + 1]; i += 32) yy += (double)q.vals[i] * (double)q.vals[i];
        yy = warp_sum(yy);
        const float tol_eff = __fmul_rn(q.tol, (float)yy);

        float dual;
        float gap = gap_of(q, p, R, w, xta, dual, lane);
        int iters = 0;
        if (!(gap <= tol_eff)) {
            int n_active = screen(q, p, R, w, norm, xta, dual, gap, active, excl, true, lane);
            uint32_t state = q.seed;
            for (int it = 0; it < q.max_iter; it++) {
                float w_max = 0.f, d_max = 0.f;
                for (int f = 0; f < n_active; f++) {
                    const uint32_t r = xorshift(state);
                    const int j = (int)active[r % (uint32_t)n_active];
                    const float nj = norm[j];
                    if (nj == 0.f) continue;
                    const float wj = w[j];
                    float tmp = col_dot(q, j, p, R, lane);
                    tmp = __fadd_rn(tmp, __fmul_rn(wj, nj));
                    float wn = 0.f;
                    if (!(tmp < 0.f)) {
                        const double sgn = tmp == 0.f ? 0.0 : 1.0;
                        const double num = fmax(fabs((double)tmp) - (double)q.l1, 0.0);
                        wn = __double2float_rn(__ddiv_rn(__dmul_rn(sgn, num), (double)__fadd_rn(nj, q.l2)));
                    }
                    if (wn != wj) {
                        col_axpy(q, j, p, __fsub_rn(wj, wn), R, lane);
                        if (lane == 0) w[j] = wn;
                        __syncwarp();
                    }
                    d_max = fmaxf(d_max, fabsf(__fsub_rn(wn, wj)));
                    w_max = fmaxf(w_max, fabsf(wn));
                }
                iters = it + 1;
                if (w_max == 0.f || __fdiv_rn(d_max, w_max) <= q.tol || it == q.max_iter - 1) {
                    gap = gap_of(q, p, R, w, xta, dual, lane);
                    if (gap <= tol_eff) break;
                    n_active = screen(q, p, R, w, norm, xta, dual, gap, active, excl, false, lane);
                }
            }
        }
        // epilogue: nnz, the entry the min(nnz - 1, neighborhood) rule drops, W's dense column p
        int cnt = 0;
        uint64_t mink = ~0ull;
        for (int j = lane; j < n; j += 32) {
            const float v = w[j];
            if (v != 0.f) {
                cnt++;
                const uint64_t k = pair_key(v, (uint32_t)j);
                mink = k < mink ? k : mink;
            }
            q.coef_t[(int64_t)j * n + p] = v;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            cnt += __shfl_xor_sync(FULL, cnt, o);
            const uint64_t m = __shfl_xor_sync(FULL, mink, o);
            mink = m < mink ? m : mink;
        }
        if (lane == 0) {
            q.n_iter[p] = iters;
            q.gap[p] = __fdiv_rn(gap, (float)U);
            q.nnz[p] = cnt;
            q.drop[p] = (cnt >= 1 && cnt <= q.neighborhood) ? pair_index(mink) : -1;
        }
        __syncwarp();
    }
}

// the column norms of X: sum of x^2 in stored order, fp32
__global__ void slim_norms_kernel(const int64_t *__restrict__ colptr, const float *__restrict__ vals, int32_t n, float *out) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int64_t i = colptr[j]; i < colptr[j + 1]; i++) s = __fadd_rn(s, __fmul_rn(vals[i], vals[i]));
        out[j] = s;
    }
}

__global__ void slim_drop_kernel(int32_t n, const int32_t *__restrict__ drop, float *coef_t) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x)
        if (drop[p] >= 0) coef_t[(int64_t)drop[p] * n + p] = 0.f;
}

static size_t slot_bytes(int32_t n_users, int32_t n_items, int shared_residual) {
    return (size_t)n_items * 17 + (shared_residual ? 0 : (size_t)n_users * 4) + 64;
}

}  // namespace eb

using namespace eb;

extern "C" int eb_slim_shared_residual_fits(int32_t n_users) {
    int dev = 0, max_optin = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return 0;
    return (size_t)n_users * 4 <= (size_t)max_optin ? 1 : 0;
}

extern "C" int eb_slim_slots(int32_t n_users, int shared_residual) {
    int per_sm = 0;
    const size_t smem = shared_residual ? (size_t)n_users * 4 : 0;
    if (shared_residual &&
        cudaFuncSetAttribute(slim_cd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, slim_cd_kernel, 32, smem) != cudaSuccess) return 0;
    return per_sm * sm_count();
}

extern "C" size_t eb_slim_workspace_bytes(int32_t n_users, int32_t n_items, int32_t slots, int shared_residual) {
    return (size_t)n_items * 4 + 256 + (size_t)slots * slot_bytes(n_users, n_items, shared_residual);
}

extern "C" int eb_slim_fit_f32(const int64_t *colptr, const int32_t *rows, const float *vals, const int64_t *rowptr,
                               const int32_t *cols, int32_t n_users, int32_t n_items, int32_t item_begin,
                               int32_t n_problems, float l1, float l2, float tol, uint32_t seed, int max_iter,
                               int neighborhood, int shared_residual, int32_t slots, float *coef_t, int32_t *n_iter,
                               float *gap, int32_t *nnz, int32_t *drop, void *workspace, size_t workspace_bytes,
                               void *stream) {
    EB_ARG(colptr && rows && vals && rowptr && cols && coef_t && n_iter && gap && nnz && drop && workspace, "null pointer");
    EB_ARG(n_users >= 1 && n_items >= 1 && n_items <= n_users, "bad shape n_users=%d n_items=%d: need 1 <= n_items <= n_users",
           n_users, n_items);
    EB_ARG(item_begin >= 0 && n_problems >= 0 && item_begin + n_problems <= n_items, "bad range %d + %d of %d items",
           item_begin, n_problems, n_items);
    EB_ARG(l1 > 0.f && l2 >= 0.f && max_iter >= 1 && neighborhood >= 1 && slots >= 1,
           "bad parameters l1=%g l2=%g max_iter=%d neighborhood=%d slots=%d", l1, l2, max_iter, neighborhood, slots);
    EB_ARG(workspace_bytes >= eb_slim_workspace_bytes(n_users, n_items, slots, shared_residual),
           "workspace: %zu bytes, need %zu", workspace_bytes, eb_slim_workspace_bytes(n_users, n_items, slots, shared_residual));
    if (n_problems == 0) return EB_OK;
    const int cap = eb_slim_slots(n_users, shared_residual);
    EB_ARG(cap >= 1, "the shared-memory residual of %d users does not fit a CTA", n_users);
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char *b = (unsigned char *)workspace;
    SlimParams q{};
    q.colptr = colptr; q.rows = rows; q.vals = vals; q.rowptr = rowptr; q.cols = cols;
    q.n_users = n_users; q.n_items = n_items; q.item_begin = item_begin; q.n_problems = n_problems;
    q.l1 = l1; q.l2 = l2; q.tol = tol; q.seed = seed; q.max_iter = max_iter; q.neighborhood = neighborhood;
    q.shared_residual = shared_residual;
    float *nb = (float *)b;
    size_t o = ((size_t)n_items * 4 + 255) / 256 * 256;
    const size_t S = (size_t)slots, n = (size_t)n_items;
    q.w = (float *)(b + o); o += S * n * 4;
    q.norm = (float *)(b + o); o += S * n * 4;
    q.xta = (float *)(b + o); o += S * n * 4;
    q.active = (uint32_t *)(b + o); o += S * n * 4;
    q.resid = shared_residual ? nullptr : (float *)(b + o); o += shared_residual ? 0 : S * (size_t)n_users * 4;
    q.excl = (uint8_t *)(b + o);
    q.norm_base = nb;
    q.coef_t = coef_t; q.n_iter = n_iter; q.nnz = nnz; q.drop = drop; q.gap = gap;
    slim_norms_kernel<<<(n_items + 255) / 256, 256, 0, st>>>(colptr, vals, n_items, nb);
    int64_t grid = slots < cap ? slots : cap;
    if (grid > n_problems) grid = n_problems;
    slim_cd_kernel<<<(unsigned)grid, 32, shared_residual ? (size_t)n_users * 4 : 0, st>>>(q);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_slim_drop_f32(int32_t n_items, const int32_t *drop, float *coef_t, void *stream) {
    EB_ARG(drop && coef_t && n_items >= 1, "bad arguments");
    slim_drop_kernel<<<(n_items + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_items, drop, coef_t);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
