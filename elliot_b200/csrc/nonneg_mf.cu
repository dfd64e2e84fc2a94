// nonneg_mf.cu — NonNegMF (latent_factor_models/NonNegMF/non_negative_matrix_factorization_model.py:42-84) on the GPU,
// every rounding of the reference's fp64 epoch reproduced (explicit __d*_rn intrinsics: nothing is contracted to FMA).
//   nnmf_dots_kernel       : dot_k = sum_f Q[i,f] P[u,f] from +0.0 in f order, for every rating k of the dict-order
//                            CSR: one warp per user, its lanes over the user's ratings;
//   nnmf_bias_chain_kernel : est_k = ((mu + bu[u]) + bi[i]) + dot_k, err = r_k - est_k, bu[u] += lr (err - reg bu[u]),
//                            bi[i] += lr (err - reg bi[i]), walked in rating order by ONE thread.  Every step reads the
//                            bu or bi the previous steps of the same user or item wrote: on the C1 shape the ratings
//                            fall on 636 177 dependency levels out of 811 200, so a wavefront would gain nothing.
//                            bu stays in a register for the user's run; bi lives in shared memory when I doubles fit
//                            the opt-in dynamic shared memory (global memory otherwise).  The (item, rating, dot)
//                            loads run CH_D ratings ahead of the chain, and bi of the next rating is read before this
//                            rating's bi is stored (forwarded from the register when both are the same item);
//   nnmf_row_update_kernel : for every (row, f): num = sum T[col,f] r_k, den = sum T[col,f] est_k in the row's stored
//                            order from +0.0, den += (n_row reg) S[row,f], S_out[row,f] = S[row,f] (num / den).  The
//                            user side is the dict-order CSR with T = Q; the item side the CSC in ascending user order
//                            with each entry's rating position k, T = P.  IEEE inf / NaN of a zero denominator stand.
#include "common.cuh"

namespace eb {

constexpr int CH_D = 16;          // ratings whose (item, rating, dot) loads are in flight ahead of the chain
constexpr int CH_PF = 512;        // ratings ahead of the chain whose lines are pulled into L2 with prefetch hints
constexpr int CH_COPY = 256;      // threads that stage bi into shared memory and back (168 registers each)

// ---------------------------------------------------------------- dots
__global__ void nnmf_dots_kernel(const double *__restrict__ P, const double *__restrict__ Q, int F,
                                 const int64_t *__restrict__ indptr, const int32_t *__restrict__ items, int32_t n_users,
                                 double *__restrict__ dots) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < n_users; u += warps) {
        const double *pu = P + u * F;
        for (int64_t k = __ldg(indptr + u) + lane, k1 = __ldg(indptr + u + 1); k < k1; k += 32) {
            const double *qi = Q + (int64_t)__ldg(items + k) * F;
            double d = 0.0;
            for (int f = 0; f < F; f++) d = __dadd_rn(d, __dmul_rn(__ldg(qi + f), __ldg(pu + f)));
            dots[k] = d;
        }
    }
}

// ---------------------------------------------------------------- the bias chain
struct ChainParams {
    const int64_t *indptr;
    const int32_t *items;
    const double *ratings, *dots;
    int32_t n_users, n_items;
    double mu, lr, reg;
    double *bu, *bi, *est;
};

// one rating of the chain: returns est_k, updates b (bu of the rating's user) and writes bi's new value to `bnew`
__device__ __forceinline__ double chain_step(const ChainParams &p, double &b, double bcur, double r, double d,
                                             double &bnew) {
    const double e = __dadd_rn(__dadd_rn(__dadd_rn(p.mu, b), bcur), d);
    const double err = __dsub_rn(r, e);
    b = __dadd_rn(b, __dmul_rn(p.lr, __dsub_rn(err, __dmul_rn(p.reg, b))));
    bnew = __dadd_rn(bcur, __dmul_rn(p.lr, __dsub_rn(err, __dmul_rn(p.reg, bcur))));
    return e;
}

// thread 0 walks every rating; bt is bi (shared or global memory), read and written by this thread only
__device__ __forceinline__ void chain_walk(const ChainParams &p, double *bt) {
    const int64_t n = p.indptr[p.n_users];
    if (n == 0) return;
    // user cursor: u is the user of the current rating, uend the end of its run; the next user's run end and bu are
    // loaded one user ahead (bu[v] is written only when v's run ends, so reading it early is safe)
    int u = 0;
    int64_t uend = p.indptr[1];
    double b = p.bu[0];
    int64_t pend = p.n_users > 1 ? p.indptr[2] : 0;
    double pb = p.n_users > 1 ? p.bu[1] : 0.0;
    int it[CH_D];
    double rt[CH_D], dt[CH_D];
#pragma unroll
    for (int j = 0; j < CH_D; j++) {
        it[j] = j < n ? __ldg(p.items + j) : 0;
        rt[j] = j < n ? __ldg(p.ratings + j) : 0.0;
        dt[j] = j < n ? __ldg(p.dots + j) : 0.0;
    }
    double bcur = bt[it[0]];
    for (int64_t k0 = 0; k0 < n; k0 += CH_D) {
        int in[CH_D];
        double rn[CH_D], dn[CH_D];
#pragma unroll
        for (int j = 0; j < CH_D; j++) {
            const int64_t k = k0 + CH_D + j;
            in[j] = k < n ? __ldg(p.items + k) : 0;
            rn[j] = k < n ? __ldg(p.ratings + k) : 0.0;
            dn[j] = k < n ? __ldg(p.dots + k) : 0.0;
        }
        if (k0 + CH_PF < n) {
            prefetch_l2(p.ratings + k0 + CH_PF);
            prefetch_l2(p.dots + k0 + CH_PF);
            prefetch_l2(p.est + k0 + CH_PF);
            if ((k0 & 31) == 0) prefetch_l2(p.items + k0 + CH_PF);
        }
#pragma unroll
        for (int j = 0; j < CH_D; j++) {
            const int64_t k = k0 + j;
            if (k >= n) break;
            while (k == uend) {                      // the run of user u ends (users without ratings pass unchanged)
                p.bu[u] = b;
                ++u;
                uend = pend;
                b = pb;
                pend = u + 1 < p.n_users ? p.indptr[u + 2] : 0;
                pb = u + 1 < p.n_users ? p.bu[u + 1] : 0.0;
            }
            const int inext = j + 1 < CH_D ? it[j + 1] : in[0];
            const double bnext = k + 1 < n ? bt[inext] : 0.0;    // read before this rating's store below
            double bnew;
            p.est[k] = chain_step(p, b, bcur, rt[j], dt[j], bnew);
            bt[it[j]] = bnew;
            bcur = inext == it[j] ? bnew : bnext;
        }
#pragma unroll
        for (int j = 0; j < CH_D; j++) { it[j] = in[j]; rt[j] = rn[j]; dt[j] = dn[j]; }
    }
    p.bu[u] = b;
}

template <bool SMEM>
__global__ void nnmf_bias_chain_kernel(const ChainParams p) {
    extern __shared__ __align__(16) double bs[];
    if (SMEM) {
        for (int i = threadIdx.x; i < p.n_items; i += blockDim.x) bs[i] = p.bi[i];
        __syncthreads();
    }
    if (threadIdx.x == 0) chain_walk(p, SMEM ? bs : p.bi);
    if (SMEM) {
        __syncthreads();
        for (int i = threadIdx.x; i < p.n_items; i += blockDim.x) p.bi[i] = bs[i];
    }
}

// ---------------------------------------------------------------- the multiplicative row update
__global__ void nnmf_row_update_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ cols,
                                       const int64_t *__restrict__ pos, int32_t n_rows, const double *__restrict__ ratings,
                                       const double *__restrict__ est, const double *__restrict__ T, const double *S,
                                       double *S_out, int F, double reg) {
    const int64_t total = (int64_t)n_rows * F;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = t / F;
        const int f = (int)(t - row * F);
        const int64_t e0 = __ldg(indptr + row), e1 = __ldg(indptr + row + 1);
        double num = 0.0, den = 0.0;
        for (int64_t e = e0; e < e1; e++) {
            const int64_t k = pos ? __ldg(pos + e) : e;
            const double tv = __ldg(T + (int64_t)__ldg(cols + e) * F + f);
            num = __dadd_rn(num, __dmul_rn(tv, __ldg(ratings + k)));
            den = __dadd_rn(den, __dmul_rn(tv, __ldg(est + k)));
        }
        const double s = S[t];
        den = __dadd_rn(den, __dmul_rn(__dmul_rn((double)(e1 - e0), reg), s));
        S_out[t] = __dmul_rn(s, __ddiv_rn(num, den));
    }
}

static int max_dyn_smem() {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
        return 0;
    return v;
}

static unsigned grid_for(int64_t threads, int per_block) {
    int64_t g = (threads + per_block - 1) / per_block;
    const int64_t cap = (int64_t)sm_count() * 16;
    return (unsigned)(g < 1 ? 1 : g > cap ? cap : g);
}

}  // namespace eb

using namespace eb;

extern "C" int eb_nnmf_dots_f64(const double *P, const double *Q, int F, const int64_t *indptr, const int32_t *items,
                                int32_t n_users, double *dots, void *stream) {
    EB_ARG(P && Q && indptr && dots, "null pointer");
    EB_ARG(F >= 1 && n_users >= 0, "bad shape F=%d n_users=%d", F, n_users);
    if (n_users == 0) return EB_OK;
    nnmf_dots_kernel<<<grid_for((int64_t)n_users * 32, 256), 256, 0, (cudaStream_t)stream>>>(P, Q, F, indptr, items, n_users,
                                                                                              dots);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_nnmf_bias_chain_f64(const int64_t *indptr, const int32_t *items, const double *ratings, const double *dots,
                                      int32_t n_users, int32_t n_items, double mu, double lr, double reg, double *bu,
                                      double *bi, double *est, void *stream) {
    EB_ARG(indptr && bu && bi, "null pointer");
    EB_ARG(n_users >= 0 && n_items >= 0, "bad shape n_users=%d n_items=%d", n_users, n_items);
    if (n_users == 0) return EB_OK;
    const ChainParams p{indptr, items, ratings, dots, n_users, n_items, mu, lr, reg, bu, bi, est};
    const size_t smem = (size_t)n_items * 8;
    if ((int64_t)smem <= max_dyn_smem()) {
        EB_CUDA(cudaFuncSetAttribute(nnmf_bias_chain_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        nnmf_bias_chain_kernel<true><<<1, CH_COPY, smem, (cudaStream_t)stream>>>(p);
    } else {
        nnmf_bias_chain_kernel<false><<<1, 32, 0, (cudaStream_t)stream>>>(p);
    }
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_nnmf_row_update_f64(const int64_t *indptr, const int32_t *cols, const int64_t *pos, int32_t n_rows,
                                      const double *ratings, const double *est, const double *T, const double *S,
                                      double *S_out, int F, double reg, void *stream) {
    EB_ARG(indptr && ratings && est && T && S && S_out, "null pointer");
    EB_ARG(F >= 1 && n_rows >= 0, "bad shape F=%d n_rows=%d", F, n_rows);
    EB_ARG(T != S_out, "S_out must not alias T");
    if (n_rows == 0) return EB_OK;
    nnmf_row_update_kernel<<<grid_for((int64_t)n_rows * F, 256), 256, 0, (cudaStream_t)stream>>>(
        indptr, cols, pos, n_rows, ratings, est, T, S, S_out, F, reg);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
