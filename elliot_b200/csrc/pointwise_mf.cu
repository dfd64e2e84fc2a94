// pointwise_mf.cu — PMF and LMF (latent_factor_models/PMF/probabilistic_matrix_factorization_model.py,
// LogisticMF/logistic_matrix_factorization_model.py) and what MF / FM need beside rating_mf.cu's step.
//
//   eb_pointwise_mf_step_f32  ONE fused kernel per batch: gather -> score -> loss (fp64) -> vector-atomic gradient scatter.
//                             The loss is a template parameter:
//                               PMF: out = sigmoid(p.q), Keras MeanSquaredError; dP, dQ
//                               LMF: x = p.q + b_u + b_i, the summed log-posterior plus lambda (|p|^2 + |q|^2) / 2 per
//                                    sample; item side only (dQ, db_i): the reference's user pass reuses the item graph
//   eb_adagrad_rows_f32       TF's sparse Adagrad on the rows a batch touched, each exactly once, then their gradient rows
//                             cleared: an untouched row (and its accumulator) is what a dense pass with a zero gradient
//                             would leave, so this equals the dense pass at the cost of the touched rows only
//   eb_rating_labels_f32      label <- the train rating of (u, i) for every positive sample (binary search in the sorted
//                             train row): FM's pointwise_pos_neg_ratings_sampler from the pointwise sampler's stream
//   eb_sigmoid_scores_f32     sigmoid of every finite score; -inf (a train item) and NaN (outside the catalogue) stay
// Rows are float4 columns (f % 4 == 0, f <= 128).  A warp splits into 32 / G groups of G lanes (G = f/4 rounded up to a
// power of two), one sample per group, so a narrow row still keeps the warp busy.
// TensorFlow parity is UNPINNED (oracle/pointwise_mf.py is the checker).
#include <math_constants.h>

#include "common.cuh"

namespace eb {

enum { PMF_MSE = 0, LMF_LOGPOST = 1 };

__device__ __forceinline__ float4 pw_ld4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float4 pw_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float4 pw_axpy(float a, float4 x, float b, float4 y) {
    return make_float4(a * x.x + b * y.x, a * x.y + b * y.y, a * x.z + b * y.z, a * x.w + b * y.w);
}
__device__ __forceinline__ float pw_dot(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

// sigmoid and softplus in forms that neither overflow nor lose the small side: e = exp(-|x|) <= 1
__device__ __forceinline__ float stable_sigmoid(float x) {
    const float e = expf(-fabsf(x));
    return x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
}
__device__ __forceinline__ float stable_softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

// group grp of G lanes takes sample w * (32/G) + grp; lane `sub` holds columns 4 sub .. 4 sub + 3 of its two rows
template <int KIND, int G>
__global__ void __launch_bounds__(256) pointwise_step_kernel(const float *__restrict__ P, const float *__restrict__ Q, int64_t ld, int f4,
                                                             const float *__restrict__ bu, const float *__restrict__ bi,
                                                             const int32_t *__restrict__ u, const int32_t *__restrict__ it,
                                                             const float *__restrict__ label, int64_t n, float invn, float alpha,
                                                             float lambda, float *dP, float *dQ, float *dbi, double *loss) {
    const int lane = threadIdx.x & 31, sub = lane % G, grp = lane / G;
    const bool on = sub < f4;
    constexpr int PER = 32 / G;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    double acc_loss = 0.0;
    for (; w * PER < n; w += nw) {                                        // warp-uniform trip count: every lane shuffles
        const int64_t s = w * PER + grp;
        const bool live = s < n;
        const int64_t uu = live ? u[s] : 0, ii = live ? it[s] : 0;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f), q = p;
        if (live && on) {
            p = pw_ld4(P + uu * ld + sub * 4);
            q = pw_ld4(Q + ii * ld + sub * 4);
        }
        float dot = pw_dot(p, q), sq = KIND == LMF_LOGPOST ? pw_dot(p, p) + pw_dot(q, q) : 0.f;
#pragma unroll
        for (int off = G / 2; off > 0; off >>= 1) {
            dot += __shfl_xor_sync(0xffffffffu, dot, off);
            if (KIND == LMF_LOGPOST) sq += __shfl_xor_sync(0xffffffffu, sq, off);
        }
        if (!live) continue;
        const float y = label[s];
        if (KIND == PMF_MSE) {
            const float o = stable_sigmoid(dot), d = o - y;
            const float e = 2.f * d * invn * (o * (1.f - o));              // d (mean_B (sigmoid(x) - y)^2) / d x
            if (sub == 0) acc_loss += (double)d * (double)d * (double)invn;
            if (on) {
                red_add_v4(dQ + ii * ld + sub * 4, pw_scale(p, e));
                red_add_v4(dP + uu * ld + sub * 4, pw_scale(q, e));
            }
        } else {
            const float x = dot + __ldg(bu + uu) + __ldg(bi + ii), ay = alpha * y;
            const float c = stable_sigmoid(x) * (1.f + ay) - ay;            // d (-(a y x - (1 + a y) softplus(x))) / d x
            if (sub == 0) {
                acc_loss += -((double)ay * (double)x - (1.0 + (double)ay) * (double)stable_softplus(x)) + 0.5 * (double)lambda * (double)sq;
                red_add_f32(dbi + ii, c);
            }
            if (on) red_add_v4(dQ + ii * ld + sub * 4, pw_axpy(c, p, lambda, q));
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc_loss += __shfl_xor_sync(0xffffffffu, acc_loss, off);
    if (loss && lane == 0 && acc_loss != 0.0) atomicAdd(loss, acc_loss);
}

// one warp per listed row; lane 0 claims the row by swapping in this step's stamp: of all the warps holding the same row
// exactly one sees a different stamp come back (stamps only grow, and every claim this step writes `step`), and only it
// reads, updates and clears the row
__global__ void __launch_bounds__(256) adagrad_rows_kernel(float *__restrict__ var, float *__restrict__ acc, float *__restrict__ grad,
                                                           int64_t ld, int width, float *__restrict__ bvar, float *__restrict__ bacc,
                                                           float *__restrict__ bgrad, const int32_t *__restrict__ rows, int64_t n,
                                                           unsigned long long *__restrict__ stamp, unsigned long long step, float lr,
                                                           float eps) {
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (; w < n; w += nw) {
        const int64_t r = rows[w];
        int mine = 0;
        if (lane == 0) mine = atomicExch(stamp + r, step) != step;
        if (!__shfl_sync(0xffffffffu, mine, 0)) continue;
        for (int c = lane; c < width; c += 32) {                          // acc += g^2; var -= lr g / (sqrt(acc) + eps)
            const int64_t e = r * ld + c;
            const float g = grad[e], a = acc[e] + g * g;
            acc[e] = a;
            var[e] -= g * lr / (sqrtf(a) + eps);
            grad[e] = 0.f;
        }
        if (bvar && lane == 0) {
            const float g = bgrad[r], a = bacc[r] + g * g;
            bacc[r] = a;
            bvar[r] -= g * lr / (sqrtf(a) + eps);
            bgrad[r] = 0.f;
        }
    }
}

__global__ void __launch_bounds__(256) rating_labels_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                            const float *__restrict__ ratings, const int32_t *__restrict__ u,
                                                            const int32_t *__restrict__ it, float *__restrict__ label, int64_t n) {
    for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += (int64_t)gridDim.x * blockDim.x) {
        if (label[s] == 0.f) continue;                                    // a negative keeps its 0
        int64_t lo = __ldg(indptr + u[s]), hi = __ldg(indptr + u[s] + 1);
        const int32_t key = it[s];
        while (lo < hi) {                                                 // first entry >= key; a positive is in the row
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg(indices + mid) < key) lo = mid + 1; else hi = mid;
        }
        label[s] = __ldg(ratings + lo);
    }
}

__global__ void __launch_bounds__(256) sigmoid_scores_kernel(float *x, int64_t n) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const float v = x[e];
        if (v != -CUDART_INF_F) x[e] = 1.f / (1.f + __expf(-v));           // the same map as eb_sigmoid_inplace; NaN stays NaN
    }
}

static inline unsigned pw_grid(int64_t threads) {
    int64_t g = (threads + 255) / 256; const int64_t cap = (int64_t)sm_count() * 8;
    return (unsigned)(g > cap ? cap : (g < 1 ? 1 : g));
}

static inline int pw_lanes(int f) {
    int G = 1;
    while (G < f / 4) G <<= 1;
    return G;
}

template <int KIND>
static void launch_step(int G, int64_t n, cudaStream_t st, const float *P, const float *Q, int64_t ld, int f4, const float *bu,
                        const float *bi, const int32_t *u, const int32_t *it, const float *label, float invn, float alpha,
                        float lambda, float *dP, float *dQ, float *dbi, double *loss) {
    const unsigned grid = pw_grid((n + 32 / G - 1) / (32 / G) * 32);
#define EB_PW_STEP(GG) pointwise_step_kernel<KIND, GG><<<grid, 256, 0, st>>>(P, Q, ld, f4, bu, bi, u, it, label, n, invn, alpha, lambda, dP, dQ, dbi, loss)
    switch (G) {
    case 1: EB_PW_STEP(1); break;
    case 2: EB_PW_STEP(2); break;
    case 4: EB_PW_STEP(4); break;
    case 8: EB_PW_STEP(8); break;
    case 16: EB_PW_STEP(16); break;
    default: EB_PW_STEP(32); break;
    }
#undef EB_PW_STEP
}

}  // namespace eb

using namespace eb;

extern "C" int eb_pointwise_mf_step_f32(const float *P, const float *Q, int64_t ld, int f, const float *bu, const float *bi,
                                        const int32_t *u, const int32_t *it, const float *label, int64_t n, int kind,
                                        int64_t mean_over, float alpha, float lambda, float *dP, float *dQ, float *dbi,
                                        double *loss, void *stream) {
    EB_ARG(P && Q && u && it && label && dQ && n >= 0, "null pointer or n < 0");
    EB_ARG(f >= 4 && f % 4 == 0 && f <= 128 && ld >= f && ld % 4 == 0, "f must be a multiple of 4, <= 128, with ld >= f a multiple of 4");
    EB_ARG(kind == PMF_MSE || kind == LMF_LOGPOST, "kind=%d must be 0 (PMF) or 1 (LMF)", kind);
    EB_ARG(kind != PMF_MSE || (dP && mean_over >= 1), "PMF needs dP and mean_over >= 1");
    EB_ARG(kind != LMF_LOGPOST || (bu && bi && dbi && !dP), "LMF needs bu, bi and dbi, and updates no user row (dP NULL)");
    if (n == 0) return EB_OK;
    const cudaStream_t st = (cudaStream_t)stream;
    const float invn = kind == PMF_MSE ? 1.f / (float)mean_over : 1.f;
    if (kind == PMF_MSE)
        launch_step<PMF_MSE>(pw_lanes(f), n, st, P, Q, ld, f / 4, bu, bi, u, it, label, invn, alpha, lambda, dP, dQ, dbi, loss);
    else
        launch_step<LMF_LOGPOST>(pw_lanes(f), n, st, P, Q, ld, f / 4, bu, bi, u, it, label, invn, alpha, lambda, dP, dQ, dbi, loss);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_adagrad_rows_f32(float *var, float *acc, float *grad, int64_t ld, int width, float *bvar, float *bacc, float *bgrad,
                                   const int32_t *rows, int64_t n, uint64_t *stamp, uint64_t step, float lr, float eps, void *stream) {
    EB_ARG(var && acc && grad && rows && stamp && n >= 0 && width >= 1 && ld >= width, "null pointer or bad shape");
    EB_ARG((bvar == nullptr) == (bacc == nullptr) && (bvar == nullptr) == (bgrad == nullptr), "bias: var, acc and grad together");
    EB_ARG(step >= 1, "step stamps start at 1 (the stamp table starts at 0)");
    if (n == 0) return EB_OK;
    adagrad_rows_kernel<<<pw_grid(n * 32), 256, 0, (cudaStream_t)stream>>>(var, acc, grad, ld, width, bvar, bacc, bgrad, rows, n,
                                                                          reinterpret_cast<unsigned long long *>(stamp),
                                                                          (unsigned long long)step, lr, eps);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_rating_labels_f32(const int64_t *indptr, const int32_t *indices, const float *ratings, const int32_t *u,
                                    const int32_t *it, float *label, int64_t n, void *stream) {
    EB_ARG(indptr && indices && ratings && u && it && label && n >= 0, "null pointer or n < 0");
    if (n == 0) return EB_OK;
    rating_labels_kernel<<<pw_grid(n), 256, 0, (cudaStream_t)stream>>>(indptr, indices, ratings, u, it, label, n);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_sigmoid_scores_f32(float *x, int64_t n, void *stream) {
    EB_ARG(x && n >= 0, "null pointer or n < 0");
    if (n == 0) return EB_OK;
    sigmoid_scores_kernel<<<pw_grid(n), 256, 0, (cudaStream_t)stream>>>(x, n);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
