// rating_mf.cu — SVD++ and FunkSVD (latent_factor_models/SVDpp/svdpp_model.py, FunkSVD/funk_svd_model.py) and the pair
// pass behind MAE / MSE / RMSE (evaluation/metrics/rating/{mae,mse,rmse}).
//
//   eb_implicit_mean_f32     Z[r] = P[u_r] + (1/|N(u_r)|) sum_{j in N(u_r)} Y[j] over a list of users (N = train row): the
//                            SVD++ user vector, for a training batch or for every user before scoring
//   eb_rating_mf_step_f32    ONE fused kernel per batch: gather -> predict (z.q + b_u + b_i [+ g]) -> squared error -> loss ->
//                            vector-atomic scatter of dQ, dP, db_u, db_i, dg and, for SVD++, dY_j += e q / |N(u)| over the
//                            user's train row; the dense Keras Adam (eb_adam_dense_f32) follows.  b_u / b_i are
//                            optional (MF has neither)
//   eb_score_pairs_f32       the score of every (user, relevant item) entry of a CSR: the values the user's full list
//                            gives those items (-inf for a train item), for the rating metrics
//   eb_add_row_offset_f32    adds b_u (+ g) to the top-k values: a per-user constant changes no ranking, so the scoring
//                            kernels rank z.q + b_i alone
//   eb_rating_error_sums_f64 sum |v - r| and sum (v - r)^2 over the entries of the pair pass, one CTA, fixed order
// Rows are float4 columns (f % 4 == 0, f <= 128).  A warp splits into 32 / G groups of G lanes (G = f/4 rounded up to a
// power of two): each group takes one train-row (or relevant-item) entry, so a short row still keeps the warp busy.
// TensorFlow parity is UNPINNED (oracle/rating_mf.py is the checker).
#include <math_constants.h>

#include "common.cuh"

namespace eb {

__device__ __forceinline__ float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 f4_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float f4_dot(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float4 ld4(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float4 shfl4(float4 v, int src) {
    return make_float4(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src), __shfl_sync(0xffffffffu, v.z, src),
                       __shfl_sync(0xffffffffu, v.w, src));
}

// one warp per output row; group g of G lanes sums the entries g, g + 32/G, ... of the row, lane `sub` of a group holds the
// columns 4 sub .. 4 sub + 3; the groups' partial sums are then added across the warp
template <int G>
__global__ void __launch_bounds__(256) implicit_mean_kernel(const float *__restrict__ P, const float *__restrict__ Y, int64_t ld, int f4,
                                                            const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                            const int32_t *__restrict__ users, int64_t n, float *__restrict__ Z,
                                                            int64_t ldz) {
    const int lane = threadIdx.x & 31, sub = lane % G, grp = lane / G;
    const bool on = sub < f4;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (; w < n; w += nw) {
        const int64_t u = users ? (int64_t)users[w] : w;
        const int64_t beg = __ldg(indptr + u), end = __ldg(indptr + u + 1);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (on)
            for (int64_t e = beg + grp; e < end; e += 32 / G) acc = f4_add(acc, ld4(Y + (int64_t)__ldg(indices + e) * ld + sub * 4));
#pragma unroll
        for (int off = 16; off >= G; off >>= 1)
            acc = make_float4(acc.x + __shfl_xor_sync(0xffffffffu, acc.x, off), acc.y + __shfl_xor_sync(0xffffffffu, acc.y, off),
                              acc.z + __shfl_xor_sync(0xffffffffu, acc.z, off), acc.w + __shfl_xor_sync(0xffffffffu, acc.w, off));
        if (grp == 0 && on) {
            const float inv = end > beg ? 1.f / (float)(end - beg) : 0.f;
            *reinterpret_cast<float4 *>(Z + w * ldz + sub * 4) = f4_add(ld4(P + u * ld + sub * 4), f4_scale(acc, inv));
        }
    }
}

// one warp per sample: lane c < f/4 holds columns 4c .. 4c + 3 of the user vector z and the item row q; the train-row
// scatter of SVD++ regroups the lanes as implicit_mean_kernel does
template <int G>
__global__ void __launch_bounds__(256) step_kernel(const float *__restrict__ P, const float *__restrict__ Q, int64_t ld, int f4,
                                                   const float *__restrict__ bu, const float *__restrict__ bi, const float *__restrict__ g,
                                                   const float *__restrict__ Z, int64_t ldz, const int64_t *__restrict__ indptr,
                                                   const int32_t *__restrict__ indices, const int32_t *__restrict__ u,
                                                   const int32_t *__restrict__ it, const float *__restrict__ label, int64_t n, float invn,
                                                   float *dP, float *dQ, float *dY, float *dbu, float *dbi, float *dg, double *loss) {
    const int lane = threadIdx.x & 31, sub = lane % G, grp = lane / G;
    const bool on = lane < f4;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float gv = g ? __ldg(g) : 0.f;
    float acc_g = 0.f;
    double acc_loss = 0.0;
    for (; w < n; w += nw) {
        const int64_t uu = u[w], ii = it[w];
        float4 z = make_float4(0.f, 0.f, 0.f, 0.f), q = z;
        if (on) {
            z = Z ? ld4(Z + w * ldz + lane * 4) : ld4(P + uu * ld + lane * 4);
            q = ld4(Q + ii * ld + lane * 4);
        }
        float part = f4_dot(z, q);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
        const float d = part + (bu ? __ldg(bu + uu) : 0.f) + (bi ? __ldg(bi + ii) : 0.f) + gv - label[w];
        const float e = 2.f * d * invn;                                   // d (mean_B (out - y)^2) / d out
        if (lane == 0) {
            acc_loss += (double)d * (double)d;
            if (dbu) red_add_f32(dbu + uu, e);
            if (dbi) red_add_f32(dbi + ii, e);
            acc_g += e;
        }
        if (on) {
            red_add_v4(dQ + ii * ld + lane * 4, f4_scale(z, e));
            red_add_v4(dP + uu * ld + lane * 4, f4_scale(q, e));
        }
        if (dY) {
            const int64_t beg = __ldg(indptr + uu), end = __ldg(indptr + uu + 1);
            const float4 s = f4_scale(shfl4(q, sub), e / (float)(end - beg));
            if (sub < f4)
                for (int64_t k = beg + grp; k < end; k += 32 / G) red_add_v4(dY + (int64_t)__ldg(indices + k) * ld + sub * 4, s);
        }
    }
    if (dg && lane == 0 && acc_g != 0.f) red_add_f32(dg, acc_g);
    if (loss && lane == 0 && acc_loss != 0.0) atomicAdd(loss, acc_loss * (double)invn);
}

// one warp per user; group g of G lanes scores the relevant entries g, g + 32/G, ... of the user's row
template <int G>
__global__ void __launch_bounds__(256) score_pairs_kernel(const float *__restrict__ U, const float *__restrict__ V, int64_t ld, int f4,
                                                          const float *__restrict__ item_bias, const float *__restrict__ user_off,
                                                          const float *__restrict__ global_off, const int64_t *__restrict__ rel_indptr,
                                                          const int32_t *__restrict__ rel_items, int64_t n_users,
                                                          const int64_t *__restrict__ mask_indptr, const int32_t *__restrict__ mask_indices,
                                                          float *__restrict__ out) {
    const int lane = threadIdx.x & 31, sub = lane % G, grp = lane / G;
    const bool on = sub < f4;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const float go = global_off ? __ldg(global_off) : 0.f;
    for (; w < n_users; w += nw) {
        const int64_t beg = __ldg(rel_indptr + w), end = __ldg(rel_indptr + w + 1);
        if (beg == end) continue;
        const float4 x = on ? ld4(U + w * ld + sub * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float off = user_off ? __ldg(user_off + w) + go : go;
        const int32_t *mrow = mask_indptr ? mask_indices + __ldg(mask_indptr + w) : nullptr;
        const int mlen = mask_indptr ? (int)(__ldg(mask_indptr + w + 1) - __ldg(mask_indptr + w)) : 0;
        for (int64_t k0 = beg; k0 < end; k0 += 32 / G) {                // warp-uniform trip count: every lane shuffles
            const int64_t k = k0 + grp;
            const int32_t item = k < end ? __ldg(rel_items + k) : -1;
            float part = (on && item >= 0) ? f4_dot(x, ld4(V + (int64_t)item * ld + sub * 4)) : 0.f;
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
            if (k < end && sub == 0) {
                float s = CUDART_NAN_F;                                    // outside the catalogue: never in a list
                if (item >= 0) {
                    if (mrow && contains_sorted(mrow, mlen, item)) s = -CUDART_INF_F;
                    else s = (part + (item_bias ? __ldg(item_bias + item) : 0.f)) + off;
                }
                out[k] = s;
            }
        }
    }
}

__global__ void __launch_bounds__(256) add_row_offset_kernel(float *x, int64_t rows, int cols, int64_t ldx, const float *__restrict__ row_off,
                                                             const float *__restrict__ scalar_off) {
    const float so = scalar_off ? __ldg(scalar_off) : 0.f;
    const int64_t total = rows * cols;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / cols;
        x[r * ldx + (e - r * cols)] += __ldg(row_off + r) + so;          // -inf (no candidate) stays -inf
    }
}

constexpr int SUMS_NT = 512;

// one CTA: thread t sums the entries t, t + SUMS_NT, ... then a fixed tree adds the threads (the same bits every run)
__global__ void __launch_bounds__(SUMS_NT) error_sums_kernel(const float *__restrict__ scores, const double *__restrict__ ratings,
                                                             const int32_t *__restrict__ items, int64_t n, double *__restrict__ out) {
    __shared__ double sa[SUMS_NT], sq[SUMS_NT];
    double a = 0.0, q = 0.0;
    for (int64_t e = threadIdx.x; e < n; e += SUMS_NT) {
        if (__ldg(items + e) < 0) continue;                               // outside the catalogue: no list holds it
        const double d = (double)__ldg(scores + e) - __ldg(ratings + e);
        a += fabs(d);
        q += d * d;
    }
    sa[threadIdx.x] = a; sq[threadIdx.x] = q;
    __syncthreads();
    for (int s = SUMS_NT / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) { sa[threadIdx.x] += sa[threadIdx.x + s]; sq[threadIdx.x] += sq[threadIdx.x + s]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { out[0] = sa[0]; out[1] = sq[0]; }
}

static inline unsigned warp_grid(int64_t warps) {
    int64_t g = (warps * 32 + 255) / 256; const int64_t cap = (int64_t)sm_count() * 8;
    return (unsigned)(g > cap ? cap : (g < 1 ? 1 : g));
}

// lanes per group: f/4 rounded up to a power of two
static inline int lanes_for(int f) {
    int G = 1;
    while (G < f / 4) G <<= 1;
    return G;
}

#define EB_LANES_DISPATCH(G, KERNEL, ...)                                                                 \
    switch (G) {                                                                                         \
    case 1: KERNEL<1><<<__VA_ARGS__; break;                                                              \
    case 2: KERNEL<2><<<__VA_ARGS__; break;                                                              \
    case 4: KERNEL<4><<<__VA_ARGS__; break;                                                              \
    case 8: KERNEL<8><<<__VA_ARGS__; break;                                                              \
    case 16: KERNEL<16><<<__VA_ARGS__; break;                                                            \
    default: KERNEL<32><<<__VA_ARGS__; break;                                                            \
    }

static inline bool rows_ok(int f, int64_t ld) { return f >= 4 && f % 4 == 0 && f <= 128 && ld >= f && ld % 4 == 0; }

}  // namespace eb

using namespace eb;

extern "C" int eb_implicit_mean_f32(const float *P, const float *Y, int64_t ld, int f, const int64_t *indptr, const int32_t *indices,
                                    const int32_t *users, int64_t n, float *Z, int64_t ldz, void *stream) {
    EB_ARG(P && Y && indptr && indices && Z && n >= 0, "null pointer or n < 0");
    EB_ARG(rows_ok(f, ld) && ldz >= f && ldz % 4 == 0, "f must be a multiple of 4, <= 128, with ld, ldz >= f multiples of 4");
    if (n == 0) return EB_OK;
    EB_LANES_DISPATCH(lanes_for(f), implicit_mean_kernel, warp_grid(n), 256, 0, (cudaStream_t)stream>>>(P, Y, ld, f / 4, indptr, indices,
                                                                                                         users, n, Z, ldz));
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_rating_mf_step_f32(const float *P, const float *Q, int64_t ld, int f, const float *bu, const float *bi, const float *g,
                                     const float *Z, int64_t ldz, const int64_t *indptr, const int32_t *indices, const int32_t *u,
                                     const int32_t *it, const float *label, int64_t n, int64_t mean_over, float *dP, float *dQ,
                                     float *dY, float *dbu, float *dbi, float *dg, double *loss, void *stream) {
    EB_ARG(P && Q && u && it && label && dP && dQ, "null pointer");
    EB_ARG((bu == nullptr) == (dbu == nullptr) && (bi == nullptr) == (dbi == nullptr), "bu and dbu, bi and dbi go together");
    EB_ARG(rows_ok(f, ld) && mean_over >= 1 && n >= 0, "f must be a multiple of 4, <= 128, with ld >= f a multiple of 4");
    EB_ARG((g == nullptr) == (dg == nullptr), "g and dg go together");
    EB_ARG((Z == nullptr) == (dY == nullptr), "Z (the batch's implicit means) and dY go together");
    EB_ARG(!dY || (indptr && indices && ldz >= f && ldz % 4 == 0), "SVD++ needs the train CSR and ldz >= f");
    if (n == 0) return EB_OK;
    EB_LANES_DISPATCH(lanes_for(f), step_kernel, warp_grid(n), 256, 0, (cudaStream_t)stream>>>(P, Q, ld, f / 4, bu, bi, g, Z, ldz, indptr,
                                                                                                indices, u, it, label, n,
                                                                                                1.f / (float)mean_over, dP, dQ, dY,
                                                                                                dbu, dbi, dg, loss));
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_score_pairs_f32(const float *U, const float *V, int64_t ld, int f, const float *item_bias, const float *user_off,
                                  const float *global_off, const int64_t *rel_indptr, const int32_t *rel_items, int32_t n_users,
                                  const int64_t *mask_indptr, const int32_t *mask_indices, float *out, void *stream) {
    EB_ARG(U && V && rel_indptr && rel_items && out && n_users >= 0, "null pointer or n_users < 0");
    EB_ARG(rows_ok(f, ld), "f must be a multiple of 4, <= 128, with ld >= f a multiple of 4");
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both parts or neither");
    if (n_users == 0) return EB_OK;
    EB_LANES_DISPATCH(lanes_for(f), score_pairs_kernel, warp_grid(n_users), 256, 0, (cudaStream_t)stream>>>(
        U, V, ld, f / 4, item_bias, user_off, global_off, rel_indptr, rel_items, n_users, mask_indptr, mask_indices, out));
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_add_row_offset_f32(float *x, int64_t rows, int cols, int64_t ldx, const float *row_off, const float *scalar_off,
                                     void *stream) {
    EB_ARG(x && row_off && rows >= 0 && cols >= 0 && ldx >= cols, "bad argument");
    if (rows == 0 || cols == 0) return EB_OK;
    add_row_offset_kernel<<<capped_grid(rows * cols), 256, 0, (cudaStream_t)stream>>>(x, rows, cols, ldx, row_off, scalar_off);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_rating_error_sums_f64(const float *scores, const double *ratings, const int32_t *items, int64_t n, double *out,
                                        void *stream) {
    EB_ARG(scores && ratings && items && out && n >= 0, "bad argument");
    error_sums_kernel<<<1, SUMS_NT, 0, (cudaStream_t)stream>>>(scores, ratings, items, n, out);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
