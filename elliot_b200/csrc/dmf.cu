// dmf.cu — the non-GEMM pieces of DMF (elliot/recommender/neural/DMF/deep_matrix_factorization_model.py).
//
//   eb_dmf_sparse_fwd_f32      h1 = act(X[rows] . W1 + b1) for rows of the train rating matrix (CSR for the user tower,
//                              CSC for the item tower), X holding the rating VALUES (model.py:46-52 feeds dense rating
//                              rows through frozen embeddings; the dense row is never built here)
//   eb_dmf_sparse_bwd_f32      dW1 += X[rows]^T . dpre1 (vector atomics)
//   eb_dmf_head_f32            the whole head of train_step (:76-77, 93-105) for one batch, with no host synchronisation:
//                              tf.nn.l2_normalize(x, 0) of both tower outputs (each factor COLUMN over the batch), the
//                              row sums of their product, Keras BinaryCrossentropy (in float32: clip to [1e-7, 1 - 1e-7], log(p + 1e-7),
//                              batch mean; the loss summed in fp64) and the gradients back through both normalisations
//   eb_dmf_score_operands_f32  U^ for every user block and V^ for every item (get_recs, :106-121) so that the dot-product
//                              scorers rank U^ . V^ with no scoring kernel of their own
// Dense hidden layers go through eb_gemm_bf16_tn / eb_gemm_bf16 (gemm_tc.cu).  Column reductions run in fp64 in a fixed
// order (chunks of rows, then the chunks in index order), so a batch's result does not depend on scheduling.
#include "common.cuh"

namespace eb {

constexpr int DMF_MAX_F = 256;
constexpr int DMF_MAX_CHUNKS = 1024;
constexpr double L2_EPS = 1e-12;      // tf.nn.l2_normalize's epsilon
constexpr float BCE_EPS = 1e-7f;      // keras.backend.epsilon()

// One CTA per batch row: thread t takes the 4 columns 4 (t % G) (G = H / 4) of the row's entries t / G, t / G + S, ...
// (S = 256 / G slices), so a long row (the most rated item's column holds 42 790 users at the bench's ML-20M shape) is read by every
// thread of the CTA, not by one.  The slices' partial sums are added in slice order: the result does not depend on
// scheduling.
constexpr int SPARSE_THREADS = 256;

__global__ void __launch_bounds__(SPARSE_THREADS) dmf_sparse_fwd_kernel(const float *__restrict__ W1, const float *__restrict__ b1,
                                                                        int H, const int64_t *__restrict__ indptr,
                                                                        const int32_t *__restrict__ indices,
                                                                        const float *__restrict__ values,
                                                                        const int32_t *__restrict__ rows, int relu,
                                                                        float *__restrict__ h1, int64_t ldh) {
    __shared__ float4 part[SPARSE_THREADS];
    const int G = H / 4, S = SPARSE_THREADS / G;
    const int c = threadIdx.x % G, sl = threadIdx.x / G;
    const int64_t b = blockIdx.x;
    const int r = __ldg(rows + b);
    const int64_t beg = __ldg(indptr + r), end = __ldg(indptr + r + 1);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (sl < S) {
        for (int64_t p = beg + sl; p < end; p += S) {
            const float x = __ldg(values + p);
            const float4 w = __ldg(reinterpret_cast<const float4 *>(W1 + (int64_t)__ldg(indices + p) * H + 4 * c));
            acc.x = fmaf(x, w.x, acc.x); acc.y = fmaf(x, w.y, acc.y); acc.z = fmaf(x, w.z, acc.z); acc.w = fmaf(x, w.w, acc.w);
        }
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x < G) {
        float4 o = *reinterpret_cast<const float4 *>(b1 + 4 * c);
        for (int k = 0; k < S; k++) {
            const float4 q = part[k * G + c];
            o.x += q.x; o.y += q.y; o.z += q.z; o.w += q.w;
        }
        if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
        *reinterpret_cast<float4 *>(h1 + b * ldh + 4 * c) = o;
    }
}

// the same split of the row's entries; each entry's row of dW1 gets values[p] dpre1[b] by a vector atomic
__global__ void __launch_bounds__(SPARSE_THREADS) dmf_sparse_bwd_kernel(float *__restrict__ dW1, int H,
                                                                        const int64_t *__restrict__ indptr,
                                                                        const int32_t *__restrict__ indices,
                                                                        const float *__restrict__ values,
                                                                        const int32_t *__restrict__ rows,
                                                                        const float *__restrict__ dpre1, int64_t ldd) {
    const int G = H / 4, S = SPARSE_THREADS / G;
    const int c = threadIdx.x % G, sl = threadIdx.x / G;
    if (sl >= S) return;
    const int64_t b = blockIdx.x;
    const int r = __ldg(rows + b);
    const int64_t beg = __ldg(indptr + r), end = __ldg(indptr + r + 1);
    const float4 g = *reinterpret_cast<const float4 *>(dpre1 + b * ldd + 4 * c);
    for (int64_t p = beg + sl; p < end; p += S) {
        const float x = __ldg(values + p);
        red_add_v4(dW1 + (int64_t)__ldg(indices + p) * H + 4 * c, make_float4(x * g.x, x * g.y, x * g.z, x * g.w));
    }
}

// ---------------------------------------------------------------- head
struct HeadParams {
    const float *U, *V;          // tower outputs [B][ld]
    int64_t ld, B;
    int F, cosine, n_chunks;
    int64_t rows_per_chunk;
    const float *label;
    float inv_max;
    double *part;                // [n_chunks][2F] column partials; [n_chunks] loss partials after them
    float *norm;                 // [4F]: inv_u, inv_v, flag_u, flag_v (flag 1: the sum of squares passed the floor)
    double *colsum;              // [F]: sum_b g_b u^_bf v^_bf
    float *g;                    // [B] dloss/doutput
    float *prob;                 // optional [B] outputs
    double *loss;
    float *dU, *dV;
    int64_t ldg;
};

// per chunk: column partials of sum u^2 and sum v^2, warps in a fixed order
__global__ void __launch_bounds__(256) dmf_colsq_kernel(const HeadParams p) {
    __shared__ double sm[8][2 * DMF_MAX_F];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, F = p.F;
    const int64_t r0 = blockIdx.x * p.rows_per_chunk;
    const int64_t r1 = min(r0 + p.rows_per_chunk, p.B);
    double au[DMF_MAX_F / 32], av[DMF_MAX_F / 32];
#pragma unroll
    for (int k = 0; k < DMF_MAX_F / 32; k++) au[k] = av[k] = 0.0;
    for (int64_t b = r0 + warp; b < r1; b += 8) {
#pragma unroll
        for (int k = 0; k < DMF_MAX_F / 32; k++) {
            const int f = lane + 32 * k;
            if (f < F) {
                const double u = p.U[b * p.ld + f], v = p.V[b * p.ld + f];
                au[k] += u * u; av[k] += v * v;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < DMF_MAX_F / 32; k++) {
        const int f = lane + 32 * k;
        if (f < F) { sm[warp][f] = au[k]; sm[warp][F + f] = av[k]; }
    }
    __syncthreads();
    for (int f = threadIdx.x; f < 2 * F; f += blockDim.x) {
        double s = 0.0;
        for (int w = 0; w < 8; w++) s += sm[w][f];
        p.part[(int64_t)blockIdx.x * 2 * F + f] = s;
    }
}

// one CTA: the column norms (which = 0) or the column sums of g u^ v^ and the loss (which = 1), chunks in index order
__global__ void __launch_bounds__(256) dmf_colfinish_kernel(const HeadParams p, int which) {
    const int F = p.F;
    if (which == 0) {
        for (int f = threadIdx.x; f < 2 * F; f += blockDim.x) {
            double s = 0.0;
            for (int c = 0; c < p.n_chunks; c++) s += p.part[(int64_t)c * 2 * F + f];
            p.norm[f] = (float)(1.0 / sqrt(s > L2_EPS ? s : L2_EPS));
            p.norm[2 * F + f] = s >= L2_EPS ? 1.f : 0.f;          // Maximum's gradient goes to x where x >= y
        }
    } else {
        for (int f = threadIdx.x; f < F; f += blockDim.x) {
            double s = 0.0;
            for (int c = 0; c < p.n_chunks; c++) s += p.part[(int64_t)c * 2 * F + f];
            p.colsum[f] = s;
        }
        if (threadIdx.x == 0) {
            double s = 0.0;
            const double *lp = p.part + (int64_t)p.n_chunks * 2 * F;
            for (int c = 0; c < p.n_chunks; c++) s += lp[c];
            *p.loss += s / (double)p.B;
        }
    }
}

// per row: the output, the clipped BCE term and its gradient g_b; per chunk: sum_b g_b u^ v^ per column and the loss sum
__global__ void __launch_bounds__(256) dmf_out_kernel(const HeadParams p) {
    __shared__ double sm[8][DMF_MAX_F];
    __shared__ double sl[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, F = p.F;
    const int64_t r0 = blockIdx.x * p.rows_per_chunk;
    const int64_t r1 = min(r0 + p.rows_per_chunk, p.B);
    double ac[DMF_MAX_F / 32];
    double al = 0.0;
#pragma unroll
    for (int k = 0; k < DMF_MAX_F / 32; k++) ac[k] = 0.0;
    for (int64_t b = r0 + warp; b < r1; b += 8) {
        float uv[DMF_MAX_F / 32];
        float o = 0.f;
#pragma unroll
        for (int k = 0; k < DMF_MAX_F / 32; k++) {
            const int f = lane + 32 * k;
            uv[k] = 0.f;
            if (f < F) {
                float u = p.U[b * p.ld + f], v = p.V[b * p.ld + f];
                if (p.cosine) { u *= p.norm[f]; v *= p.norm[F + f]; }
                uv[k] = u * v;
                o += uv[k];
            }
        }
#pragma unroll
        for (int s = 16; s >= 1; s >>= 1) o += __shfl_xor_sync(0xffffffffu, o, s);
        const float y = p.label[b] * p.inv_max;
        const float pc = fminf(fmaxf(o, BCE_EPS), 1.f - BCE_EPS);
        const double pe = (double)pc + (double)BCE_EPS, qe = 1.0 - (double)pc + (double)BCE_EPS;
        const bool pass = o >= BCE_EPS && o <= 1.f - BCE_EPS;     // clip_by_value passes the gradient on the closed interval
        const float g = pass ? (float)(-((double)y / pe - (1.0 - (double)y) / qe) / (double)p.B) : 0.f;
        if (lane == 0) {
            al += -((double)y * log(pe) + (1.0 - (double)y) * log(qe));
            p.g[b] = g;
            if (p.prob) p.prob[b] = o;
        }
        if (p.cosine) {
#pragma unroll
            for (int k = 0; k < DMF_MAX_F / 32; k++) ac[k] += (double)g * (double)uv[k];
        }
    }
#pragma unroll
    for (int k = 0; k < DMF_MAX_F / 32; k++) {
        const int f = lane + 32 * k;
        if (f < F) sm[warp][f] = ac[k];
    }
    if (lane == 0) sl[warp] = al;
    __syncthreads();
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        double s = 0.0;
        for (int w = 0; w < 8; w++) s += sm[w][f];
        p.part[(int64_t)blockIdx.x * 2 * F + f] = s;
    }
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < 8; w++) s += sl[w];
        p.part[(int64_t)p.n_chunks * 2 * F + blockIdx.x] = s;
    }
}

// dx = n (dx^ - x^ sum_b x^ dx^) with n = 1/|x|, dx^ = g times the other side's x^; below the floor only n dx^
__global__ void __launch_bounds__(256) dmf_grad_kernel(const HeadParams p) {
    const int F = p.F;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < p.B * F; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = t / F;
        const int f = (int)(t - b * F);
        const float g = p.g[b];
        const float u = p.U[b * p.ld + f], v = p.V[b * p.ld + f];
        float du, dv;
        if (p.cosine) {
            const float nu = p.norm[f], nv = p.norm[F + f];
            const float uh = u * nu, vh = v * nv;
            const float c = (float)p.colsum[f];
            du = nu * (g * vh - (p.norm[2 * F + f] != 0.f ? uh * c : 0.f));
            dv = nv * (g * uh - (p.norm[3 * F + f] != 0.f ? vh * c : 0.f));
        } else {
            du = g * v;
            dv = g * u;
        }
        p.dU[b * p.ldg + f] = du;
        p.dV[b * p.ldg + f] = dv;
    }
}

static int head_chunks(int64_t B, int64_t &rows_per_chunk) {
    int64_t n = (B + 7) / 8;
    if (n > DMF_MAX_CHUNKS) n = DMF_MAX_CHUNKS;
    if (n < 1) n = 1;
    rows_per_chunk = (B + n - 1) / n;
    return (int)((B + rows_per_chunk - 1) / rows_per_chunk);
}

struct HeadLayout {
    size_t part, norm, colsum, g, total;
};

static HeadLayout head_layout(int64_t B, int F) {
    int64_t rpc;
    const int nc = head_chunks(B, rpc);
    HeadLayout L;
    size_t off = 0;
    L.part = off; off += align_up(sizeof(double) * ((size_t)nc * 2 * F + nc));
    L.norm = off; off += align_up(sizeof(float) * 4 * F);
    L.colsum = off; off += align_up(sizeof(double) * F);
    L.g = off; off += align_up(sizeof(float) * (size_t)B);
    L.total = off;
    return L;
}

// ---------------------------------------------------------------- scoring operands
// one CTA per (user block, column): U^[u,f] = U[u,f] / sqrt(max(sum over the block of U[v,f]^2, 1e-12))
__global__ void __launch_bounds__(256) dmf_user_operand_kernel(const float *__restrict__ Uo, int64_t ldu, int F, int n_users,
                                                               int block, float *__restrict__ Uh, int64_t ld) {
    __shared__ double sm[256];
    const int ub = blockIdx.x / F, f = blockIdx.x - ub * F;
    const int64_t u0 = (int64_t)ub * block, u1 = min(u0 + block, (int64_t)n_users);
    double s = 0.0;
    for (int64_t u = u0 + threadIdx.x; u < u1; u += blockDim.x) {
        const double x = Uo[u * ldu + f];
        s += x * x;
    }
    sm[threadIdx.x] = s;
    __syncthreads();
    for (int w = 128; w >= 1; w >>= 1) {
        if (threadIdx.x < w) sm[threadIdx.x] += sm[threadIdx.x + w];
        __syncthreads();
    }
    const float inv = (float)(1.0 / sqrt(sm[0] > L2_EPS ? sm[0] : L2_EPS));
    for (int64_t u = u0 + threadIdx.x; u < u1; u += blockDim.x) Uh[u * ld + f] = Uo[u * ldu + f] * inv;
}

// V^[i,f] = V[i,f] / sqrt(max(B V[i,f]^2, 1e-12)): the B identical copies of item i's column in a block of B users;
// cosine = 0 copies.  Padding columns are zeroed.
__global__ void __launch_bounds__(256) dmf_item_operand_kernel(const float *__restrict__ Vo, int64_t ldv, int F, int n_items,
                                                               int64_t Bsz, int cosine, float *__restrict__ Vh, int64_t ld) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (int64_t)n_items * ld; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = t / ld;
        const int f = (int)(t - i * ld);
        float o = 0.f;
        if (f < F) {
            const float x = Vo[i * ldv + f];
            if (cosine) {
                const double ss = (double)Bsz * (double)x * (double)x;
                o = x * (float)(1.0 / sqrt(ss > L2_EPS ? ss : L2_EPS));
            } else {
                o = x;
            }
        }
        Vh[t] = o;
    }
}

__global__ void __launch_bounds__(256) dmf_copy_pad_kernel(const float *__restrict__ src, int64_t lds, int F, int64_t rows,
                                                           float *__restrict__ dst, int64_t ld) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < rows * ld; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / ld;
        const int f = (int)(t - r * ld);
        dst[t] = f < F ? src[r * lds + f] : 0.f;
    }
}

}  // namespace eb

using namespace eb;

extern "C" int eb_dmf_sparse_fwd_f32(const float *W1, const float *b1, int H, const int64_t *indptr, const int32_t *indices,
                                     const float *values, const int32_t *rows, int64_t B, int relu, float *h1, int64_t ldh,
                                     void *stream) {
    EB_ARG(W1 && b1 && indptr && indices && values && rows && h1, "null pointer");
    EB_ARG(H >= 4 && H <= 4 * SPARSE_THREADS && H % 4 == 0 && ldh >= H && ldh % 4 == 0,
           "H=%d must be a multiple of 4 in [4, %d] and ldh >= H", H, 4 * SPARSE_THREADS);
    EB_ARG(((uintptr_t)W1 % 16) == 0 && ((uintptr_t)b1 % 16) == 0 && ((uintptr_t)h1 % 16) == 0, "16-byte alignment");
    EB_ARG(B < INT32_MAX, "B=%lld rows exceed one grid", (long long)B);
    if (B <= 0) return EB_OK;
    dmf_sparse_fwd_kernel<<<(unsigned)B, SPARSE_THREADS, 0, (cudaStream_t)stream>>>(W1, b1, H, indptr, indices, values, rows,
                                                                                   relu, h1, ldh);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_dmf_sparse_bwd_f32(float *dW1, int H, const int64_t *indptr, const int32_t *indices, const float *values,
                                     const int32_t *rows, int64_t B, const float *dpre1, int64_t ldd, void *stream) {
    EB_ARG(dW1 && indptr && indices && values && rows && dpre1, "null pointer");
    EB_ARG(H >= 4 && H <= 4 * SPARSE_THREADS && H % 4 == 0 && ldd >= H && ldd % 4 == 0,
           "H=%d must be a multiple of 4 in [4, %d] and ldd >= H", H, 4 * SPARSE_THREADS);
    EB_ARG(((uintptr_t)dW1 % 16) == 0 && ((uintptr_t)dpre1 % 16) == 0, "16-byte alignment");
    EB_ARG(B < INT32_MAX, "B=%lld rows exceed one grid", (long long)B);
    if (B <= 0) return EB_OK;
    dmf_sparse_bwd_kernel<<<(unsigned)B, SPARSE_THREADS, 0, (cudaStream_t)stream>>>(dW1, H, indptr, indices, values, rows, dpre1,
                                                                                   ldd);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" size_t eb_dmf_head_workspace_bytes(int64_t B, int F) {
    if (F < 1 || F > DMF_MAX_F) return 0;
    return head_layout(B < 1 ? 1 : B, F).total;
}

extern "C" int eb_dmf_head_f32(const float *U, const float *V, int64_t ld, int F, int64_t B, const float *label, float max_rating,
                               int cosine, double *loss, float *dU, float *dV, int64_t ldg, float *prob, void *workspace,
                               size_t workspace_bytes, void *stream) {
    EB_ARG(U && V && label && loss && dU && dV, "null pointer");
    EB_ARG(F >= 1 && F <= DMF_MAX_F && ld >= F && ldg >= F, "need 1 <= F=%d <= %d, ld and ldg >= F", F, DMF_MAX_F);
    EB_ARG(max_rating > 0.f, "max_rating=%g must be positive", max_rating);
    if (B <= 0) return EB_OK;
    const HeadLayout L = head_layout(B, F);
    if (!workspace || workspace_bytes < L.total)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace_bytes, L.total);
    char *ws = (char *)workspace;
    HeadParams p;
    p.U = U; p.V = V; p.ld = ld; p.B = B; p.F = F; p.cosine = cosine ? 1 : 0;
    p.n_chunks = head_chunks(B, p.rows_per_chunk);
    p.label = label; p.inv_max = 1.f / max_rating;
    p.part = (double *)(ws + L.part); p.norm = (float *)(ws + L.norm); p.colsum = (double *)(ws + L.colsum);
    p.g = (float *)(ws + L.g); p.prob = prob; p.loss = loss; p.dU = dU; p.dV = dV; p.ldg = ldg;
    cudaStream_t st = (cudaStream_t)stream;
    if (p.cosine) {
        dmf_colsq_kernel<<<p.n_chunks, 256, 0, st>>>(p);
        dmf_colfinish_kernel<<<1, 256, 0, st>>>(p, 0);
    }
    dmf_out_kernel<<<p.n_chunks, 256, 0, st>>>(p);
    dmf_colfinish_kernel<<<1, 256, 0, st>>>(p, 1);
    dmf_grad_kernel<<<capped_grid(B * F), 256, 0, st>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_dmf_score_operands_f32(const float *Uo, int64_t ldu, const float *Vo, int64_t ldv, int F, int32_t n_users,
                                         int32_t n_items, int64_t block, int cosine, float *Uh, float *Vh, float *Vh_last,
                                         int64_t ld, void *stream) {
    EB_ARG(Uo && Vo && Uh && Vh, "null pointer");
    EB_ARG(F >= 1 && ldu >= F && ldv >= F && ld >= F, "need ldu, ldv, ld >= F=%d", F);
    EB_ARG(n_users >= 1 && n_items >= 1 && block >= 1, "bad sizes");
    const int64_t bl = block < n_users ? block : n_users;
    const int64_t last = n_users % bl;
    EB_ARG(!cosine || last == 0 || Vh_last, "a short last block needs Vh_last");
    cudaStream_t st = (cudaStream_t)stream;
    if (cosine) {
        const int64_t n_blocks = (n_users + bl - 1) / bl;
        EB_ARG(n_blocks * F < INT32_MAX, "too many user blocks");
        dmf_copy_pad_kernel<<<capped_grid((int64_t)n_users * ld), 256, 0, st>>>(Uo, ldu, F, n_users, Uh, ld);
        dmf_user_operand_kernel<<<(unsigned)(n_blocks * F), 256, 0, st>>>(Uo, ldu, F, n_users, (int)bl, Uh, ld);
        dmf_item_operand_kernel<<<capped_grid((int64_t)n_items * ld), 256, 0, st>>>(Vo, ldv, F, n_items, bl, 1, Vh, ld);
        if (last)
            dmf_item_operand_kernel<<<capped_grid((int64_t)n_items * ld), 256, 0, st>>>(Vo, ldv, F, n_items, last, 1, Vh_last, ld);
    } else {
        dmf_copy_pad_kernel<<<capped_grid((int64_t)n_users * ld), 256, 0, st>>>(Uo, ldu, F, n_users, Uh, ld);
        dmf_item_operand_kernel<<<capped_grid((int64_t)n_items * ld), 256, 0, st>>>(Vo, ldv, F, n_items, 1, 0, Vh, ld);
    }
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
