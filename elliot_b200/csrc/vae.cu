// vae.cu — the non-GEMM pieces of MultiVAE (elliot/recommender/autoencoders/vae/multi_vae_model.py).
//
//   eb_vae_embed_fwd      x_hat = l2_normalize(x) (rows are binary: 1/sqrt(nnz)); pre1 = x_hat W1 + b1; h1 = tanh(pre1)
//                         (multi_vae_model.py:42,44-47,57-59) — the B x I . I x 600 "GEMM" is a gather-sum
//                         over the user's train items, the dense B x I batch of sparse_sampler.py:25 is never built
//   eb_vae_reparam_fwd    z = mu + exp(lv/2) eps, eps ~ N(0,1) (Philox; multi_vae_model.py:20-29), KL sum (:119-121)
//   eb_vae_softmax_grad   row log-softmax, nll_b = -sum_i log_softmax_bi x_bi (:131-135), dlogits in place
//   eb_vae_reparam_bwd    d(mu|lv) from dz and the annealed KL term
//   eb_tanh_bwd           d_pre = d_out * (1 - out^2)
//   eb_colsum             bias gradients
//   eb_vae_embed_bwd      dW1[i,:] += d_pre1[b,:] / sqrt(nnz_b) for the user's items (vector atomics)
//   eb_dense_topk_f32     masked top-k on an existing dense score block (predict path, :144-159)
// Dense layers go through eb_gemm_bf16_tn (gemm_tc.cu).  tensorflow==2.3.2 cannot be executed in
// the build container: parity with TF is UNPINNED; checker = oracle/tf_models.py (fp64 numpy).
#include <math_constants.h>

#include <cuda_bf16.h>

#include "common.cuh"

namespace eb {

__device__ __forceinline__ void vred4(float *p, float4 v) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// one CTA per batch row; H columns (multiple of 4) processed as float4 by threads
__global__ void __launch_bounds__(256) vae_embed_fwd_kernel(const float *__restrict__ W1, const float *__restrict__ b1, int H,
                                                            const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                            const int32_t *__restrict__ rows, float *__restrict__ h1, int64_t ldh,
                                                            float drop_rate, uint64_t seed) {
    const int b = blockIdx.x;
    const int u = rows[b];
    const int64_t beg = indptr[u], end = indptr[u + 1];
    const float scale = end > beg ? rsqrtf((float)(end - beg)) : 0.f;
    const float keep_scale = drop_rate > 0.f ? 1.f / (1.f - drop_rate) : 1.f;
    for (int c4 = threadIdx.x; c4 * 4 < H; c4 += blockDim.x) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int64_t p = beg; p < end; p++) {
            if (drop_rate > 0.f) {       // Dropout on the normalised input (multi_vae_model.py:43,58): per (row, item) Bernoulli
                uint32_t r[4];
                Philox::gen(seed, (uint64_t)b, (uint32_t)(p - beg), r);
                if ((float)(r[0] >> 8) * (1.f / 16777216.f) < drop_rate) continue;
            }
            const float4 w = *reinterpret_cast<const float4 *>(W1 + (int64_t)indices[p] * H + c4 * 4);
            acc.x += w.x; acc.y += w.y; acc.z += w.z; acc.w += w.w;
        }
        const float s = scale * keep_scale;
        const float4 bb = *reinterpret_cast<const float4 *>(b1 + c4 * 4);
        float4 o;
        o.x = tanhf(acc.x * s + bb.x); o.y = tanhf(acc.y * s + bb.y); o.z = tanhf(acc.z * s + bb.z); o.w = tanhf(acc.w * s + bb.w);
        *reinterpret_cast<float4 *>(h1 + (int64_t)b * ldh + c4 * 4) = o;
    }
}

__global__ void __launch_bounds__(256) vae_embed_bwd_kernel(float *__restrict__ dW1, int H, const int64_t *__restrict__ indptr,
                                                            const int32_t *__restrict__ indices, const int32_t *__restrict__ rows,
                                                            const float *__restrict__ dpre1, int64_t ldd, float drop_rate,
                                                            uint64_t seed) {
    const int b = blockIdx.x;
    const int u = rows[b];
    const int64_t beg = indptr[u], end = indptr[u + 1];
    const float scale = (end > beg ? rsqrtf((float)(end - beg)) : 0.f) * (drop_rate > 0.f ? 1.f / (1.f - drop_rate) : 1.f);
    for (int c4 = threadIdx.x; c4 * 4 < H; c4 += blockDim.x) {
        float4 g = *reinterpret_cast<const float4 *>(dpre1 + (int64_t)b * ldd + c4 * 4);
        g.x *= scale; g.y *= scale; g.z *= scale; g.w *= scale;
        for (int64_t p = beg; p < end; p++) {
            if (drop_rate > 0.f) {
                uint32_t r[4];
                Philox::gen(seed, (uint64_t)b, (uint32_t)(p - beg), r);
                if ((float)(r[0] >> 8) * (1.f / 16777216.f) < drop_rate) continue;
            }
            vred4(dW1 + (int64_t)indices[p] * H + c4 * 4, g);
        }
    }
}

// counter = (step, element): distinct (step, e) never share a draw, whatever B is from step to step (e < B L < 2^32)
__device__ __forceinline__ float philox_normal(uint64_t seed, uint64_t ctr, uint32_t sub) {
    uint32_t r[4];
    Philox::gen(seed, ctr, sub, r);
    const float u1 = ((float)(r[0] >> 8) + 0.5f) * (1.f / 16777216.f), u2 = (float)(r[1] >> 8) * (1.f / 16777216.f);
    return sqrtf(-2.f * __logf(u1)) * __cosf(6.283185307179586f * u2);      // Box-Muller
}

// ml: [B][2L] = (mu | log_var); z: [B][L]; kl_sum += sum(lv - mu^2 - e^lv + 1)
__global__ void __launch_bounds__(256) vae_reparam_fwd_kernel(const float *__restrict__ ml, int64_t ldml, int B, int L,
                                                              float *__restrict__ z, int64_t ldz, uint64_t seed, uint64_t step,
                                                              double *kl_sum) {
    const int64_t n = (int64_t)B * L;
    float acc = 0.f;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(e / L), l = (int)(e - (int64_t)b * L);
        const float mu = ml[(int64_t)b * ldml + l], lv = ml[(int64_t)b * ldml + L + l];
        const float eps = philox_normal(seed, step, (uint32_t)e);
        z[(int64_t)b * ldz + l] = mu + __expf(0.5f * lv) * eps;
        acc += lv - mu * mu - __expf(lv) + 1.f;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (kl_sum && (threadIdx.x & 31) == 0 && acc != 0.f) atomicAdd(kl_sum, (double)acc);
}

// dml[b][l] = dz + anneal mu/(B L);  dml[b][L+l] = dz * 0.5 e^{lv/2} eps + anneal 0.5 (e^lv - 1)/(B L)
__global__ void __launch_bounds__(256) vae_reparam_bwd_kernel(const float *__restrict__ ml, int64_t ldml, int B, int L,
                                                              const float *__restrict__ dz, int64_t lddz, float *__restrict__ dml,
                                                              int64_t lddml, uint64_t seed, uint64_t step, float anneal) {
    const int64_t n = (int64_t)B * L;
    const float c = anneal / (float)n;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(e / L), l = (int)(e - (int64_t)b * L);
        const float mu = ml[(int64_t)b * ldml + l], lv = ml[(int64_t)b * ldml + L + l];
        const float eps = philox_normal(seed, step, (uint32_t)e);
        const float g = dz[(int64_t)b * lddz + l];
        dml[(int64_t)b * lddml + l] = g + c * mu;
        dml[(int64_t)b * lddml + L + l] = g * 0.5f * __expf(0.5f * lv) * eps + c * 0.5f * (__expf(lv) - 1.f);
    }
}

// one CTA per batch row: logits[b,:] -> dlogits = (softmax * nnz_b - x) / B in place; nll += -sum_{i in row}(logit_i - lse)
// lse_out (optional) receives the row's log-sum-exp (predict path: log_softmax = logit - lse)
__global__ void __launch_bounds__(256) vae_softmax_kernel(float *__restrict__ logits, int64_t ld, int n_items,
                                                          const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                          const int32_t *__restrict__ rows, int B, double *nll_sum,
                                                          float *lse_out, int write_grad) {
    __shared__ float red[8];
    __shared__ float s_bcast;
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *row = logits + (int64_t)b * ld;
    float m = -CUDART_INF_F;
    for (int i = threadIdx.x; i < n_items; i += blockDim.x) m = fmaxf(m, row[i]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if (lane == 0) red[warp] = m;
    __syncthreads();
    if (threadIdx.x == 0) { float t = red[0]; for (int w = 1; w < 8; w++) t = fmaxf(t, red[w]); s_bcast = t; }
    __syncthreads();
    m = s_bcast;
    float s = 0.f;
    for (int i = threadIdx.x; i < n_items; i += blockDim.x) s += __expf(row[i] - m);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    __syncthreads();
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < 8; w++) t += red[w]; s_bcast = m + __logf(t); }
    __syncthreads();
    const float lse = s_bcast;
    if (lse_out && threadIdx.x == 0) lse_out[b] = lse;
    const int u = rows[b];
    const int64_t beg = indptr[u], end = indptr[u + 1];
    if (nll_sum) {
        float a = 0.f;
        for (int64_t p = beg + threadIdx.x; p < end; p += blockDim.x) a += row[indices[p]] - lse;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
        if (lane == 0 && a != 0.f) atomicAdd(nll_sum, -(double)a);
    }
    if (!write_grad) return;
    __syncthreads();
    const float nb = (float)(end - beg), invB = 1.f / (float)B;
    for (int i = threadIdx.x; i < n_items; i += blockDim.x) row[i] = __expf(row[i] - lse) * nb * invB;
    __syncthreads();
    for (int64_t p = beg + threadIdx.x; p < end; p += blockDim.x) row[indices[p]] -= invB;
}

// The same with the row staged in shared memory: ONE read of the row from HBM/L2 (128-bit loads), max / sum-exp / gradient
// from shared memory, the gradient written once as fp32 (for the bias column sums) and, optionally, as the bf16 operand
// copy the backward GEMMs read (so no separate conversion pass over the B x I block).  n_items * 4 bytes must fit the
// dynamic shared memory given at launch; row starts must be 16-byte aligned (ld % 4 == 0).
__global__ void __launch_bounds__(512) vae_softmax_smem_kernel(float *__restrict__ logits, int64_t ld, int n_items,
                                                               const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                               const int32_t *__restrict__ rows, int B, double *nll_sum, float *lse_out,
                                                               int write_grad, __nv_bfloat16 *__restrict__ grad_bf16, int64_t ldb) {
    extern __shared__ __align__(16) float srow[];
    __shared__ float red[16];
    __shared__ float s_bcast;
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    float *row = logits + (int64_t)b * ld;
    const int n4 = n_items >> 2;
    float m = -CUDART_INF_F;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 v = reinterpret_cast<const float4 *>(row)[i];
        reinterpret_cast<float4 *>(srow)[i] = v;
        m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n_items; i += blockDim.x) { const float v = row[i]; srow[i] = v; m = fmaxf(m, v); }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if (lane == 0) red[warp] = m;
    __syncthreads();
    if (threadIdx.x == 0) { float t = red[0]; for (int w = 1; w < nwarp; w++) t = fmaxf(t, red[w]); s_bcast = t; }
    __syncthreads();
    m = s_bcast;
    float s = 0.f;
    for (int i = threadIdx.x; i < n_items; i += blockDim.x) s += __expf(srow[i] - m);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    __syncthreads();
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (threadIdx.x == 0) { float t = 0.f; for (int w = 0; w < nwarp; w++) t += red[w]; s_bcast = m + __logf(t); }
    __syncthreads();
    const float lse = s_bcast;
    if (lse_out && threadIdx.x == 0) lse_out[b] = lse;
    const int u = rows[b];
    const int64_t beg = indptr[u], end = indptr[u + 1];
    if (nll_sum) {
        float a = 0.f;
        for (int64_t p = beg + threadIdx.x; p < end; p += blockDim.x) a += srow[indices[p]] - lse;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
        if (lane == 0 && a != 0.f) atomicAdd(nll_sum, -(double)a);
    }
    if (!write_grad) return;
    __syncthreads();
    const float nb = (float)(end - beg), invB = 1.f / (float)B;
    for (int i = threadIdx.x; i < n_items; i += blockDim.x) srow[i] = __expf(srow[i] - lse) * nb * invB;
    __syncthreads();
    for (int64_t p = beg + threadIdx.x; p < end; p += blockDim.x) srow[indices[p]] -= invB;
    __syncthreads();
    __nv_bfloat16 *brow = grad_bf16 ? grad_bf16 + (int64_t)b * ldb : nullptr;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        const float4 v = reinterpret_cast<const float4 *>(srow)[i];
        reinterpret_cast<float4 *>(row)[i] = v;
        if (brow) {
            reinterpret_cast<__nv_bfloat162 *>(brow)[2 * i] = __floats2bfloat162_rn(v.x, v.y);
            reinterpret_cast<__nv_bfloat162 *>(brow)[2 * i + 1] = __floats2bfloat162_rn(v.z, v.w);
        }
    }
    for (int i = (n4 << 2) + threadIdx.x; i < n_items; i += blockDim.x) { row[i] = srow[i]; if (brow) brow[i] = __float2bfloat16_rn(srow[i]); }
    if (brow) for (int64_t i = n_items + threadIdx.x; i < ldb; i += blockDim.x) brow[i] = __float2bfloat16_rn(0.f);   // padding columns
}

__global__ void __launch_bounds__(256) tanh_bwd_kernel(const float *__restrict__ dout, const float *__restrict__ out,
                                                       float *__restrict__ dpre, int64_t n) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const float o = out[e];
        dpre[e] = dout[e] * (1.f - o * o);
    }
}

// out[c] = sum_r src[r][c].  Each thread owns one column of a 32-column stripe (coalesced 128-byte row segments), the
// CTA's 8 warps stride over the rows of its SLAB (blockIdx.y); one slab writes the sums, several slabs add them with
// atomics into a zeroed `out` (tall matrices: the bias gradients of a 1 M-sample NeuMF batch would otherwise run on
// cols/32 CTAs and take 13 ms each).
__global__ void __launch_bounds__(256) colsum_kernel(const float *__restrict__ src, int R, int C, int64_t ld, float *__restrict__ out,
                                                     int rows_per_slab) {
    __shared__ float part[8][33];
    const int c = blockIdx.x * 32 + (threadIdx.x & 31), w = threadIdx.x >> 5;
    const int r0 = blockIdx.y * rows_per_slab, r1 = min(R, r0 + rows_per_slab);
    float a = 0.f;
    if (c < C)
        for (int r = r0 + w; r < r1; r += 8) a += src[(int64_t)r * ld + c];
    part[w][threadIdx.x & 31] = a;
    __syncthreads();
    if (w == 0 && c < C) {
        float t = 0.f;
        for (int k = 0; k < 8; k++) t += part[k][threadIdx.x & 31];
        if (gridDim.y == 1) out[c] = t; else atomicAdd(out + c, t);
    }
}

// masked top-k over an existing dense score block (scores are destroyed); out_val = score + shift[row]
__global__ void __launch_bounds__(256) dense_topk_kernel(float *__restrict__ scores, int64_t ld, int n_items,
                                                         const int64_t *__restrict__ mask_indptr,
                                                         const int32_t *__restrict__ mask_indices, const int32_t *__restrict__ rows,
                                                         const float *__restrict__ shift, int k, int32_t *__restrict__ out_idx,
                                                         float *__restrict__ out_val) {
    __shared__ float red_v[8];
    __shared__ int red_i[8];
    __shared__ int win_i;
    const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *s = scores + (int64_t)b * ld;
    const float NEG = -CUDART_INF_F;
    if (mask_indptr) {
        const int u = rows[b];
        for (int64_t p = mask_indptr[u] + threadIdx.x; p < mask_indptr[u + 1]; p += blockDim.x) s[mask_indices[p]] = NEG;
    }
    __syncthreads();
    const float sh = shift ? shift[b] : 0.f;
    for (int r = 0; r < k; r++) {
        float bv = NEG; int bi = 0x7fffffff;
        for (int it = threadIdx.x; it < n_items; it += blockDim.x) {
            const float v = s[it];
            if (v > bv || (v == bv && v > NEG && it < bi)) { bv = v; bi = it; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, off); const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
            if (ov > bv || (ov == bv && ov > NEG && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { red_v[warp] = bv; red_i[warp] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < 8; w++)
                if (red_v[w] > bv || (red_v[w] == bv && bv > NEG && red_i[w] < bi)) { bv = red_v[w]; bi = red_i[w]; }
            const bool ok = bv > NEG;
            out_idx[(int64_t)b * k + r] = ok ? bi : -1;
            out_val[(int64_t)b * k + r] = ok ? bv + sh : NEG;
            win_i = ok ? bi : -1;
            if (ok) s[bi] = NEG;
        }
        __syncthreads();
        if (win_i < 0) {
            for (int rr = r + 1 + threadIdx.x; rr < k; rr += blockDim.x) { out_idx[(int64_t)b * k + rr] = -1; out_val[(int64_t)b * k + rr] = NEG; }
            break;
        }
    }
}

static inline unsigned grid_for(int64_t n) {
    int64_t g = (n + 255) / 256; const int64_t cap = (int64_t)sm_count() * 8;
    return (unsigned)(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace eb

using namespace eb;

extern "C" int eb_vae_embed_fwd(const float *W1, const float *b1, int H, const int64_t *indptr, const int32_t *indices,
                                const int32_t *rows, int B, float *h1, int64_t ldh, float drop_rate, uint64_t seed, void *stream) {
    EB_ARG(W1 && b1 && indptr && indices && rows && h1 && B >= 1 && H >= 4 && H % 4 == 0 && ldh >= H && ldh % 4 == 0, "bad argument");
    vae_embed_fwd_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(W1, b1, H, indptr, indices, rows, h1, ldh, drop_rate, seed);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_vae_embed_bwd(float *dW1, int H, const int64_t *indptr, const int32_t *indices, const int32_t *rows, int B,
                                const float *dpre1, int64_t ldd, float drop_rate, uint64_t seed, void *stream) {
    EB_ARG(dW1 && indptr && indices && rows && dpre1 && B >= 1 && H % 4 == 0 && ldd % 4 == 0, "bad argument");
    vae_embed_bwd_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(dW1, H, indptr, indices, rows, dpre1, ldd, drop_rate, seed);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_vae_reparam_fwd(const float *ml, int64_t ldml, int B, int L, float *z, int64_t ldz, uint64_t seed, uint64_t step,
                                  double *kl_sum, void *stream) {
    EB_ARG(ml && z && B >= 1 && L >= 1, "bad argument");
    EB_ARG((int64_t)B * L < (1ll << 32), "B * L must be below 2^32 (the noise counter's element word)");
    vae_reparam_fwd_kernel<<<grid_for((int64_t)B * L), 256, 0, (cudaStream_t)stream>>>(ml, ldml, B, L, z, ldz, seed, step, kl_sum);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_vae_reparam_bwd(const float *ml, int64_t ldml, int B, int L, const float *dz, int64_t lddz, float *dml,
                                  int64_t lddml, uint64_t seed, uint64_t step, float anneal, void *stream) {
    EB_ARG(ml && dz && dml && B >= 1 && L >= 1, "bad argument");
    EB_ARG((int64_t)B * L < (1ll << 32), "B * L must be below 2^32 (the noise counter's element word)");
    vae_reparam_bwd_kernel<<<grid_for((int64_t)B * L), 256, 0, (cudaStream_t)stream>>>(ml, ldml, B, L, dz, lddz, dml, lddml, seed,
                                                                                        step, anneal);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_vae_softmax_bf16(float *logits, int64_t ld, int n_items, const int64_t *indptr, const int32_t *indices,
                                   const int32_t *rows, int B, double *nll_sum, float *lse_out, int write_grad, void *grad_bf16,
                                   int64_t ld_bf16, void *stream) {
    EB_ARG(logits && indptr && indices && rows && B >= 1 && n_items >= 1 && ld >= n_items, "bad argument");
    // the bf16 copy is a GEMM operand: 16-byte rows on both paths (the unstaged one converts through eb_convert_bf16)
    EB_ARG(!grad_bf16 || (write_grad && ld_bf16 >= n_items && ld_bf16 % 8 == 0 && ((uintptr_t)grad_bf16 % 16) == 0),
           "bad bf16 gradient buffer (ld_bf16 must be a multiple of 8 covering the row, 16-byte aligned)");
    const size_t smem = (size_t)n_items * sizeof(float);
    const bool staged = smem <= 200 * 1024 && ld % 4 == 0 && ((uintptr_t)logits % 16) == 0;
    if (staged) {
        EB_CUDA(cudaFuncSetAttribute(vae_softmax_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        vae_softmax_smem_kernel<<<B, 512, smem, (cudaStream_t)stream>>>(logits, ld, n_items, indptr, indices, rows, B, nll_sum, lse_out,
                                                                        write_grad, (__nv_bfloat16 *)grad_bf16, ld_bf16);
    } else {
        vae_softmax_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(logits, ld, n_items, indptr, indices, rows, B, nll_sum, lse_out, write_grad);
        if (grad_bf16) {
            EB_CUDA(cudaGetLastError());
            return eb_convert_bf16(logits, B, n_items, ld, grad_bf16, ld_bf16, 0, stream);
        }
    }
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_vae_softmax(float *logits, int64_t ld, int n_items, const int64_t *indptr, const int32_t *indices,
                              const int32_t *rows, int B, double *nll_sum, float *lse_out, int write_grad, void *stream) {
    return eb_vae_softmax_bf16(logits, ld, n_items, indptr, indices, rows, B, nll_sum, lse_out, write_grad, nullptr, 0, stream);
}

extern "C" int eb_tanh_bwd(const float *dout, const float *out, float *dpre, int64_t n, void *stream) {
    EB_ARG(dout && out && dpre && n >= 0, "bad argument");
    if (n == 0) return EB_OK;
    tanh_bwd_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(dout, out, dpre, n);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_colsum(const float *src, int rows, int cols, int64_t ld, float *out, void *stream) {
    EB_ARG(src && out && rows >= 1 && cols >= 1 && ld >= cols, "bad argument");
    const int stripes = (cols + 31) / 32;
    int slabs = 1;
    if (rows > 8192) {                                         // short matrices keep the single-slab, fixed-order sum
        slabs = (sm_count() * 4 + stripes - 1) / stripes;
        const int max_slabs = (rows + 1023) / 1024;            // at least 1024 rows per slab
        if (slabs > max_slabs) slabs = max_slabs;
        if (slabs < 1) slabs = 1;
    }
    const int rows_per_slab = (rows + slabs - 1) / slabs;
    if (slabs > 1) EB_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)cols, (cudaStream_t)stream));
    colsum_kernel<<<dim3((unsigned)stripes, (unsigned)slabs), 256, 0, (cudaStream_t)stream>>>(src, rows, cols, ld, out, rows_per_slab);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_dense_topk_f32(float *scores, int64_t ld, int n_rows, int n_items, const int64_t *mask_indptr,
                                 const int32_t *mask_indices, const int32_t *rows, const float *shift, int k, int32_t *out_idx,
                                 float *out_val, void *stream) {
    EB_ARG(scores && out_idx && out_val && n_rows >= 1 && n_items >= 1 && k >= 1 && ld >= n_items, "bad argument");
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr) && (!mask_indptr || rows), "mask CSR needs indptr, indices and rows");
    dense_topk_kernel<<<n_rows, 256, 0, (cudaStream_t)stream>>>(scores, ld, n_items, mask_indptr, mask_indices, rows, shift, k, out_idx,
                                                                out_val);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
