// bpr_sample.cu — the samplers on their own: membership signatures for the sampler's rejection test, BPR triples and
// pointwise and rated samples drawn from the Philox stream of bpr_sampler.cuh (the same triples the fused steps draw).
#include "bpr_sampler.cuh"

namespace eb {

// one warp per user: OR the two signature bits of every train item into the user's words
__global__ void __launch_bounds__(256) bloom_build_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                                          int32_t n_users, int log2bits, uint32_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int words = 1 << (log2bits - 5);
    for (; w < n_users; w += nw) {
        uint32_t *f = out + w * words;
        for (int k = lane; k < words; k += 32) f[k] = 0u;
        __syncwarp();
        const int64_t beg = indptr[w], end = indptr[w + 1];
        for (int64_t e = beg + lane; e < end; e += 32) {
            uint32_t a, b;
            bloom_bits((uint32_t)indices[e], log2bits, a, b);
            atomicOr(f + (a >> 5), 1u << (a & 31));
            atomicOr(f + (b >> 5), 1u << (b & 31));
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(256) philox_sample_kernel(const SamplerParams p, int64_t n, int32_t *out_u, int32_t *out_i,
                                                            int32_t *out_j) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        int u, i, j;
        sample_triple(p, t, u, i, j);
        out_u[t] = u; out_i[t] = i; out_j[t] = j;
    }
}

// pointwise_pos_neg_sampler.py:24-48: u uniform; one fair bit decides between a uniform train item of u (label 1) and a
// uniform non-train item (label 0).  The BPR sampler already draws both for u: keep one of them.
__global__ void __launch_bounds__(256) pointwise_sample_kernel(const SamplerParams p, int64_t n, int32_t *out_u, int32_t *out_i,
                                                               float *__restrict__ out_label) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        int u, i, j;
        sample_triple(p, t, u, i, j);
        uint32_t r[4];
        Philox::gen(p.seed, p.first + (uint64_t)t, 0x20000000u, r);
        const bool pos = (r[0] >> 31) != 0;
        out_u[t] = u; out_i[t] = pos ? i : j; out_label[t] = pos ? 1.f : 0.f;
    }
}

// custom_pointwise_sparse_sampler.py:24-39: u uniform, i uniform over u's train items, label = u's train rating of i.  The
// user and item are the BPR sampler's draws; `ratings` is aligned with the sorted train CSR.
__global__ void __launch_bounds__(256) rated_sample_kernel(const SamplerParams p, const float *__restrict__ ratings, int64_t n,
                                                           int32_t *out_u, int32_t *out_i, float *__restrict__ out_r) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        uint32_t r[4];
        int u, len;
        int64_t beg;
        sample_user(p, t, r, u, beg, len);
        const int64_t e = beg + bounded(r[1], (uint32_t)len);
        out_u[t] = u; out_i[t] = __ldg(p.indices + e); out_r[t] = __ldg(ratings + e);
    }
}

}  // namespace eb

using namespace eb;

extern "C" int eb_bloom_build(const int64_t *csr_indptr, const int32_t *csr_indices, int32_t n_users, int filter_words,
                              uint32_t *out, void *stream) {
    EB_ARG(csr_indptr && csr_indices && out && n_users >= 1, "bad argument");
    SamplerParams p{};
    if (int rc = set_filter(p, out, filter_words)) return rc;
    bloom_build_kernel<<<capped_grid((int64_t)n_users * 32), 256, 0, (cudaStream_t)stream>>>(csr_indptr, csr_indices, n_users,
                                                                                             p.filter_log2bits, out);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_bpr_sample_philox_filter(int32_t n_users, int32_t n_items, const int64_t *csr_indptr,
                                           const int32_t *csr_indices, const uint32_t *filter, int filter_words, int64_t n,
                                           uint64_t seed, uint64_t first_triple, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                                           void *stream) {
    SamplerParams p;
    if (int rc = sampler_params(p, n_users, n_items, csr_indptr, csr_indices, filter, filter_words, seed, first_triple)) return rc;
    EB_ARG(n >= 0 && out_u && out_i && out_j, "n < 0 or null output");
    if (n == 0) return EB_OK;
    philox_sample_kernel<<<capped_grid(n), 256, 0, (cudaStream_t)stream>>>(p, n, out_u, out_i, out_j);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_pointwise_sample_philox(int32_t n_users, int32_t n_items, const int64_t *csr_indptr, const int32_t *csr_indices,
                                          const uint32_t *filter, int filter_words, int64_t n, uint64_t seed, uint64_t first,
                                          int32_t *out_u, int32_t *out_i, float *out_label, void *stream) {
    SamplerParams p;
    if (int rc = sampler_params(p, n_users, n_items, csr_indptr, csr_indices, filter, filter_words, seed, first)) return rc;
    EB_ARG(n >= 0 && out_u && out_i && out_label, "n < 0 or null output");
    if (n == 0) return EB_OK;
    pointwise_sample_kernel<<<capped_grid(n), 256, 0, (cudaStream_t)stream>>>(p, n, out_u, out_i, out_label);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_rated_sample_philox(int32_t n_users, int32_t n_items, const int64_t *csr_indptr, const int32_t *csr_indices,
                                      const float *csr_ratings, int64_t n, uint64_t seed, uint64_t first, int32_t *out_u,
                                      int32_t *out_i, float *out_rating, void *stream) {
    SamplerParams p;
    if (int rc = sampler_params(p, n_users, n_items, csr_indptr, csr_indices, nullptr, 0, seed, first)) return rc;
    EB_ARG(csr_ratings && n >= 0 && out_u && out_i && out_rating, "n < 0 or null ratings / output");
    if (n == 0) return EB_OK;
    rated_sample_kernel<<<capped_grid(n), 256, 0, (cudaStream_t)stream>>>(p, csr_ratings, n, out_u, out_i, out_rating);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
