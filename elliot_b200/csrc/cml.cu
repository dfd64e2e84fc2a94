// cml.cu — CML, collaborative metric learning (Hsieh et al., WWW 2017), the reference's TensorFlow model.
//
// Replaces CML_model.call/train_step (elliot/recommender/latent_factor_models/CML/CML_model.py:59-98).  The sampler's
// (B, 1) index arrays make the squared distances (B, 1) and the squeezed biases (B,), so score, difference and loss
// broadcast to B x B: every triple's distance term meets every triple's bias term.  With
//   D_a = |gu_a - gj_a|^2 - |gu_a - gi_a|^2   (fp32, as TF)      E_b = Bi[pos_b] - Bi[neg_b]   (fp32)
// the loss is
//   L = sum_a sum_b max(m - clip(D_a + E_b, -80, 1e8), 0)
//       + l_w/2 sum_a (|gu_a|^2 + |gi_a|^2 + |gj_a|^2) + l_b/2 sum_b Bi[pos_b]^2 + l_b/20 sum_b Bi[neg_b]^2.
// A pair passes a gradient ("is active") when -80 < D_a + E_b <= m: clip_by_value passes it strictly inside its bounds
// (the convention of oracle/tf_models.py for BPRMF_batch) and Maximum passes it to its first argument on a tie.  With
// n_a = #{b active with a} and n'_b = #{a active with b}:
//   dgu_a = -2 n_a (gi_a - gj_a) + l_w gu_a   dgi_a = -2 n_a (gu_a - gi_a) + l_w gi_a   dgj_a = 2 n_a (gu_a - gj_a) + l_w gj_a
//   dBi[pos_b] = -n'_b + l_b Bi[pos_b]        dBi[neg_b] = n'_b + l_b Bi[neg_b] / 10     (duplicates summed)
// and, since sum_a sum_{b active} E_b = sum_b n'_b E_b, the hinge sum is
//   sum_a [(m + 80) #{b : D_a + E_b <= -80} + (m - D_a) n_a] - sum_b n'_b E_b       (m > -80, m < 1e8).
// So nothing of size B x B is formed: D and E are sorted, and each count is two binary searches.  Pairs are classified
// on the fp64 sum of the fp32 D_a and E_b (fp64 addition is monotone, so each predicate holds on a prefix of a sorted
// array), which makes every count a deterministic function of D and E; counts are int64.  Cost O(B f + B log B).
// Launches: terms (warp per triple: D, E, the regularisation loss), two key sorts, scatter (thread per triple searches
// its n_a, then the warp adds the three rows' gradients with vector atomics), bias (thread per triple searches n'_b).
// tensorflow==2.3.2 cannot be executed here: parity with TF is UNPINNED; the checker is oracle/cml.py.
#include <cub/cub.cuh>

#include "common.cuh"

namespace eb {

struct CmlParams {
    const float *Gu, *Gi, *Bi;
    float *dGu, *dGi, *dBi;
    int ld;
    const int32_t *tu, *ti, *tj;
    int64_t n;
    float l_w, l_b;
    double m;                                  // the fp32 margin, widened
    float *D, *E;                              // triple order
    const float *Ds, *Es;                      // sorted
    double *loss;
};

// (#{k : x + s[k] <= t1}, #{k : x + s[k] <= t2}) over the sorted s[0..n), sums in fp64: both predicates hold on a prefix,
// so each count is found by binary lifting; the two searches' loads are independent and interleave.
__device__ __forceinline__ void count_two(const float *__restrict__ s, int64_t n, double x, double t1, double t2,
                                          int64_t &c1, int64_t &c2) {
    c1 = 0; c2 = 0;
    int64_t step = 1;
    while (step * 2 <= n) step *= 2;
    for (; n > 0 && step > 0; step >>= 1) {
        const int64_t k1 = c1 + step, k2 = c2 + step;
        const bool y1 = k1 <= n && x + (double)__ldg(s + k1 - 1) <= t1;
        const bool y2 = k2 <= n && x + (double)__ldg(s + k2 - 1) <= t2;
        if (y1) c1 = k1;
        if (y2) c2 = k2;
    }
}

__device__ __forceinline__ void add_loss(double acc, double *loss) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if ((threadIdx.x & 31) == 0 && acc != 0.0) atomicAdd(loss, acc);
}

__device__ __forceinline__ float sq4(float4 a) { return a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w; }
__device__ __forceinline__ float4 sub4(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
// c x + r y, per component
__device__ __forceinline__ float4 axpby4(float c, float4 x, float r, float4 y) {
    return make_float4(c * x.x + r * y.x, c * x.y + r * y.y, c * x.z + r * y.z, c * x.w + r * y.w);
}

// Rows are read as in bpr_batch_grad_kernel: a group of G lanes per triple, VPL float4 per lane; the 32 triples of a
// warp's tile are handed to the groups by shuffles.
template <int DP>
__global__ void __launch_bounds__(256) cml_terms_kernel(const CmlParams p) {
    constexpr int NV = DP / 4, G = NV >= 32 ? 32 : NV, VPL = NV / G;
    const int lane = threadIdx.x & 31, gl = lane % G, gbase = lane - gl;
    const int64_t warp_id = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t ld = p.ld;
    double loss_acc = 0.0;
    for (int64_t tile = warp_id; tile * 32 < p.n; tile += nwarps) {
        const int64_t t = tile * 32 + lane;
        int u = -1, i = 0, j = 0;
        if (t < p.n) { u = __ldg(p.tu + t); i = __ldg(p.ti + t); j = __ldg(p.tj + t); }
#pragma unroll 1
        for (int s = 0; s < G; s++) {
            const int cu = __shfl_sync(0xffffffffu, u, gbase + s), ci = __shfl_sync(0xffffffffu, i, gbase + s),
                      cj = __shfl_sync(0xffffffffu, j, gbase + s);
            float dp = 0.f, dq = 0.f, sq = 0.f;
            if (cu >= 0) {
#pragma unroll
                for (int v = 0; v < VPL; v++) {
                    const float4 a = reinterpret_cast<const float4 *>(p.Gu + (int64_t)cu * ld)[v * G + gl];
                    const float4 vi = reinterpret_cast<const float4 *>(p.Gi + (int64_t)ci * ld)[v * G + gl];
                    const float4 vj = reinterpret_cast<const float4 *>(p.Gi + (int64_t)cj * ld)[v * G + gl];
                    dp += sq4(sub4(a, vi));
                    dq += sq4(sub4(a, vj));
                    sq += sq4(a) + sq4(vi) + sq4(vj);
                }
            }
#pragma unroll
            for (int off = G / 2; off > 0; off >>= 1) {
                dp += __shfl_xor_sync(0xffffffffu, dp, off);
                dq += __shfl_xor_sync(0xffffffffu, dq, off);
                sq += __shfl_xor_sync(0xffffffffu, sq, off);
            }
            if (cu >= 0 && gl == 0) {
                const int64_t ct = tile * 32 + gbase + s;
                const float bi = p.Bi[ci], bj = p.Bi[cj];
                p.D[ct] = dq - dp;
                p.E[ct] = bi - bj;
                loss_acc += 0.5 * p.l_w * (double)sq + 0.5 * p.l_b * (double)bi * bi + 0.05 * p.l_b * (double)bj * bj;
            }
        }
    }
    if (p.loss) add_loss(loss_acc, p.loss);
}

template <int DP>
__global__ void __launch_bounds__(256) cml_scatter_kernel(const CmlParams p) {
    constexpr int NV = DP / 4, G = NV >= 32 ? 32 : NV, VPL = NV / G;
    const int lane = threadIdx.x & 31, gl = lane % G, gbase = lane - gl;
    const int64_t warp_id = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t ld = p.ld;
    double loss_acc = 0.0;
    for (int64_t tile = warp_id; tile * 32 < p.n; tile += nwarps) {
        const int64_t t = tile * 32 + lane;
        int u = -1, i = 0, j = 0;
        float c = 0.f;                                                  // 2 n_t
        if (t < p.n) {
            u = __ldg(p.tu + t); i = __ldg(p.ti + t); j = __ldg(p.tj + t);
            const double d = p.D[t];
            int64_t below, upto;
            count_two(p.Es, p.n, d, -80.0, p.m, below, upto);
            const int64_t na = upto - below;
            loss_acc += (p.m + 80.0) * (double)below + (p.m - d) * (double)na;
            c = 2.f * (float)na;
        }
#pragma unroll 1
        for (int s = 0; s < G; s++) {
            const int cu = __shfl_sync(0xffffffffu, u, gbase + s), ci = __shfl_sync(0xffffffffu, i, gbase + s),
                      cj = __shfl_sync(0xffffffffu, j, gbase + s);
            const float cc = __shfl_sync(0xffffffffu, c, gbase + s);
            if (cu < 0) continue;
#pragma unroll
            for (int v = 0; v < VPL; v++) {
                const int e = (v * G + gl) * 4;
                const float4 a = reinterpret_cast<const float4 *>(p.Gu + (int64_t)cu * ld)[v * G + gl];
                const float4 vi = reinterpret_cast<const float4 *>(p.Gi + (int64_t)ci * ld)[v * G + gl];
                const float4 vj = reinterpret_cast<const float4 *>(p.Gi + (int64_t)cj * ld)[v * G + gl];
                red_add_v4(p.dGu + (int64_t)cu * ld + e, axpby4(-cc, sub4(vi, vj), p.l_w, a));
                red_add_v4(p.dGi + (int64_t)ci * ld + e, axpby4(-cc, sub4(a, vi), p.l_w, vi));
                red_add_v4(p.dGi + (int64_t)cj * ld + e, axpby4(cc, sub4(a, vj), p.l_w, vj));
            }
        }
    }
    if (p.loss) add_loss(loss_acc, p.loss);
}

__global__ void __launch_bounds__(256) cml_bias_kernel(const CmlParams p) {
    double loss_acc = 0.0;
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < p.n; b += (int64_t)gridDim.x * blockDim.x) {
        const float e = p.E[b];
        int64_t below, upto;
        count_two(p.Ds, p.n, (double)e, -80.0, p.m, below, upto);
        const int64_t nb = upto - below;
        loss_acc -= (double)e * (double)nb;
        const int i = __ldg(p.ti + b), j = __ldg(p.tj + b);
        const float g = (float)nb;
        red_add_f32(p.dBi + i, -g + p.l_b * p.Bi[i]);
        red_add_f32(p.dBi + j, g + 0.1f * p.l_b * p.Bi[j]);
    }
    if (p.loss) add_loss(loss_acc, p.loss);
}

// U2 = 2 Gu (every column), user_off[u] = -|Gu[u]|^2, item_off[i] = Bi[i] - |Gi[i]|^2: the operands on which the
// dot-product scorers give Bi[i] - |Gu[u] - Gi[i]|^2 once user_off is added.  One warp per row.
__global__ void __launch_bounds__(256) cml_score_operands_kernel(const float *__restrict__ Gu, const float *__restrict__ Gi,
                                                                 const float *__restrict__ Bi, int64_t ld, int32_t n_users,
                                                                 int32_t n_items, float *__restrict__ U2,
                                                                 float *__restrict__ item_off, float *__restrict__ user_off) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < (int64_t)n_users + n_items; r += nwarps) {
        const bool user = r < n_users;
        const float4 *row = reinterpret_cast<const float4 *>(user ? Gu + r * ld : Gi + (r - n_users) * ld);
        float acc = 0.f;
        for (int64_t c = lane; c < ld / 4; c += 32) {
            const float4 x = __ldg(row + c);
            acc += sq4(x);
            if (user) reinterpret_cast<float4 *>(U2 + r * ld)[c] = make_float4(2.f * x.x, 2.f * x.y, 2.f * x.z, 2.f * x.w);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
        if (lane == 0) {
            if (user) user_off[r] = -acc;
            else item_off[r - n_users] = Bi[r - n_users] - acc;
        }
    }
}

struct CmlLayout {
    size_t ds, es, cub, cub_bytes, total;
};

static CmlLayout cml_layout(int64_t n) {
    CmlLayout L{};
    size_t off = 0;
    L.ds = off; off += align_up((size_t)n * 4);
    L.es = off; off += align_up((size_t)n * 4);
    size_t cb = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, cb, (const float *)nullptr, (float *)nullptr, (int)n);
    L.cub_bytes = cb;
    L.cub = off; off += align_up(cb);
    L.total = off;
    return L;
}

}  // namespace eb

using namespace eb;

extern "C" size_t eb_cml_workspace_bytes(int64_t n) {
    if (n < 1) n = 1;
    if (n > INT32_MAX) return 0;
    return cml_layout(n).total;
}

extern "C" int eb_cml_grad_f32(const float *Gu, const float *Gi, const float *Bi, float *dGu, float *dGi, float *dBi, int d,
                               int ld, const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n, float l_w, float l_b,
                               float margin, float *terms, double *loss, void *workspace, size_t workspace_bytes,
                               void *stream) {
    EB_ARG(dGu && dGi && dBi, "null gradient table");
    if (int rc = check_tables(Gu, Gi, Bi, d, ld)) return rc;
    EB_ARG(((uintptr_t)dGu % 16) == 0 && ((uintptr_t)dGi % 16) == 0, "gradient tables must be 16-byte aligned");
    EB_ARG(margin > -80.f && margin < 1e8f, "margin=%g must lie in (-80, 1e8), inside the clip of the difference", margin);
    if (n <= 0) return EB_OK;
    EB_ARG(n <= INT32_MAX, "n=%lld triples exceed the sort's int32 count", (long long)n);
    EB_ARG(tu && ti && tj && terms, "null triple or terms array");
    const CmlLayout L = cml_layout(n);
    EB_ARG(workspace, "null workspace");
    if (workspace_bytes < L.total)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu bytes < %zu", workspace_bytes, L.total);
    char *ws = (char *)workspace;
    CmlParams p{Gu, Gi, Bi, dGu, dGi, dBi, ld, tu, ti, tj, n, l_w, l_b, (double)margin, terms, terms + n,
                (const float *)(ws + L.ds), (const float *)(ws + L.es), loss};
    cudaStream_t st = (cudaStream_t)stream;
    int64_t grid = ((n + 31) / 32 + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
#define EB_CML_ROWS(K)                                                                                          \
    switch (ld) {                                                                                               \
        case 8: K<8><<<(unsigned)grid, 256, 0, st>>>(p); break;                                                 \
        case 16: K<16><<<(unsigned)grid, 256, 0, st>>>(p); break;                                               \
        case 32: K<32><<<(unsigned)grid, 256, 0, st>>>(p); break;                                               \
        case 64: K<64><<<(unsigned)grid, 256, 0, st>>>(p); break;                                               \
        case 128: K<128><<<(unsigned)grid, 256, 0, st>>>(p); break;                                             \
        case 256: K<256><<<(unsigned)grid, 256, 0, st>>>(p); break;                                             \
        default: return set_err(EB_ERR_ARG, "row stride ld=%d must be one of 8,16,32,64,128,256 floats", ld);  \
    }
    EB_CML_ROWS(cml_terms_kernel);
    EB_CUDA(cudaGetLastError());
    size_t cb = L.cub_bytes;
    EB_CUDA(cub::DeviceRadixSort::SortKeys(ws + L.cub, cb, (const float *)p.D, (float *)(ws + L.ds), (int)n, 0, 32, st));
    cb = L.cub_bytes;
    EB_CUDA(cub::DeviceRadixSort::SortKeys(ws + L.cub, cb, (const float *)p.E, (float *)(ws + L.es), (int)n, 0, 32, st));
    EB_CML_ROWS(cml_scatter_kernel);
    EB_CUDA(cudaGetLastError());
#undef EB_CML_ROWS
    cml_bias_kernel<<<capped_grid(n), 256, 0, st>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_cml_score_operands_f32(const float *Gu, const float *Gi, const float *Bi, int ld, int32_t n_users,
                                         int32_t n_items, float *U2, float *item_off, float *user_off, void *stream) {
    EB_ARG(Gu && Gi && Bi && U2 && item_off && user_off, "null pointer");
    EB_ARG(ld >= 4 && ld % 4 == 0, "row stride ld=%d must be a positive multiple of 4", ld);
    EB_ARG(((uintptr_t)Gu % 16) == 0 && ((uintptr_t)Gi % 16) == 0 && ((uintptr_t)U2 % 16) == 0, "tables must be 16-byte aligned");
    EB_ARG(n_users >= 0 && n_items >= 0, "negative row count");
    const int64_t rows = (int64_t)n_users + n_items;
    if (rows == 0) return EB_OK;
    cml_score_operands_kernel<<<capped_grid(rows * 32), 256, 0, (cudaStream_t)stream>>>(Gu, Gi, Bi, ld, n_users, n_items, U2,
                                                                                          item_off, user_off);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
