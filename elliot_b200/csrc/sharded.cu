// sharded.cu — kernels for ROW-SHARDED embedding tables (SURVEY.md §8e; no reference counterpart: the
// reference is single-device).  A rank that needs rows it does not own asks the owners (NCCL all-to-all of
// ids, done by the host in elliot_b200/parallel.py), owners gather them (eb_gather_rows_f32), the requester
// runs the BPR update against the fetched copies (eb_bpr_step_rows_f32: user rows are local and updated in
// place, item-row DELTAS are written per triple), deltas travel back and owners add them
// (eb_scatter_add_rows_f32).  Same update as bpr_hogwild_kernel (bpr_update.cuh, BPRMF_model.py:91-117).
#include "bpr_update.cuh"

namespace eb {

// out[t][0..w) = table[ids[t]][0..w)   (w % 4 == 0)
__global__ void __launch_bounds__(256) gather_rows_kernel(const float *table, int64_t ld, const int32_t *ids, int64_t n, int w,
                                                          float *out, int64_t ldo) {
    const int64_t total = n * (w / 4);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = e / (w / 4); const int c = (int)(e - t * (w / 4)) * 4;
        *reinterpret_cast<float4 *>(out + t * ldo + c) = *reinterpret_cast<const float4 *>(table + (int64_t)ids[t] * ld + c);
    }
}
// table[ids[t]][0..w) += rows[t][0..w)
__global__ void __launch_bounds__(256) scatter_add_rows_kernel(float *table, int64_t ld, const int32_t *ids, int64_t n, int w,
                                                               const float *rows, int64_t ldr) {
    const int64_t total = n * (w / 4);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = e / (w / 4); const int c = (int)(e - t * (w / 4)) * 4;
        red_add_v4(table + (int64_t)ids[t] * ld + c, *reinterpret_cast<const float4 *>(rows + t * ldr + c));
    }
}

// one warp-group of G = DP/4 lanes per triple (like bpr_hogwild_kernel), item rows come from fetched buffers.
// The fetched item buffers carry the item bias in column `d` when bias_col >= 0 (tables padded so that d < ld).
template <int DP>
__global__ void __launch_bounds__(256) bpr_rows_kernel(float *U, int64_t ldu, const int32_t *tu, const float *Ri, const float *Rj,
                                                       int64_t ldr, int64_t n, int bias_col, const BprHyper h, float *dRi, float *dRj,
                                                       double *loss) {
    constexpr int NV = DP / 4, G = NV >= 32 ? 32 : NV, VPL = NV / G;
    const int lane = threadIdx.x & 31, gl = lane % G;
    const int64_t grp = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * (32 / G) + lane / G;
    const int64_t ngrp = (((int64_t)gridDim.x * blockDim.x) >> 5) * (32 / G);
    float loss_acc = 0.f;
    const int64_t n_round = (n + ngrp - 1) / ngrp * ngrp;         // keep shuffles warp-uniform
    for (int64_t t = grp; t < n_round; t += ngrp) {
        const bool on = t < n;
        float4 a[VPL], vi[VPL], vj[VPL];
        float part = 0.f;
        int u = 0;
        if (on) {
            u = tu[t];
#pragma unroll
            for (int v = 0; v < VPL; v++) {
                a[v] = *reinterpret_cast<const float4 *>(U + (int64_t)u * ldu + (v * G + gl) * 4);
                vi[v] = *reinterpret_cast<const float4 *>(Ri + t * ldr + (v * G + gl) * 4);
                vj[v] = *reinterpret_cast<const float4 *>(Rj + t * ldr + (v * G + gl) * 4);
            }
        }
        // the bias column (if any) lives inside the padded row: exclude it from the dot product
        float bi = 0.f, bj = 0.f;
        if (on && bias_col >= 0) { bi = Ri[t * ldr + bias_col]; bj = Rj[t * ldr + bias_col]; }
        if (on) {
#pragma unroll
            for (int v = 0; v < VPL; v++) {
                const int e = (v * G + gl) * 4;
                const float m0 = (e + 0 == bias_col) ? 0.f : 1.f, m1 = (e + 1 == bias_col) ? 0.f : 1.f,
                            m2 = (e + 2 == bias_col) ? 0.f : 1.f, m3 = (e + 3 == bias_col) ? 0.f : 1.f;
                part += m0 * a[v].x * (vi[v].x - vj[v].x) + m1 * a[v].y * (vi[v].y - vj[v].y) +
                        m2 * a[v].z * (vi[v].z - vj[v].z) + m3 * a[v].w * (vi[v].w - vj[v].w);
            }
        }
        part = group_sum<G>(part);
        if (!on) continue;
        const float z = bpr_sigmoid_loss(part + (bi - bj), loss_acc, gl);
#pragma unroll
        for (int v = 0; v < VPL; v++) {
            const int e = (v * G + gl) * 4;
            float4 du, di, dj;
            bpr_row_deltas(a[v], vi[v], vj[v], z, h, du, di, dj);
            // the bias entries of the item rows take the bias update; the user row has no bias
            auto bias_entry = [&](int c, float &du_c, float &di_c, float &dj_c, float bi_c, float bj_c) {
                if (e + c == bias_col) { du_c = 0.f; bpr_bias_deltas(z, bi_c, bj_c, h, di_c, dj_c); }
            };
            bias_entry(0, du.x, di.x, dj.x, vi[v].x, vj[v].x);
            bias_entry(1, du.y, di.y, dj.y, vi[v].y, vj[v].y);
            bias_entry(2, du.z, di.z, dj.z, vi[v].z, vj[v].z);
            bias_entry(3, du.w, di.w, dj.w, vi[v].w, vj[v].w);
            red_add_v4(U + (int64_t)u * ldu + e, du);
            *reinterpret_cast<float4 *>(dRi + t * ldr + e) = di;
            *reinterpret_cast<float4 *>(dRj + t * ldr + e) = dj;
        }
    }
    if (loss) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, off);
        if (lane == 0 && loss_acc != 0.f) atomicAdd(loss, (double)loss_acc);
    }
}

static inline unsigned sgrid(int64_t threads) {
    int64_t g = (threads + 255) / 256; const int64_t cap = (int64_t)sm_count() * 8;
    return (unsigned)(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace eb

using namespace eb;

extern "C" int eb_gather_rows_f32(const float *table, int64_t ld, const int32_t *ids, int64_t n, int width, float *out, int64_t ldo,
                                  void *stream) {
    EB_ARG(table && ids && out && n >= 0 && width >= 4 && width % 4 == 0 && ld >= width && ldo >= width && ld % 4 == 0 && ldo % 4 == 0,
           "bad argument (width, ld, ldo must be multiples of 4)");
    if (n == 0) return EB_OK;
    gather_rows_kernel<<<sgrid(n * (width / 4)), 256, 0, (cudaStream_t)stream>>>(table, ld, ids, n, width, out, ldo);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_scatter_add_rows_f32(float *table, int64_t ld, const int32_t *ids, int64_t n, int width, const float *rows,
                                       int64_t ldr, void *stream) {
    EB_ARG(table && ids && rows && n >= 0 && width >= 4 && width % 4 == 0 && ld >= width && ldr >= width && ld % 4 == 0 && ldr % 4 == 0,
           "bad argument (width, ld, ldr must be multiples of 4)");
    if (n == 0) return EB_OK;
    scatter_add_rows_kernel<<<sgrid(n * (width / 4)), 256, 0, (cudaStream_t)stream>>>(table, ld, ids, n, width, rows, ldr);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_bpr_step_rows_f32(float *U, int64_t ldu, const int32_t *tu, const float *Ri, const float *Rj, int64_t ldr, int64_t n,
                                    int bias_col, float lr, float reg_u, float reg_b, float reg_pos, float reg_neg, float *dRi,
                                    float *dRj, double *loss, void *stream) {
    EB_ARG(U && tu && Ri && Rj && dRi && dRj && n >= 0, "null pointer");
    EB_ARG(ldu == ldr && (bias_col < 0 || bias_col < ldr), "user and item rows must share the row stride; bias_col inside the row");
    if (n == 0) return EB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = sgrid(n * 16);
    const BprHyper h{lr, reg_u, reg_b, reg_pos, reg_neg};
#define EB_ROWS(DPV) case DPV: bpr_rows_kernel<DPV><<<grid, 256, 0, st>>>(U, ldu, tu, Ri, Rj, ldr, n, bias_col, h, dRi, dRj, loss); break;
    switch ((int)ldr) {
        EB_ROWS(8) EB_ROWS(16) EB_ROWS(32) EB_ROWS(64) EB_ROWS(128) EB_ROWS(256)
        default: return set_err(EB_ERR_ARG, "row stride %lld must be one of 8,16,32,64,128,256 floats", (long long)ldr);
    }
#undef EB_ROWS
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
