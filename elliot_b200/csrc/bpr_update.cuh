// bpr_update.cuh — the fp32 BPR update of one triple (BPRMF_model.py:91-117), shared by the Hogwild kernels of
// bpr_train.cu and the fetched-rows kernel of sharded.cu.  A group of G lanes owns one triple, each lane a slice of
// float4 columns of the three rows.
#pragma once
#include "common.cuh"

namespace eb {

struct BprHyper {
    float lr, reg_u, reg_b, reg_pos, reg_neg;
};

// one lane's float4 share of u.(v_i - v_j)
__device__ __forceinline__ float bpr_partial_dot(float4 a, float4 vi, float4 vj) {
    return a.x * (vi.x - vj.x) + a.y * (vi.y - vj.y) + a.z * (vi.z - vj.z) + a.w * (vi.w - vj.w);
}

// sum over the G lanes of a group (every lane receives it)
template <int G>
__device__ __forceinline__ float group_sum(float part) {
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
    return part;
}

// x = (b_i - b_j) + u.(v_i - v_j): returns z = 1 / (1 + e^x) (BPRMF_model.py:98); the group's lane 0 adds softplus(-x)
__device__ __forceinline__ float bpr_sigmoid_loss(float x, float &loss_acc, int gl) {
    const float z = __fdividef(1.f, 1.f + __expf(x));
    if (gl == 0) loss_acc += fmaxf(-x, 0.f) + __logf(1.f + __expf(-fabsf(x)));
    return z;
}

// deltas of one float4 of the user row a and the item rows vi, vj
__device__ __forceinline__ void bpr_row_deltas(float4 a, float4 vi, float4 vj, float z, const BprHyper &h, float4 &du, float4 &di,
                                               float4 &dj) {
    du.x = h.lr * ((vi.x - vj.x) * z - h.reg_u * a.x);
    du.y = h.lr * ((vi.y - vj.y) * z - h.reg_u * a.y);
    du.z = h.lr * ((vi.z - vj.z) * z - h.reg_u * a.z);
    du.w = h.lr * ((vi.w - vj.w) * z - h.reg_u * a.w);
    float4 un;
    un.x = a.x + du.x; un.y = a.y + du.y; un.z = a.z + du.z; un.w = a.w + du.w;
    // item rows see the UPDATED user row (view aliasing, BPRMF_model.py:92,109-116)
    di.x = h.lr * (un.x * z - h.reg_pos * vi.x);
    di.y = h.lr * (un.y * z - h.reg_pos * vi.y);
    di.z = h.lr * (un.z * z - h.reg_pos * vi.z);
    di.w = h.lr * (un.w * z - h.reg_pos * vi.w);
    dj.x = h.lr * (-un.x * z - h.reg_neg * vj.x);
    dj.y = h.lr * (-un.y * z - h.reg_neg * vj.y);
    dj.z = h.lr * (-un.z * z - h.reg_neg * vj.z);
    dj.w = h.lr * (-un.w * z - h.reg_neg * vj.w);
}

__device__ __forceinline__ void bpr_bias_deltas(float z, float bi, float bj, const BprHyper &h, float &dbi, float &dbj) {
    dbi = h.lr * (z - h.reg_b * bi);
    dbj = h.lr * (-z - h.reg_b * bj);
}

}  // namespace eb
