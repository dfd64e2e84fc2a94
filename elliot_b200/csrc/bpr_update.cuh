// bpr_update.cuh — the fp32 BPR update of one triple (BPRMF_model.py:91-117), shared by the Hogwild kernels of
// bpr_train.cu and the fetched-rows kernel of sharded.cu.  A group of G lanes owns one triple, each lane a slice of
// float4 columns of the three rows.
#pragma once
#include "common.cuh"

namespace eb {

struct BprHyper {
    float lr, reg_u, reg_b, reg_pos, reg_neg;
};

// Lane groups for rows of DP floats: G lanes own one triple, lane gl of the group holds float4 v * G + gl (v < VPL) of each
// row; UNR triples of a group have their row loads in flight at once.
template <int DP>
struct LaneGroup {
    static constexpr int NV = DP / 4;                 // float4 per row
    static constexpr int G = NV >= 32 ? 32 : NV;      // lanes per triple
    static constexpr int VPL = NV / G;                // float4 per lane
    static constexpr int UNR = G >= 4 ? 4 : G;
    int lane, gl, gbase;                              // lane in the warp, in the group, the group's first lane
    int64_t warp, nwarps;                             // this warp and the warps of the grid
    __device__ __forceinline__ LaneGroup()
        : lane(threadIdx.x & 31), gl(lane % G), gbase(lane - gl), warp(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5),
          nwarps(((int64_t)gridDim.x * blockDim.x) >> 5) {}
};

// the triple lane src holds, on every lane
__device__ __forceinline__ void bcast_triple(int u, int i, int j, int src, int &bu, int &bi, int &bj) {
    bu = __shfl_sync(0xffffffffu, u, src);
    bi = __shfl_sync(0xffffffffu, i, src);
    bj = __shfl_sync(0xffffffffu, j, src);
}

// How an update reaches a row: a vector atomic add at GPU scope (local tables), one at system scope (rows that may live
// in a peer GPU's memory), or a plain store of old + delta (racy Hogwild, flags bit 0).
enum class Write { Atomic, AtomicSys, Store };

template <Write W>
__device__ __forceinline__ void write_row(float *p, float4 old, float4 d) {
    if constexpr (W == Write::Atomic) red_add_v4(p, d);
    else if constexpr (W == Write::AtomicSys) red_add_v4_sys(p, d);
    else *reinterpret_cast<float4 *>(p) = make_float4(old.x + d.x, old.y + d.y, old.z + d.z, old.w + d.w);
}

template <Write W>
__device__ __forceinline__ void write_bias(float *p, float old, float d) {
    if constexpr (W == Write::Atomic) red_add_f32(p, d);
    else if constexpr (W == Write::AtomicSys) red_add_f32_sys(p, d);
    else *p = old + d;
}

// the warp's summed loss, added to *loss (if any) with one fp64 atomic
__device__ __forceinline__ void flush_loss(float loss_acc, double *loss, int lane) {
    if (loss) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, off);
        if (lane == 0 && loss_acc != 0.f) atomicAdd(loss, (double)loss_acc);
    }
}

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
