// ConvNeuMF (outer-product CNN, convolutional_neural_matrix_factorization_model.py:19-183): the level-1 convolution of
// a batch's (user, item) pairs, forward and backward, the MLP head with the clipped BPR loss, the fused full-catalogue
// scorer and the rank pass over a dense score block.
//
// Geometry.  Every layer is a 2 x 2 'valid' convolution of stride 2, so level l has H_l = floor(f / 2^l) positions per
// axis and the final position (p, q) of level L reads exactly the 2^L x 2^L block [2^L p, 2^L (p + 1)) x [2^L q, ...) of
// the map M[x][y] = u[x] i[y].  Rows of level l are stored per pair in Z-order: local row
//   ((p H_L + q) << 2 (L - l)) | sum_k (abit_k 2 + bbit_k) 4^k       (a, b the level-l position, k over its low L - l bits)
// so the four level-(l-1) rows of one level-l position are consecutive and a level-l layer is the plain GEMM
// [rows_l][4 c_(l-1)] x [4 c_(l-1)][c_l] with K ordered (da, db, c), Keras's [kh, kw, c_in, c_out] kernel layout.
// Level 1 is bilinear: with S0[a][c] = W1[0,0,c] u[2a] + W1[1,0,c] u[2a+1] and S1[a][c] = W1[0,1,c] u[2a] + W1[1,1,c] u[2a+1],
//   x1[a][b][c] = relu(S0[a][c] i[2b] + S1[a][c] i[2b+1] + b1[c])
// (W1 as the flat [2][2][1][c1] Keras kernel: W1[(da 2 + db) c1 + c]).  Every kernel here evaluates it with l1_s / l1_pre,
// so the training forward, its backward (which recomputes the ReLU mask) and the scorer agree bit for bit.
#include <cuda_bf16.h>
#include <math_constants.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace eb {

namespace {

__device__ __forceinline__ float l1_s(float w0, float w1, float u0, float u1) { return fmaf(w1, u1, w0 * u0); }
__device__ __forceinline__ float l1_pre(float s0, float s1, float i0, float i1, float b) { return fmaf(s1, i1, fmaf(s0, i0, b)); }

// level-l position (a, b) of local row r, lr = L - l low bit pairs
__device__ __forceinline__ void zdecode(int64_t r, int lr, int HL, int &a, int &b) {
    const int64_t t = r >> (2 * lr);
    const uint32_t rem = (uint32_t)(r & ((1ll << (2 * lr)) - 1));
    int da = 0, db = 0;
    for (int k = 0; k < lr; k++) {
        da |= ((rem >> (2 * k + 1)) & 1u) << k;
        db |= ((rem >> (2 * k)) & 1u) << k;
    }
    a = (int)(t / HL) << lr | da;
    b = (int)(t % HL) << lr | db;
}

__device__ __forceinline__ void zdecode32(int r, int lr, int HL, int &a, int &b) {
    const int t = r >> (2 * lr);
    const uint32_t rem = (uint32_t)r & ((1u << (2 * lr)) - 1);
    int da = 0, db = 0;
    for (int k = 0; k < lr; k++) {
        da |= ((rem >> (2 * k + 1)) & 1u) << k;
        db |= ((rem >> (2 * k)) & 1u) << k;
    }
    a = (t / HL) << lr | da;
    b = (t % HL) << lr | db;
}

// local row of level-l position (a, b)
__device__ __forceinline__ int64_t zencode(int a, int b, int lr, int HL) {
    uint32_t rem = 0;
    for (int k = 0; k < lr; k++) rem |= (((uint32_t)(a >> k) & 1u) << (2 * k + 1)) | (((uint32_t)(b >> k) & 1u) << (2 * k));
    return ((int64_t)(a >> lr) * HL + (b >> lr)) << (2 * lr) | rem;
}

// ---------------------------------------------------------------- level 1, training forward
// One thread per (pair, level-1 row, 8 channels): relu'd values in Z-order, fp32 or bf16 rows of c1.
__global__ void __launch_bounds__(256) l1_fwd_kernel(const float *__restrict__ U, const float *__restrict__ I, int64_t ld,
                                                     const int32_t *__restrict__ pu, const int32_t *__restrict__ pi,
                                                     int64_t n_pairs, int L, int HL, int c1, const float *__restrict__ W1,
                                                     const float *__restrict__ b1, float *__restrict__ out32,
                                                     __nv_bfloat16 *__restrict__ out16) {
    const int64_t R1 = (int64_t)HL * HL << (2 * (L - 1));
    const int g8 = c1 / 8;
    const int64_t total = n_pairs * R1 * g8;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int cg = (int)(e % g8);
        const int64_t row = e / g8, pair = row / R1;
        int a, b;
        zdecode(row % R1, L - 1, HL, a, b);
        const float *u = U + (int64_t)pu[pair] * ld, *it = I + (int64_t)pi[pair] * ld;
        const float u0 = u[2 * a], u1 = u[2 * a + 1], i0 = it[2 * b], i1 = it[2 * b + 1];
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int c = cg * 8 + k;
            const float s0 = l1_s(W1[c], W1[2 * c1 + c], u0, u1), s1 = l1_s(W1[c1 + c], W1[3 * c1 + c], u0, u1);
            v[k] = fmaxf(l1_pre(s0, s1, i0, i1, b1[c]), 0.f);
        }
        if (out16) {
            __align__(16) __nv_bfloat162 h[4];
#pragma unroll
            for (int k = 0; k < 4; k++) h[k] = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
            *reinterpret_cast<uint4 *>(out16 + row * c1 + cg * 8) = *reinterpret_cast<const uint4 *>(h);
        } else {
            float4 *o = reinterpret_cast<float4 *>(out32 + row * c1 + cg * 8);
            o[0] = make_float4(v[0], v[1], v[2], v[3]);
            o[1] = make_float4(v[4], v[5], v[6], v[7]);
        }
    }
}

// ---------------------------------------------------------------- level 1, training backward
// One CTA per pair.  g = dx1 where the recomputed pre-activation is > 0.  Pass 1, a thread per (a, c):
//   T_db = sum_b g i[2b + db]  ->  du[2a + da] += sum_c W1[da,db,c] T_db,  dW1[da,db,c] += u[2a + da] T_db,  db1[c] += sum g.
// Pass 2, a thread per (b, c):  di[2b + db] += sum_a g S_db[a][c].
// Sums over the CTA go through shared-memory atomics, the CTA's totals to global memory as reductions; the pair's rows
// also get l_w u (pairs below n_user_reg: each triple's user once) and l_w i, the gradient of l_w l2_loss.
__global__ void __launch_bounds__(256) l1_bwd_kernel(const float *__restrict__ U, const float *__restrict__ I, int64_t ld, int f,
                                                     const int32_t *__restrict__ pu, const int32_t *__restrict__ pi,
                                                     int64_t n_user_reg, int L, int HL, int c1, const float *__restrict__ W1,
                                                     const float *__restrict__ b1, const float *__restrict__ dx1, float l_w,
                                                     float *__restrict__ dU, float *__restrict__ dI, float *__restrict__ dW1,
                                                     float *__restrict__ db1) {
    extern __shared__ float sm[];
    float *su = sm, *si = su + f, *sdu = si + f, *sdi = sdu + f, *sdw = sdi + f, *sdb = sdw + 4 * c1;
    const int64_t pair = blockIdx.x;
    const int A = HL << (L - 1);
    const int64_t R1 = (int64_t)HL * HL << (2 * (L - 1));
    const float *u = U + (int64_t)pu[pair] * ld, *it = I + (int64_t)pi[pair] * ld;
    const float *g1 = dx1 + pair * R1 * c1;
    for (int k = threadIdx.x; k < f; k += blockDim.x) { su[k] = u[k]; si[k] = it[k]; sdu[k] = 0.f; sdi[k] = 0.f; }
    for (int k = threadIdx.x; k < 5 * c1; k += blockDim.x) sdw[k] = 0.f;
    __syncthreads();
    for (int e = threadIdx.x; e < A * c1; e += blockDim.x) {
        const int a = e / c1, c = e % c1;
        const float w00 = W1[c], w01 = W1[c1 + c], w10 = W1[2 * c1 + c], w11 = W1[3 * c1 + c], bc = b1[c];
        const float u0 = su[2 * a], u1 = su[2 * a + 1];
        const float s0 = l1_s(w00, w10, u0, u1), s1 = l1_s(w01, w11, u0, u1);
        float t0 = 0.f, t1 = 0.f, gs = 0.f;
        for (int b = 0; b < A; b++) {
            const float i0 = si[2 * b], i1 = si[2 * b + 1];
            if (l1_pre(s0, s1, i0, i1, bc) > 0.f) {
                const float g = g1[zencode(a, b, L - 1, HL) * c1 + c];
                t0 = fmaf(g, i0, t0); t1 = fmaf(g, i1, t1); gs += g;
            }
        }
        atomicAdd(sdu + 2 * a, w00 * t0 + w01 * t1);
        atomicAdd(sdu + 2 * a + 1, w10 * t0 + w11 * t1);
        atomicAdd(sdw + c, u0 * t0); atomicAdd(sdw + c1 + c, u0 * t1);
        atomicAdd(sdw + 2 * c1 + c, u1 * t0); atomicAdd(sdw + 3 * c1 + c, u1 * t1);
        atomicAdd(sdb + c, gs);
    }
    for (int e = threadIdx.x; e < A * c1; e += blockDim.x) {
        const int b = e / c1, c = e % c1;
        const float w00 = W1[c], w01 = W1[c1 + c], w10 = W1[2 * c1 + c], w11 = W1[3 * c1 + c], bc = b1[c];
        const float i0 = si[2 * b], i1 = si[2 * b + 1];
        float d0 = 0.f, d1 = 0.f;
        for (int a = 0; a < A; a++) {
            const float u0 = su[2 * a], u1 = su[2 * a + 1];
            const float s0 = l1_s(w00, w10, u0, u1), s1 = l1_s(w01, w11, u0, u1);
            if (l1_pre(s0, s1, i0, i1, bc) > 0.f) {
                const float g = g1[zencode(a, b, L - 1, HL) * c1 + c];
                d0 = fmaf(g, s0, d0); d1 = fmaf(g, s1, d1);
            }
        }
        atomicAdd(sdi + 2 * b, d0);
        atomicAdd(sdi + 2 * b + 1, d1);
    }
    __syncthreads();
    float *du = dU + (int64_t)pu[pair] * ld, *di = dI + (int64_t)pi[pair] * ld;
    const bool user_reg = pair < n_user_reg;
    for (int k = threadIdx.x; k < f; k += blockDim.x) {
        red_add_f32(du + k, user_reg ? fmaf(l_w, su[k], sdu[k]) : sdu[k]);
        red_add_f32(di + k, fmaf(l_w, si[k], sdi[k]));
    }
    for (int k = threadIdx.x; k < 4 * c1; k += blockDim.x) red_add_f32(dW1 + k, sdw[k]);
    for (int k = threadIdx.x; k < c1; k += blockDim.x) red_add_f32(db1 + k, sdb[k]);
}

// ---------------------------------------------------------------- head and loss
// Keras Dropout keep mask of unit c of one layer for one pair: Philox word (key seed, counter (pair, 16 layer + c / 4)),
// kept when its top 24 bits are >= p 2^24.
__device__ __forceinline__ float drop_scale(uint64_t seed, uint64_t ctr, int layer, int c, float p) {
    if (p <= 0.f) return 1.f;
    uint32_t w[4];
    Philox::gen(seed, ctr, (uint32_t)(16 * layer + c / 4), w);
    const uint32_t x = (c & 3) == 0 ? w[0] : (c & 3) == 1 ? w[1] : (c & 3) == 2 ? w[2] : w[3];
    return (float)(x >> 8) >= p * 16777216.f ? 1.f / (1.f - p) : 0.f;
}

constexpr int HEAD_MAX_C = 64;

// One CTA (256 threads) per triple: pair 0 = (u, i), pair 1 = (u, j).  The last level's rows of each pair are summed per
// channel in a fixed order (strided partial sums, then the partials in order), the head runs in fp32, the loss in fp64.
__global__ void __launch_bounds__(256) head_kernel(const float *__restrict__ hL, int64_t RL, int cL, const float *__restrict__ Wd1,
                                                   const float *__restrict__ bd1, const float *__restrict__ wd2,
                                                   const float *__restrict__ bd2, const float *__restrict__ U,
                                                   const float *__restrict__ I, int64_t ld, int f, const int32_t *__restrict__ tu,
                                                   const int32_t *__restrict__ ti, const int32_t *__restrict__ tj, int64_t n,
                                                   int64_t first, int64_t n_total, float p_drop, uint64_t seed, float l_w,
                                                   double *__restrict__ loss, float *__restrict__ dWd1, float *__restrict__ dbd1,
                                                   float *__restrict__ dwd2, float *__restrict__ dbd2, float *__restrict__ dpre,
                                                   float *__restrict__ y_out, float *__restrict__ mask_out) {
    __shared__ float part[256];
    __shared__ float s[2][HEAD_MAX_C], x1[2][HEAD_MAX_C], x2[2][HEAD_MAX_C], m2[2][HEAD_MAX_C], dz[2][HEAD_MAX_C];
    __shared__ float ds[2][HEAD_MAX_C], y[2], dy[2];
    __shared__ double reg[8];
    const int64_t t = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nparts = 256 / cL, c_of = tid % cL, part_of = tid / cL;
    for (int pp = 0; pp < 2; pp++) {
        const float *h = hL + (pp * n + t) * RL * cL;
        float acc = 0.f;
        if (part_of < nparts)
            for (int64_t r = part_of; r < RL; r += nparts) acc += h[r * cL + c_of];
        part[tid] = acc;
        __syncthreads();
        if (tid < cL) {
            float v = 0.f;
            for (int q = 0; q < nparts; q++) v += part[q * cL + tid];
            s[pp][tid] = v;
        }
        __syncthreads();
    }
    // forward: one warp per pair
    if (warp < 2) {
        const int pp = warp;
        const uint64_t ctr = (uint64_t)(pp ? n_total : 0) + (uint64_t)(first + t);
        for (int c = lane; c < cL; c += 32) {
            const float m1 = drop_scale(seed, ctr, 0, c, p_drop);
            x1[pp][c] = s[pp][c] * m1;
            m2[pp][c] = drop_scale(seed, ctr, 1, c, p_drop);
            if (mask_out) { mask_out[((first + t) * 2 + pp) * 2 * cL + c] = m1; }
        }
        __syncwarp();
        float yp = 0.f;
        for (int o = lane; o < cL; o += 32) {
            float z = bd1[o];
            for (int c = 0; c < cL; c++) z = fmaf(x1[pp][c], Wd1[c * cL + o], z);
            x2[pp][o] = z * m2[pp][o];
            if (mask_out) mask_out[((first + t) * 2 + pp) * 2 * cL + cL + o] = m2[pp][o];
            yp = fmaf(x2[pp][o], wd2[o], yp);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) yp += __shfl_xor_sync(0xffffffffu, yp, off);
        if (lane == 0) y[pp] = yp + bd2[0];
    } else if (warp < 5) {
        // l_w l2_loss of gamma_u, gamma_i, gamma_j in fp64
        const float *row = warp == 2 ? U + (int64_t)tu[t] * ld : I + (int64_t)(warp == 3 ? ti[t] : tj[t]) * ld;
        double q = 0.0;
        for (int k = lane; k < f; k += 32) q += (double)row[k] * row[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
        if (lane == 0) reg[warp] = q;
    }
    __syncthreads();
    if (tid == 0) {
        const double x = (double)y[0] - (double)y[1];
        const double xc = fmin(fmax(x, -80.0), 1e8);
        const double sp = xc > 0 ? log1p(exp(-xc)) : -xc + log1p(exp(xc));       // softplus(-xc)
        atomicAdd(loss, sp + 0.5 * (double)l_w * (reg[2] + reg[3] + reg[4]));
        const float g = (x > -80.0 && x < 1e8) ? (float)(-1.0 / (1.0 + exp(xc))) : 0.f;   // strictly inside the clip
        dy[0] = g; dy[1] = -g;
        if (y_out) { y_out[first + t] = y[0]; y_out[n_total + first + t] = y[1]; }
    }
    __syncthreads();
    if (warp < 2) {
        const int pp = warp;
        const float d = dy[pp];
        if (lane == 0) red_add_f32(dbd2, d);
        for (int o = lane; o < cL; o += 32) {
            red_add_f32(dwd2 + o, d * x2[pp][o]);
            const float z = d * wd2[o] * m2[pp][o];
            dz[pp][o] = z;
            red_add_f32(dbd1 + o, z);
        }
    }
    __syncthreads();
    for (int e = tid; e < cL * cL; e += 256) {
        const int c = e / cL, o = e % cL;
        red_add_f32(dWd1 + e, x1[0][c] * dz[0][o] + x1[1][c] * dz[1][o]);
    }
    if (warp < 2) {
        const int pp = warp;
        const uint64_t ctr = (uint64_t)(pp ? n_total : 0) + (uint64_t)(first + t);
        for (int c = lane; c < cL; c += 32) {
            float v = 0.f;
            for (int o = 0; o < cL; o++) v = fmaf(Wd1[c * cL + o], dz[pp][o], v);
            ds[pp][c] = v * drop_scale(seed, ctr, 0, c, p_drop);
        }
    }
    __syncthreads();
    for (int pp = 0; pp < 2; pp++) {
        const float *h = hL + (pp * n + t) * RL * cL;
        float *dp = dpre + (pp * n + t) * RL * cL;
        for (int64_t e = tid; e < RL * cL; e += 256) dp[e] = h[e] > 0.f ? ds[pp][e % cL] : 0.f;
    }
}

// ---------------------------------------------------------------- fused full-catalogue scorer
// CTA = one warpgroup, one user, SC_P consecutive items.  Level 1 is generated on the CUDA cores straight into the
// registers of the wgmma A operand (from S in shared memory and the items' rows); levels 2..L are wgmma steps against
// W_l resident in shared memory (K-major, 128-byte swizzle, output columns padded to 32 or 64), their bias + ReLU
// epilogues written as the next level's A tile (levels >= 3) in shared memory.  The CTA's level-l rows are its pairs'
// rows back to back, so a 64-row tile of level l is made of four consecutive level-(l-1) tiles; a level-l tile runs as
// soon as the fourth has been written.  The last level's tiles are reduced per pair and channel by one thread per channel
// in row order, and the head runs per pair: the scores do not depend on the launch.
constexpr int SC_P = 32;
constexpr int SC_MAXL = 8;

struct ScoreParams {
    const float *U, *I;
    int64_t ld;
    int f, L, HL;
    int c[SC_MAXL + 1];                  // c[1..L]
    const float *W1, *b1;
    const __nv_bfloat16 *Wp;             // W_l [c_l][4 c_(l-1)] for l = 2..L, back to back
    const float *bp;                     // b_l for l = 2..L, back to back
    const float *Wd1, *bd1, *wd2, *bd2;
    int u0, n_ub, n_items;
    float *scores;
    int64_t lds;
    // shared-memory layout (bytes from the 1024-aligned base)
    uint32_t off_w[SC_MAXL + 1], off_a[SC_MAXL + 1], off_b, off_s, off_i, off_t, off_acc, total;
};

static inline int sc_npad(int c) { return c <= 32 ? 32 : 64; }
static inline int sc_kpad(int k) { return (k + 63) / 64 * 64; }

static void sc_layout(ScoreParams &p) {
    size_t o = 0;
    auto take = [&](size_t n) { size_t r = o; o = align_up(o + n, 1024); return (uint32_t)r; };
    for (int l = 2; l <= p.L; l++) p.off_w[l] = take((size_t)sc_npad(p.c[l]) * sc_kpad(4 * p.c[l - 1]) * 2);
    for (int l = 3; l <= p.L; l++) p.off_a[l] = take((size_t)64 * sc_kpad(4 * p.c[l - 1]) * 2);
    p.off_b = take((size_t)SC_MAXL * 64 * 4);
    const int A = p.HL << (p.L - 1), cL = p.c[p.L];
    p.off_s = take((size_t)A * p.c[1] * 8);
    p.off_i = take((size_t)SC_P * 2 * A * 4);
    p.off_t = take((size_t)4 * 64 * 4);
    p.off_acc = take((size_t)64 * cL * 4);          // up to 64 pairs: a tile of 64 single-row pairs
    p.total = (uint32_t)o + 1024;        // + the alignment of the dynamic base
}

// byte offset of bf16 element (row, k) of a K-major, 128-byte-swizzled tile of `rows` rows (64-column blocks)
__device__ __forceinline__ uint32_t sw128_off(int row, int k, int rows) {
    return (uint32_t)((k >> 6) * rows * 128 + row * 128 + ((((k & 63) >> 3) ^ (row & 7)) << 4) + ((k & 7) << 1));
}

template <int NP>
__device__ __forceinline__ void mma_ss(float *d, uint32_t a_base, uint32_t b_base, int ksteps) {
    for (int ks = 0; ks < ksteps; ks++) {
        const uint64_t da = gmma_desc_sw128(a_base + (ks >> 2) * 64 * 128 + (ks & 3) * 32);
        const uint64_t db = gmma_desc_sw128(b_base + (ks >> 2) * NP * 128 + (ks & 3) * 32);
        if constexpr (NP == 32) wgmma_m64n32k16<0, 0>(d, da, db, ks > 0);
        else wgmma_m64n64k16<0, 0>(d, da, db, ks > 0);
    }
}

// bias + ReLU epilogue of one 64-row tile of a level below L (accumulators of an NP-column wgmma): the bf16 A tile of
// level l + 1, rows 16 slot + r / 4, k = (r % 4) c_l + col
template <int NP>
__device__ __forceinline__ void epilogue(const float *d, int c, const float *bias, unsigned char *anext, int slot) {
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
#pragma unroll
    for (int j = 0; j < NP / 8; j++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int r = 16 * w + l / 4 + 8 * h, col = 8 * j + 2 * (l & 3);
            if (col >= c) continue;
            const float v0 = fmaxf(d[4 * j + 2 * h] + bias[col], 0.f), v1 = fmaxf(d[4 * j + 2 * h + 1] + bias[col + 1], 0.f);
            const int row = 16 * slot + r / 4, k = (r & 3) * c + col;
            *reinterpret_cast<__nv_bfloat162 *>(anext + sw128_off(row, k, 64)) = __floats2bfloat162_rn(v0, v1);
        }
    }
}

// The last level's tile: bias + ReLU, rows past a pair's RL (padding) zeroed, then the channel sums of each pair's rows.
// A pair owns PL consecutive rows (a power of two up to 64, else a multiple of 64), so a tile holds whole segments of
// seg = min(PL, 64) rows: summed over the lanes of a row group (xor 4, 8, 16), then the two halves of a warp, then the
// warps through shared memory, always in the same order; one thread adds each (pair, channel) sum of the tile to acc.
template <int NP>
__device__ __forceinline__ void reduce_last(const float *d, int c, const float *bias, float *acc, int cL, int row0, int PL,
                                            int RL, float *red) {
    const int tid = threadIdx.x, w = tid >> 5, l = tid & 31, g = l >> 2;
    const int seg = PL < 64 ? PL : 64;
    float x[NP / 8][2][2];
#pragma unroll
    for (int j = 0; j < NP / 8; j++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int row = 16 * w + g + 8 * h;
            const bool pad = (row0 + row) % PL >= RL;
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int col = 8 * j + 2 * (l & 3) + e;
                float v = (col < c && !pad) ? fmaxf(d[4 * j + 2 * h + e] + bias[col], 0.f) : 0.f;
                if (seg >= 2) v += __shfl_xor_sync(0xffffffffu, v, 4);
                if (seg >= 4) v += __shfl_xor_sync(0xffffffffu, v, 8);
                if (seg >= 8) v += __shfl_xor_sync(0xffffffffu, v, 16);
                x[j][h][e] = v;
            }
        }
    if (seg <= 16) {
        if (g % (seg < 8 ? seg : 8) == 0)
#pragma unroll
            for (int j = 0; j < NP / 8; j++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int col = 8 * j + 2 * (l & 3) + e;
                    if (col >= c) continue;
                    if (seg == 16) {
                        acc[((row0 + 16 * w) / PL) * cL + col] += x[j][0][e] + x[j][1][e];
                    } else {
#pragma unroll
                        for (int h = 0; h < 2; h++) acc[((row0 + 16 * w + g + 8 * h) / PL) * cL + col] += x[j][h][e];
                    }
                }
        return;
    }
    if (g == 0)
#pragma unroll
        for (int j = 0; j < NP / 8; j++)
#pragma unroll
            for (int e = 0; e < 2; e++) red[w * 64 + 8 * j + 2 * (l & 3) + e] = x[j][0][e] + x[j][1][e];
    __syncthreads();
    if (seg == 32) {
        if (tid < 2 * cL) {
            const int pw = tid / cL, cc = tid % cL;
            acc[((row0 + 32 * pw) / PL) * cL + cc] += red[2 * pw * 64 + cc] + red[(2 * pw + 1) * 64 + cc];
        }
    } else if (tid < cL) {
        acc[(row0 / PL) * cL + tid] += ((red[tid] + red[64 + tid]) + red[128 + tid]) + red[192 + tid];
    }
    __syncthreads();
}

template <int C1>
__global__ void __launch_bounds__(128) score_kernel(const ScoreParams p) {
    extern __shared__ unsigned char smraw[];
    unsigned char *sm = reinterpret_cast<unsigned char *>(((uintptr_t)smraw + 1023) & ~(uintptr_t)1023);
    const int tid = threadIdx.x, L = p.L, HL = p.HL, cL = p.c[L];
    const int A = HL << (L - 1), m2 = 2 * A;
    const int ub = blockIdx.y, user = p.u0 + ub, i0 = blockIdx.x * SC_P;
    const int Pv = min(SC_P, p.n_items - i0);
    float *sS = reinterpret_cast<float *>(sm + p.off_s);      // [A][C1][2]
    float *sI = reinterpret_cast<float *>(sm + p.off_i);      // [SC_P][2A]
    float *sB = reinterpret_cast<float *>(sm + p.off_b);      // [level][64]
    float *tile = reinterpret_cast<float *>(sm + p.off_t);    // [4][64]: the last level's per-warp sums
    float *acc = reinterpret_cast<float *>(sm + p.off_acc);   // [SC_P][cL]
    float *sB1 = sB + (SC_MAXL - 1) * 64;                     // b1
    // operands
    const float *u = p.U + (int64_t)user * p.ld;
    for (int e = tid; e < A * C1; e += 128) {
        const int a = e / C1, c = e % C1;
        const float u0 = u[2 * a], u1 = u[2 * a + 1];
        sS[2 * e] = l1_s(p.W1[c], p.W1[2 * C1 + c], u0, u1);
        sS[2 * e + 1] = l1_s(p.W1[C1 + c], p.W1[3 * C1 + c], u0, u1);
    }
    for (int e = tid; e < SC_P * m2; e += 128) {
        const int q = e / m2, k = e % m2;
        sI[e] = p.I[(int64_t)(i0 + min(q, Pv - 1)) * p.ld + k];
    }
    for (int e = tid; e < 64 * cL; e += 128) acc[e] = 0.f;
    for (int e = tid; e < C1; e += 128) sB1[e] = p.b1[e];
    for (int l = 2; l <= L; l++) {
        const int np = p.c[l] <= 32 ? 32 : 64, K = 4 * p.c[l - 1], kp = (K + 63) / 64 * 64;
        const __nv_bfloat16 *Wg = p.Wp;
        const float *bg = p.bp;
        for (int q = 2; q < l; q++) { Wg += (size_t)p.c[q] * 4 * p.c[q - 1]; bg += p.c[q]; }
        unsigned char *ws = sm + p.off_w[l];
        for (int e = tid; e < np * kp; e += 128) {
            const int n = e / kp, k = e % kp;
            const __nv_bfloat16 v = (n < p.c[l] && k < K) ? Wg[(size_t)n * K + k] : __float2bfloat16(0.f);
            *reinterpret_cast<__nv_bfloat16 *>(ws + sw128_off(n, k, np)) = v;
        }
        for (int e = tid; e < 64; e += 128) sB[(l - 2) * 64 + e] = e < p.c[l] ? bg[e] : 0.f;
    }
    fence_proxy_async();
    __syncthreads();

    if (L == 1) {
        // no tensor-core level: thread per (pair, channel) sums its pair's level-1 rows in row order
        const int64_t R1 = (int64_t)HL * HL;
        for (int e = tid; e < Pv * C1; e += 128) {
            const int q = e / C1, c = e % C1;
            float s = 0.f;
            for (int64_t r = 0; r < R1; r++) {
                const int a = (int)(r / HL), b = (int)(r % HL);
                const float *it = sI + q * m2;
                s += fmaxf(l1_pre(sS[2 * (a * C1 + c)], sS[2 * (a * C1 + c) + 1], it[2 * b], it[2 * b + 1], sB1[c]), 0.f);
            }
            acc[q * cL + c] = s;
        }
    } else {
        // each pair's level-L rows padded to PL (rows past RL are zeroed at the last level), PL2 = its level-2 rows
        const int RL = HL * HL, PL = RL <= 64 ? 1 << (RL > 1 ? 32 - __clz(RL - 1) : 0) : (RL + 63) / 64 * 64;
        const int lr2 = 2 * (L - 2), PL2 = PL << lr2;
        const int TL = (Pv * PL + 63) / 64, T2 = TL << lr2;
        const int w = tid >> 5, ln = tid & 31;
        // k-steps per round: all of them up to 8, else half (c1 = 56's two rounds of 7 spill: rounds of 4, 4, 4 and 2)
        constexpr int KS = 4 * C1 / 16, KC = KS <= 8 ? KS : (KS == 14 ? 4 : KS / 2);
        for (int j2 = 0; j2 < T2; j2++) {
            // level-1 values of this thread's two rows of the level-2 tile, generated as A fragments in rounds of at
            // most 8 k-steps (the registers of a round stay live until its wgmma completes)
            const float *srow[2];
            int a2[2], b2[2];
            for (int h = 0; h < 2; h++) {
                const int r = j2 * 64 + 16 * w + ln / 4 + 8 * h;
                const int q = min(r / PL2, Pv - 1);
                int rr = r % PL2;
                if ((rr >> lr2) >= RL) rr = 0;                 // padding: any valid row
                zdecode32(rr, L - 2, HL, a2[h], b2[h]);
                srow[h] = sI + q * m2;
            }
            const bool last2 = L == 2;
            const uint32_t wb = smem_u32(sm + p.off_w[2]);
            const int np2 = p.c[2] <= 32 ? 32 : 64;
            float d[32];
#pragma unroll
            for (int round = 0; round < (KS + KC - 1) / KC; round++) {
                uint32_t af[KC][4];
#pragma unroll
                for (int kk = 0; kk < KC; kk++) {
                    const int ks = round * KC + kk;
                    if (ks >= KS) break;
#pragma unroll
                    for (int h = 0; h < 2; h++) {
#pragma unroll
                        for (int half = 0; half < 2; half++) {
                            float v[2];
#pragma unroll
                            for (int e = 0; e < 2; e++) {
                                const int k = ks * 16 + 8 * half + 2 * (ln & 3) + e;
                                const int q4 = k / C1, c = k % C1;
                                const int a1 = 2 * a2[h] + (q4 >> 1), b1 = 2 * b2[h] + (q4 & 1);
                                const float2 s = *reinterpret_cast<const float2 *>(sS + 2 * (a1 * C1 + c));
                                const float2 it = *reinterpret_cast<const float2 *>(srow[h] + 2 * b1);
                                v[e] = fmaxf(l1_pre(s.x, s.y, it.x, it.y, sB1[c]), 0.f);
                            }
                            __nv_bfloat162 hv = __floats2bfloat162_rn(v[0], v[1]);
                            af[kk][h + 2 * half] = *reinterpret_cast<uint32_t *>(&hv);
                        }
                    }
                }
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < KC; kk++) {
                    const int ks = round * KC + kk;
                    if (ks >= KS) break;
                    const uint64_t db = gmma_desc_sw128(wb + (ks >> 2) * np2 * 128 + (ks & 3) * 32);
                    if (np2 == 32) wgmma_m64n32k16_rs(d, af[kk], db, ks > 0);
                    else wgmma_m64n64k16_rs(d, af[kk], db, ks > 0);
                }
                wgmma_commit(); wgmma_wait<0>(); wgmma_acc_fence<32>(d);
            }
            if (last2) {
                if (np2 == 32) reduce_last<32>(d, cL, sB, acc, cL, j2 * 64, PL, RL, tile);
                else reduce_last<64>(d, cL, sB, acc, cL, j2 * 64, PL, RL, tile);
            } else {
                unsigned char *an = sm + p.off_a[3];
                if (np2 == 32) epilogue<32>(d, p.c[2], sB, an, j2 & 3);
                else epilogue<64>(d, p.c[2], sB, an, j2 & 3);
            }
            // the levels whose four input tiles are now complete
            int jl = j2;
            for (int l = 3; l <= L; l++) {
                if ((jl & 3) != 3) break;
                jl >>= 2;
                fence_proxy_async();
                __syncthreads();
                const bool last = l == L;
                const uint32_t ab = smem_u32(sm + p.off_a[l]), bb = smem_u32(sm + p.off_w[l]);
                unsigned char *nx = last ? nullptr : sm + p.off_a[l + 1];
                const int ksteps = 4 * p.c[l - 1] / 16, sl = jl & 3;
                const float *bl = sB + (l - 2) * 64;
                if (p.c[l] <= 32) {
                    float d[16];
                    wgmma_fence(); mma_ss<32>(d, ab, bb, ksteps); wgmma_commit(); wgmma_wait<0>(); wgmma_acc_fence<16>(d);
                    __syncthreads();                          // every thread's reads of A_l are done before it is rewritten
                    if (last) reduce_last<32>(d, cL, bl, acc, cL, jl * 64, PL, RL, tile);
                    else epilogue<32>(d, p.c[l], bl, nx, sl);
                } else {
                    float d[32];
                    wgmma_fence(); mma_ss<64>(d, ab, bb, ksteps); wgmma_commit(); wgmma_wait<0>(); wgmma_acc_fence<32>(d);
                    __syncthreads();
                    if (last) reduce_last<64>(d, cL, bl, acc, cL, jl * 64, PL, RL, tile);
                    else epilogue<64>(d, p.c[l], bl, nx, sl);
                }
            }
        }
    }
    __syncthreads();
    // head per pair (dropout off): y = wd2 . (Wd1^T s + bd1) + bd2
    if (tid < Pv) {
        float y = 0.f;
        for (int o = 0; o < cL; o++) {
            float z = p.bd1[o];
            for (int c = 0; c < cL; c++) z = fmaf(acc[tid * cL + c], p.Wd1[c * cL + o], z);
            y = fmaf(z, p.wd2[o], y);
        }
        p.scores[(int64_t)ub * p.lds + i0 + tid] = y + p.bd2[0];
    }
}

// ---------------------------------------------------------------- rank pass over a dense score block
// Per row the list is every item outside the train mask whose score is neither -inf nor NaN, by (score desc, item asc),
// as eb_score_rank_f32 lists; each relevant item in it gets c = the non-relevant listed entries ahead of it.  One CTA per
// row; the positives go in chunks of RK_CHUNK: placed by counting, then every listed non-relevant item adds 1 to
// hist[p], p = the positives ahead of it (binary search), and sum c = sum_p hist[p] (n - p).  Integer atomics only.
constexpr int RK_CHUNK = 1024;

__device__ __forceinline__ bool rk_better(float v, int i, float bv, int bi) {
    return v > bv || (v == bv && v > -CUDART_INF_F && i < bi);
}

__global__ void __launch_bounds__(256, 1) dense_rank_kernel(const float *__restrict__ scores, int64_t lds, int n_items,
                                                         const int32_t *__restrict__ rows, int32_t row_begin,
                                                         const int64_t *__restrict__ mask_indptr,
                                                         const int32_t *__restrict__ mask_indices,
                                                         const int64_t *__restrict__ rel_indptr,
                                                         const int32_t *__restrict__ rel_items, int64_t *__restrict__ n_pos_out,
                                                         int64_t *__restrict__ sum_c_out) {
    __shared__ float cv[RK_CHUNK], sv[RK_CHUNK];
    __shared__ int32_t ci[RK_CHUNK], si[RK_CHUNK];
    __shared__ uint32_t hist[RK_CHUNK + 1];
    __shared__ unsigned long long s_sum;
    const int64_t q = blockIdx.x;
    const int u = rows ? rows[q] : row_begin + (int)q;
    const float *s = scores + q * lds;
    const int64_t rb = rel_indptr[u], re = rel_indptr[u + 1];
    const int32_t *mrow = mask_indptr ? mask_indices + mask_indptr[u] : nullptr;
    const int mn = mask_indptr ? (int)(mask_indptr[u + 1] - mask_indptr[u]) : 0;
    if (threadIdx.x == 0) s_sum = 0;
    int64_t n_pos = 0;
    for (int64_t cb = rb; cb < re; cb += RK_CHUNK) {
        const int ne = (int)min((int64_t)RK_CHUNK, re - cb);
        __syncthreads();
        for (int j = threadIdx.x; j < ne; j += blockDim.x) {
            const int32_t it = rel_items[cb + j];
            const bool listed = it >= 0 && it < n_items && !contains_sorted(mrow, mn, it);
            const float v = listed ? s[it] : -CUDART_INF_F;
            cv[j] = v; ci[j] = v > -CUDART_INF_F ? it : -1;
        }
        __syncthreads();
        for (int j = threadIdx.x; j < ne; j += blockDim.x) {
            if (ci[j] < 0) continue;
            int r = 0;
            for (int o = 0; o < ne; o++) r += ci[o] >= 0 && rk_better(cv[o], ci[o], cv[j], ci[j]);
            sv[r] = cv[j]; si[r] = ci[j];
        }
        int n = 0;
        for (int j0 = 0; j0 < RK_CHUNK; j0 += 256) n += __syncthreads_count(j0 + (int)threadIdx.x < ne && ci[j0 + threadIdx.x] >= 0);
        if (n == 0) continue;
        for (int j = threadIdx.x; j <= n; j += blockDim.x) hist[j] = 0;
        __syncthreads();
        for (int it = threadIdx.x; it < n_items; it += blockDim.x) {
            const float v = s[it];
            if (!(v > -CUDART_INF_F) || contains_sorted(rel_items + rb, (int)(re - rb), it) || contains_sorted(mrow, mn, it)) continue;
            int lo = 0, hi = n;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (rk_better(sv[mid], si[mid], v, it)) lo = mid + 1; else hi = mid;
            }
            atomicAdd(hist + lo, 1u);
        }
        __syncthreads();
        unsigned long long part = 0;
        for (int j = threadIdx.x; j <= n; j += blockDim.x) part += (unsigned long long)hist[j] * (unsigned)(n - j);
        if (part) atomicAdd(&s_sum, part);
        n_pos += n;
    }
    __syncthreads();
    if (threadIdx.x == 0) { n_pos_out[q] = n_pos; sum_c_out[q] = (int64_t)s_sum; }
}

int check_geometry(int f, int L, int HL) {
    EB_ARG(L >= 1 && L <= SC_MAXL && HL >= 1 && (HL << L) <= f && f <= 256, "bad ConvNeuMF geometry f=%d L=%d H_L=%d", f, L, HL);
    return EB_OK;
}

int unpack_widths(uint64_t widths, int L, int *c) {
    for (int l = 1; l <= L; l++) {
        c[l] = (int)((widths >> (8 * (l - 1))) & 0xff);
        EB_ARG(c[l] >= 8 && c[l] <= 64 && c[l] % 8 == 0, "channel width c_%d=%d: need a multiple of 8 in [8, 64]", l, c[l]);
    }
    return EB_OK;
}

template <int C1>
int launch_score(ScoreParams &p, void *stream) {
    if (p.total > 48 * 1024) EB_CUDA(cudaFuncSetAttribute(score_kernel<C1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.total));
    dim3 grid((unsigned)((p.n_items + SC_P - 1) / SC_P), (unsigned)p.n_ub);
    score_kernel<C1><<<grid, 128, p.total, (cudaStream_t)stream>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

}  // namespace
}  // namespace eb

using namespace eb;

extern "C" int eb_convneumf_l1_fwd(const float *U, const float *I, int64_t ld, int f, const int32_t *pu, const int32_t *pi,
                                   int64_t n_pairs, int L, int HL, int c1, const float *W1, const float *b1, void *out,
                                   int out_bf16, void *stream) {
    if (int rc = check_geometry(f, L, HL)) return rc;
    EB_ARG(U && I && pu && pi && W1 && b1 && out && ld >= f, "null pointer or ld < f");
    EB_ARG(c1 >= 8 && c1 <= 64 && c1 % 8 == 0, "c1=%d: need a multiple of 8 in [8, 64]", c1);
    if (n_pairs <= 0) return EB_OK;
    const int64_t total = n_pairs * ((int64_t)HL * HL << (2 * (L - 1))) * (c1 / 8);
    l1_fwd_kernel<<<capped_grid(total), 256, 0, (cudaStream_t)stream>>>(U, I, ld, pu, pi, n_pairs, L, HL, c1, W1, b1,
                                                                         out_bf16 ? nullptr : (float *)out,
                                                                         out_bf16 ? (__nv_bfloat16 *)out : nullptr);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_convneumf_l1_bwd(const float *U, const float *I, int64_t ld, int f, const int32_t *pu, const int32_t *pi,
                                   int64_t n_pairs, int64_t n_user_reg, int L, int HL, int c1, const float *W1, const float *b1,
                                   const float *dx1, float l_w, float *dU, float *dI, float *dW1, float *db1, void *stream) {
    if (int rc = check_geometry(f, L, HL)) return rc;
    EB_ARG(U && I && pu && pi && W1 && b1 && dx1 && dU && dI && dW1 && db1 && ld >= f, "null pointer or ld < f");
    EB_ARG(c1 >= 8 && c1 <= 64 && c1 % 8 == 0, "c1=%d: need a multiple of 8 in [8, 64]", c1);
    if (n_pairs <= 0) return EB_OK;
    EB_ARG(n_pairs < (1ll << 31), "n_pairs=%lld: one CTA per pair", (long long)n_pairs);
    const size_t smem = (size_t)(4 * f + 5 * c1) * sizeof(float);
    l1_bwd_kernel<<<(unsigned)n_pairs, 256, smem, (cudaStream_t)stream>>>(U, I, ld, f, pu, pi, n_user_reg, L, HL, c1, W1, b1, dx1,
                                                                          l_w, dU, dI, dW1, db1);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_convneumf_head(const float *hL, int64_t RL, int cL, const float *Wd1, const float *bd1, const float *wd2,
                                 const float *bd2, const float *U, const float *I, int64_t ld, int f, const int32_t *tu,
                                 const int32_t *ti, const int32_t *tj, int64_t n, int64_t first, int64_t n_total, float p_drop,
                                 uint64_t seed, float l_w, double *loss, float *dWd1, float *dbd1, float *dwd2, float *dbd2,
                                 float *dpre, float *y_out, float *mask_out, void *stream) {
    EB_ARG(hL && Wd1 && bd1 && wd2 && bd2 && U && I && tu && ti && tj && loss && dWd1 && dbd1 && dwd2 && dbd2 && dpre,
           "null pointer");
    EB_ARG(cL >= 8 && cL <= HEAD_MAX_C && cL % 8 == 0 && RL >= 1 && ld >= f, "bad shape cL=%d RL=%lld", cL, (long long)RL);
    EB_ARG(p_drop >= 0.f && p_drop < 1.f, "dropout rate %g outside [0, 1)", (double)p_drop);
    EB_ARG(first >= 0 && first + n <= n_total, "triples [%lld, %lld) outside the batch of %lld", (long long)first,
           (long long)(first + n), (long long)n_total);
    if (n <= 0) return EB_OK;
    head_kernel<<<(unsigned)n, 256, 0, (cudaStream_t)stream>>>(hL, RL, cL, Wd1, bd1, wd2, bd2, U, I, ld, f, tu, ti, tj, n, first,
                                                               n_total, p_drop, seed, l_w, loss, dWd1, dbd1, dwd2, dbd2, dpre,
                                                               y_out, mask_out);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" size_t eb_convneumf_score_smem_bytes(int f, int L, int HL, uint64_t widths) {
    ScoreParams p{};
    p.f = f; p.L = L; p.HL = HL;
    if (check_geometry(f, L, HL) || unpack_widths(widths, L, p.c)) return 0;
    sc_layout(p);
    return p.total;
}

extern "C" int eb_convneumf_score(const float *U, const float *I, int64_t ld, int f, int L, int HL, uint64_t widths,
                                  const float *W1, const float *b1, const void *Wp, const float *bp, const float *Wd1,
                                  const float *bd1, const float *wd2, const float *bd2, int u0, int n_ub, int n_items,
                                  float *scores, int64_t lds, void *stream) {
    ScoreParams p{};
    if (int rc = check_geometry(f, L, HL)) return rc;
    p.f = f; p.L = L; p.HL = HL;
    if (int rc = unpack_widths(widths, L, p.c)) return rc;
    EB_ARG(U && I && W1 && b1 && Wd1 && bd1 && wd2 && bd2 && scores && (L == 1 || (Wp && bp)), "null pointer");
    EB_ARG(ld >= f && lds >= n_items && n_items >= 1 && n_ub <= 65535, "bad shape ld=%lld lds=%lld n_items=%d n_ub=%d",
           (long long)ld, (long long)lds, n_items, n_ub);
    sc_layout(p);
    EB_ARG(p.total <= 227 * 1024, "the scorer needs %u bytes of shared memory for f=%d and these widths (at most 227 KB)",
           p.total, f);
    if (n_ub <= 0) return EB_OK;
    p.U = U; p.I = I; p.ld = ld; p.W1 = W1; p.b1 = b1; p.Wp = (const __nv_bfloat16 *)Wp; p.bp = bp;
    p.Wd1 = Wd1; p.bd1 = bd1; p.wd2 = wd2; p.bd2 = bd2; p.u0 = u0; p.n_ub = n_ub; p.n_items = n_items; p.scores = scores;
    p.lds = lds;
    switch (p.c[1]) {
        case 8: return launch_score<8>(p, stream);
        case 16: return launch_score<16>(p, stream);
        case 24: return launch_score<24>(p, stream);
        case 32: return launch_score<32>(p, stream);
        case 40: return launch_score<40>(p, stream);
        case 48: return launch_score<48>(p, stream);
        case 56: return launch_score<56>(p, stream);
        default: return launch_score<64>(p, stream);
    }
}

extern "C" int eb_dense_rank_f32(const float *scores, int64_t lds, int n_rows, int n_items, const int32_t *rows,
                                 int32_t row_begin, const int64_t *mask_indptr, const int32_t *mask_indices,
                                 const int64_t *rel_indptr, const int32_t *rel_items, int64_t *out_n_pos, int64_t *out_sum_c,
                                 void *stream) {
    EB_ARG(scores && rel_indptr && rel_items && out_n_pos && out_sum_c, "null pointer");
    EB_ARG(lds >= n_items && n_items >= 1, "bad shape lds=%lld n_items=%d", (long long)lds, n_items);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_rows <= 0) return EB_OK;
    dense_rank_kernel<<<(unsigned)n_rows, 256, 0, (cudaStream_t)stream>>>(scores, lds, n_items, rows, row_begin, mask_indptr,
                                                                          mask_indices, rel_indptr, rel_items, out_n_pos,
                                                                          out_sum_c);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
