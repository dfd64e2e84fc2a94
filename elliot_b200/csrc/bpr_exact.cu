// bpr_exact.cu — exact mode of the BPR step, fp64.  Same arithmetic as the Hogwild kernels of bpr_train.cu, but
// sequentially consistent with the array order of the triples: every row carries a turn counter, a triple waits until each
// of its three rows has seen exactly the touches that precede it in the sequence (ranks come from a radix sort of
// (row, position)).
#include <cub/cub.cuh>

#include "common.cuh"

namespace eb {

struct ExactParams {
    double *U, *V, *b;
    int d, ld;
    const int32_t *tu, *ti, *tj;
    const int32_t *ku, *ki, *kj;
    int32_t *cntU, *cntI, *ticket;
    int64_t n;
    double lr, reg_u, reg_b, reg_pos, reg_neg;
    double *loss;
};

__device__ __forceinline__ int ld_acquire(const int32_t *p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int32_t *p, int v) {
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

template <int NE>  // elements per lane, d <= 32*NE
__global__ void __launch_bounds__(128) bpr_exact_kernel(const ExactParams p) {
    const int lane = threadIdx.x & 31;
    double loss_acc = 0.0;
    for (;;) {
        int t = 0;
        if (lane == 0) t = atomicAdd(p.ticket, 1);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= p.n) break;
        const int u = __ldg(p.tu + t), i = __ldg(p.ti + t), j = __ldg(p.tj + t);
        const int wu = __ldg(p.ku + t), wi = __ldg(p.ki + t), wj = __ldg(p.kj + t);
        int32_t *cu = p.cntU + u, *ci = p.cntI + i, *cj = p.cntI + j;
        // Every lane performs the three acquire loads itself and the exit decision is a
        // warp vote: control flow stays warp-uniform and each lane's later row loads are
        // ordered after ITS OWN acquires (no reliance on cross-lane ordering).
        {
            unsigned ns = 8;
            for (;;) {
                const bool ready = (ld_acquire(cu) == wu) & (ld_acquire(ci) == wi) & (ld_acquire(cj) == wj);
                if (__all_sync(0xffffffffu, ready)) break;
                __nanosleep(ns);
                if (ns < 128) ns <<= 1;
            }
        }
        double *pu = p.U + (int64_t)u * p.ld, *pi = p.V + (int64_t)i * p.ld, *pj = p.V + (int64_t)j * p.ld;
        double a[NE], vi[NE], vj[NE];
        double xi = 0.0, xj = 0.0;
#pragma unroll
        for (int e = 0; e < NE; e++) {
            const int k = lane + 32 * e;
            a[e] = 0.0; vi[e] = 0.0; vj[e] = 0.0;
            if (k < p.d) {
                a[e] = __ldcg(pu + k); vi[e] = __ldcg(pi + k); vj[e] = __ldcg(pj + k);
                xi = __dadd_rn(xi, __dmul_rn(a[e], vi[e]));
                xj = __dadd_rn(xj, __dmul_rn(a[e], vj[e]));
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            xi = __dadd_rn(xi, __shfl_xor_sync(0xffffffffu, xi, off));
            xj = __dadd_rn(xj, __shfl_xor_sync(0xffffffffu, xj, off));
        }
        const double bi = __ldcg(p.b + i), bj = __ldcg(p.b + j);
        xi = __dadd_rn(xi, bi);
        xj = __dadd_rn(xj, bj);
        const double x = __dadd_rn(xi, -xj);
        const double z = 1.0 / (1.0 + exp(x));  // BPRMF_model.py:98
        const double sp = (x > 0) ? log1p(exp(-x)) : (-x + log1p(exp(x)));   // all lanes: no divergence
        loss_acc += (lane == 0) ? sp : 0.0;
#pragma unroll
        for (int e = 0; e < NE; e++) {
            const int k = lane + 32 * e;
            // d_u = (V_i - V_j) z - reg_u U[u];  U[u] += lr d_u   (BPRMF_model.py:108-109)
            const double un = __dadd_rn(
                a[e], __dmul_rn(p.lr, __dadd_rn(__dmul_rn(__dadd_rn(vi[e], -vj[e]), z), -__dmul_rn(p.reg_u, a[e]))));
            // d_i = U'[u] z - reg_pos V_i (BPRMF_model.py:112-113), d_j = -U'[u] z - reg_neg V_j (:116-117)
            const double uz = __dmul_rn(un, z);
            const double in_ = __dadd_rn(vi[e], __dmul_rn(p.lr, __dadd_rn(uz, -__dmul_rn(p.reg_pos, vi[e]))));
            const double jn = __dadd_rn(vj[e], __dmul_rn(p.lr, __dadd_rn(-uz, -__dmul_rn(p.reg_neg, vj[e]))));
            if (k < p.d) { __stcg(pu + k, un); __stcg(pi + k, in_); __stcg(pj + k, jn); }
        }
        const double bin = __dadd_rn(bi, __dmul_rn(p.lr, __dadd_rn(z, -__dmul_rn(p.reg_b, bi))));
        const double bjn = __dadd_rn(bj, __dmul_rn(p.lr, __dadd_rn(-z, -__dmul_rn(p.reg_b, bj))));
        if (lane == 0) { __stcg(p.b + i, bin); __stcg(p.b + j, bjn); }
        __threadfence();
        // the release stores depend on a full-warp vote that every lane reaches only after
        // its own fence: all 32 lanes' row stores are visible before any counter moves
        const unsigned done = __ballot_sync(0xffffffffu, true);
        if (done == 0xffffffffu) {
            if (lane == 0) st_release(cu, wu + 1);
            else if (lane == 1) st_release(ci, wi + 1);
            else if (lane == 2) st_release(cj, wj + 1);
        }
    }
    if (p.loss && lane == 0 && loss_acc != 0.0) atomicAdd(p.loss, loss_acc);
}

// keys: (row << ebits) | event ; events of table `which`: users -> event = t, items -> event = 2t+slot
__global__ void make_keys_kernel(const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n, int ebits,
                                 uint64_t *keysU, uint64_t *keysI, int32_t n_users, int32_t n_items, int32_t *status) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    // a triple with i == j would wait on the same row counter twice (the turn never comes: the kernel would spin for
    // ever), an id out of range would touch foreign memory: report both before the ordered kernel is launched
    const uint32_t uu = (uint32_t)tu[t], ii = (uint32_t)ti[t], jj = (uint32_t)tj[t];
    if (ii == jj) atomicOr(status, 1);
    if (uu >= (uint32_t)n_users || ii >= (uint32_t)n_items || jj >= (uint32_t)n_items) { atomicOr(status, 2); return; }
    keysU[t] = ((uint64_t)(uint32_t)tu[t] << ebits) | (uint64_t)t;
    keysI[2 * t] = ((uint64_t)(uint32_t)ti[t] << ebits) | (uint64_t)(2 * t);
    keysI[2 * t + 1] = ((uint64_t)(uint32_t)tj[t] << ebits) | (uint64_t)(2 * t + 1);
}

// rank of each event inside its row segment of the sorted key array
__global__ void ranks_kernel(const uint64_t *keys, int64_t m, int ebits, int is_items, int32_t *ka, int32_t *kb) {
    int64_t pos = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= m) return;
    const uint64_t key = keys[pos];
    const uint64_t first = (key >> ebits) << ebits;
    int64_t lo = 0, hi = pos;  // lower_bound of `first`
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < first) lo = mid + 1; else hi = mid;
    }
    const int32_t rank = (int32_t)(pos - lo);
    const uint64_t ev = key & ((1ull << ebits) - 1);
    if (!is_items) ka[ev] = rank;
    else if (ev & 1) kb[ev >> 1] = rank;
    else ka[ev >> 1] = rank;
}

struct ExactLayout {
    size_t keys_in, keys_out, ku, ki, kj, cnt, cub, total, cub_bytes;
};

// keys_in / keys_out hold 3n entries each: user keys in [0,n), item keys in [n,3n)
static ExactLayout exact_layout(int64_t n, int32_t n_users, int32_t n_items) {
    ExactLayout L;
    size_t off = 0;
    L.keys_in = off; off += align_up(sizeof(uint64_t) * 3 * (size_t)n);
    L.keys_out = off; off += align_up(sizeof(uint64_t) * 3 * (size_t)n);
    L.ku = off; off += align_up(sizeof(int32_t) * (size_t)n);
    L.ki = off; off += align_up(sizeof(int32_t) * (size_t)n);
    L.kj = off; off += align_up(sizeof(int32_t) * (size_t)n);
    L.cnt = off; off += align_up(sizeof(int32_t) * ((size_t)n_users + (size_t)n_items + 64));
    size_t cb = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, cb, (const uint64_t *)nullptr, (uint64_t *)nullptr, (int64_t)(2 * n), 0, 64);
    L.cub_bytes = cb;
    L.cub = off; off += align_up(cb);
    L.total = off;
    return L;
}

}  // namespace eb

using namespace eb;

extern "C" size_t eb_bpr_exact_workspace_bytes(int64_t n, int32_t n_users, int32_t n_items) {
    if (n <= 0) return 256;
    return exact_layout(n, n_users, n_items).total;
}

extern "C" int eb_bpr_exact_f64(double *U, double *V, double *item_bias, int d, int ld, int32_t n_users,
                                int32_t n_items, const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n,
                                double lr, double reg_u, double reg_b, double reg_pos, double reg_neg, double *loss,
                                void *workspace, size_t workspace_bytes, void *stream) {
    if (int rc = check_tables(U, V, item_bias, d, ld)) return rc;
    EB_ARG(d <= 256, "exact mode supports d <= 256 (d=%d)", d);
    EB_ARG(n >= 0 && n < (1ll << 30), "n out of range");
    if (n == 0) return EB_OK;
    EB_ARG(tu && ti && tj && workspace, "null pointer");
    const ExactLayout L = exact_layout(n, n_users, n_items);
    if (workspace_bytes < L.total)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace_bytes, L.total);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    uint64_t *keys_in = (uint64_t *)(ws + L.keys_in), *keys_out = (uint64_t *)(ws + L.keys_out);
    int32_t *ku = (int32_t *)(ws + L.ku), *ki = (int32_t *)(ws + L.ki), *kj = (int32_t *)(ws + L.kj);
    int32_t *cnt = (int32_t *)(ws + L.cnt);
    const int ebits = bits_for((uint64_t)(2 * n));
    const int rbits_u = bits_for((uint64_t)n_users), rbits_i = bits_for((uint64_t)n_items);
    const unsigned blocks = (unsigned)((n + 255) / 256);
    int32_t *status = cnt + (size_t)n_users + (size_t)n_items + 8;
    EB_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
    make_keys_kernel<<<blocks, 256, 0, st>>>(tu, ti, tj, n, ebits, keys_in, keys_in + n, n_users, n_items, status);
    EB_CUDA(cudaGetLastError());
    {   // exact mode is latency-insensitive (one call per epoch): validate synchronously rather than risk a spin that never ends
        int32_t bad = 0;
        EB_CUDA(cudaMemcpyAsync(&bad, status, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        EB_CUDA(cudaStreamSynchronize(st));
        if (bad & 2) return set_err(EB_ERR_ARG, "triple ids out of range (need u < %d, i and j < %d)", n_users, n_items);
        if (bad & 1) return set_err(EB_ERR_ARG, "a triple has i == j (the reference sampler never emits one, custom_sampler.py:39-41)");
    }
    size_t cb = L.cub_bytes;
    EB_CUDA(cub::DeviceRadixSort::SortKeys(ws + L.cub, cb, keys_in, keys_out, n, 0, ebits + rbits_u, st));
    ranks_kernel<<<blocks, 256, 0, st>>>(keys_out, n, ebits, 0, ku, nullptr);
    EB_CUDA(cudaGetLastError());
    cb = L.cub_bytes;
    EB_CUDA(cub::DeviceRadixSort::SortKeys(ws + L.cub, cb, keys_in + n, keys_out + n, 2 * n, 0, ebits + rbits_i, st));
    ranks_kernel<<<(unsigned)((2 * n + 255) / 256), 256, 0, st>>>(keys_out + n, 2 * n, ebits, 1, ki, kj);
    EB_CUDA(cudaGetLastError());
    EB_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * ((size_t)n_users + (size_t)n_items + 64), st));
    ExactParams p{};
    p.U = U; p.V = V; p.b = item_bias; p.d = d; p.ld = ld; p.tu = tu; p.ti = ti; p.tj = tj;
    p.ku = ku; p.ki = ki; p.kj = kj; p.cntU = cnt; p.cntI = cnt + n_users; p.ticket = cnt + n_users + n_items;
    p.n = n; p.lr = lr; p.reg_u = reg_u; p.reg_b = reg_b; p.reg_pos = reg_pos; p.reg_neg = reg_neg; p.loss = loss;
    const int ne = (d + 31) / 32;
    int64_t grid = (int64_t)sm_count() * 4;
    if (grid * 4 > n) grid = (n + 3) / 4;
    if (ne <= 1) bpr_exact_kernel<1><<<(unsigned)grid, 128, 0, st>>>(p);
    else if (ne <= 2) bpr_exact_kernel<2><<<(unsigned)grid, 128, 0, st>>>(p);
    else if (ne <= 4) bpr_exact_kernel<4><<<(unsigned)grid, 128, 0, st>>>(p);
    else bpr_exact_kernel<8><<<(unsigned)grid, 128, 0, st>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
