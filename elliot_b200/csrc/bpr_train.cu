// bpr_train.cu — fused BPR-MF training step kernels (sm_90a).
//
// Replaces MFModel.train_step/update_factors
// (elliot/recommender/latent_factor_models/BPRMF/BPRMF_model.py:87-117) and, in the
// sampled variant, Sampler.step (elliot/dataset/samplers/custom_sampler.py:24-46).
//
//  * bpr_hogwild_kernel  — throughput mode, fp32.  A group of G = d/4 lanes owns one
//    triple: 128-bit loads of the three embedding rows, warp-shuffle reduction of the
//    two dot products, log-sigmoid gradient, 128-bit vector atomics (REDG.F32x4) for
//    the scatter-add.  Each lane of a warp first fetches/samples ONE triple (coalesced
//    index loads or Philox), the groups then walk the warp's 32 triples with shuffles,
//    prefetching the next triple's rows while the current one is reduced.
//  * bpr_grouped_kernel  — the free-running sampled step on local tables: the same update, applied to the triples
//    grouped by user (user_key_kernel + a stable radix sort first), the user row kept in registers across a run.
//  * bpr_exact_kernel   — exact mode, fp64.  Same arithmetic, but sequentially
//    consistent with the array order of the triples: every row carries a turn counter,
//    a triple waits until each of its three rows has seen exactly the touches that
//    precede it in the sequence (ranks come from a radix sort of (row, position)).
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <stdlib.h>

#include <type_traits>

#include "bpr_update.cuh"

namespace eb {

struct HogwildParams {
    float *U, *V, *b;
    int ld;
    const int32_t *tu, *ti, *tj;
    int64_t n;
    BprHyper hp;
    double *loss;
    // sampler
    int32_t n_users, n_items;
    const int64_t *indptr;
    const int32_t *indices;
    uint64_t seed, first;
    int32_t *out_u, *out_i, *out_j;
    // PEER mode (item table row-sharded over the GPUs of one NVSwitch box, SURVEY.md §8e): shard s holds item rows
    // [s*shards.rows, (s+1)*shards.rows) at Vp[s] / bp[s] — local memory for this rank's shard, peer-mapped memory
    // (cudaIpcOpenMemHandle, peer.cu) for the others; loads and vector atomics go straight over NVLink.
    float *Vp[EB_MAX_PEERS], *bp[EB_MAX_PEERS];
    ShardMap shards;
    // optional per-user membership signatures (eb_bloom_build): filter_log2bits bits per user
    const uint32_t *filter;
    int filter_log2bits;
    // optional PACKED triples (host boundary: 8 B instead of 12 B per triple over PCIe): u | i << bits_u | j << (bits_u + bits_i)
    const uint64_t *packed;
    int bits_u, bits_i;
    int no_item_updates;      // profiling only (flags bit 2): item rows are read but not updated
    // grouped sampled step: the call's triple indices ordered by user (ascending u, then ascending t)
    const int32_t *order;
};

// u of triple t: uniform over the users that own at least one and not every item.  r keeps the Philox block that drew the
// accepted u (its other words pick i and j), beg / len the user's CSR row.
__device__ __forceinline__ void sample_user(const HogwildParams &p, int64_t t, uint32_t (&r)[4], int &u, int64_t &beg, int &len) {
    Philox::gen(p.seed, p.first + (uint64_t)t, 0u, r);
    u = (int)bounded(r[0], (uint32_t)p.n_users);
    beg = __ldg(p.indptr + u);
    int64_t end = __ldg(p.indptr + u + 1);
    len = (int)(end - beg);
    uint32_t attempt = 0;
    while (len == 0 || len >= p.n_items) {  // users without train items never appear in the reference's dict; a user owning
                                            // every item has no negative at all (the reference would loop forever)
        Philox::gen(p.seed, p.first + (uint64_t)t, ++attempt | 0x80000000u, r);
        u = (int)bounded(r[0], (uint32_t)p.n_users);
        beg = __ldg(p.indptr + u); end = __ldg(p.indptr + u + 1); len = (int)(end - beg);
    }
}

// u uniform over users, i uniform over the user's train items, j uniform over the
// complement (rejection against the sorted CSR row) — custom_sampler.py:31-42 semantics,
// Philox stream instead of MT19937.
__device__ __forceinline__ void sample_triple(const HogwildParams &p, int64_t t, int &u, int &i, int &j) {
    uint32_t r[4];
    int64_t beg;
    int len;
    sample_user(p, t, r, u, beg, len);
    uint32_t attempt = 0;
    const int32_t *row = p.indices + beg;
    int cand = (int)bounded(r[2], (uint32_t)p.n_items);
    // the signature words depend on u only: their loads are in flight together with the pick of i
    const bool maybe = p.filter ? bloom_maybe(p.filter + ((int64_t)u << (p.filter_log2bits - 5)), p.filter_log2bits, (uint32_t)cand) : true;
    i = __ldg(row + bounded(r[1], (uint32_t)len));
    if (!maybe || !contains_sorted(row, len, cand)) { j = cand; return; }
    cand = (int)bounded(r[3], (uint32_t)p.n_items);
    attempt = 0;
    int q = 4;
    while (contains_sorted(row, len, cand) && attempt < 16u) {
        if (q == 4) { Philox::gen(p.seed, p.first + (uint64_t)t, ++attempt, r); q = 0; }
        cand = (int)bounded(r[q++], (uint32_t)p.n_items);
    }
    if (attempt >= 16u && contains_sorted(row, len, cand)) {
        // near-dense user: stop rejecting and draw the rank-th item of the complement directly (same uniform
        // distribution over the non-train items, never a train item): smallest pos with row[pos] - pos > rank
        Philox::gen(p.seed, p.first + (uint64_t)t, 0x40000000u, r);          // a fresh block: independent of the rejected candidates
        const uint32_t rank = bounded(r[0], (uint32_t)(p.n_items - len));
        int lo = 0, hi = len;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((uint32_t)(__ldg(row + mid) - mid) > rank) hi = mid; else lo = mid + 1;
        }
        cand = (int)rank + lo;
    }
    j = cand;
}

// triple t: sampled (and written to out_* when asked), unpacked from the 8-byte host format, or read from three arrays
template <bool SAMPLE>
__device__ __forceinline__ void fetch_triple(const HogwildParams &p, int64_t t, int &u, int &i, int &j) {
    if (SAMPLE) {
        sample_triple(p, t, u, i, j);
        if (p.out_u) { p.out_u[t] = u; p.out_i[t] = i; p.out_j[t] = j; }
    } else if (p.packed) {
        const uint64_t w = __ldg(p.packed + t);
        u = (int)(w & ((1ull << p.bits_u) - 1));
        i = (int)((w >> p.bits_u) & ((1ull << p.bits_i) - 1));
        j = (int)(w >> (p.bits_u + p.bits_i));
    } else {
        u = __ldg(p.tu + t); i = __ldg(p.ti + t); j = __ldg(p.tj + t);
    }
}

// item row / bias addresses: one table, or the owner shard's (possibly peer-mapped) memory
template <bool PEER>
__device__ __forceinline__ void item_row(const HogwildParams &p, int i, float *&row, float *&bias) {
    if constexpr (PEER) {
        int o, l;
        p.shards.locate(i, o, l);
        row = p.Vp[o] + (int64_t)l * p.ld; bias = p.bp[o] + l;
    } else {
        row = p.V + (int64_t)i * p.ld; bias = p.b + i;
    }
}

template <int VPL>
struct Rows {
    float4 u[VPL], vi[VPL], vj[VPL];
    float bi, bj;
};

// ROUNDS (opt-in, flags bit 6 / deterministic=True in ops) makes the step deterministic.  The launch is cooperative and runs in
// rounds: every warp loads the rows of UNR triples per lane group, computes their updates from those values, the whole grid
// waits, every warp adds its updates, the grid waits again.  A triple therefore reads exactly the values left by the
// previous rounds — which round a triple falls into is fixed by its index and the grid size, not by timing — so the same
// inputs give the same tables on every run (up to the order in which one round's atomic adds to a shared row land, i.e.
// fp32 rounding).  Staleness stays bounded by one round (the grid's lane groups x UNR triples).  The barriers cost
// throughput (the row loads of one round no longer overlap the previous round's atomics), so the default is free-running
// Hogwild; rounds exist for local tables with atomic updates only.
template <int DP, bool SAMPLE, bool ATOMIC, bool PEER, bool ROUNDS = false>
__global__ void __launch_bounds__(256) bpr_hogwild_kernel(const HogwildParams p) {
    static_assert(!ROUNDS || (ATOMIC && !PEER), "deterministic rounds: local tables, atomic updates");
    constexpr int NV = DP / 4;                 // float4 per row
    constexpr int G = NV >= 32 ? 32 : NV;      // lanes per triple
    constexpr int VPL = NV / G;                // float4 per lane
    const int lane = threadIdx.x & 31;
    const int gl = lane % G;
    const int gbase = lane - gl;
    const int64_t warp_id = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t ld = p.ld;
    float loss_acc = 0.f;

    auto load_rows = [&](Rows<VPL> &r, int u, int i, int j) {
        if (u >= 0) {
            float *ri, *rj, *bi, *bj;
            item_row<PEER>(p, i, ri, bi); item_row<PEER>(p, j, rj, bj);
            const float4 *pu = reinterpret_cast<const float4 *>(p.U + (int64_t)u * ld);
            const float4 *pi = reinterpret_cast<const float4 *>(ri);
            const float4 *pj = reinterpret_cast<const float4 *>(rj);
#pragma unroll
            for (int v = 0; v < VPL; v++) {
                r.u[v] = pu[v * G + gl];
                r.vi[v] = PEER ? ld_sys_v4(pi + v * G + gl) : pi[v * G + gl];
                r.vj[v] = PEER ? ld_sys_v4(pj + v * G + gl) : pj[v * G + gl];
            }
            r.bi = *bi;
            r.bj = *bj;
        }
    };

    // ROUNDS: every warp runs the same number of iterations (idle ones with u = -1), so all of them reach every grid barrier
    const int64_t n_tiles = (p.n + 31) / 32;
    const int64_t tile_end = ROUNDS ? (n_tiles + nwarps - 1) / nwarps * nwarps : n_tiles;
    for (int64_t tile = warp_id; tile < tile_end; tile += nwarps) {
        const int64_t t = tile * 32 + lane;
        int u = -1, i = 0, j = 0;
        if (t < p.n) fetch_triple<SAMPLE>(p, t, u, i, j);
        // UNR triples of the group in flight at once: all their row loads are issued before the first reduction
        constexpr int UNR = G >= 4 ? 4 : G;
#pragma unroll 1
        for (int s0 = 0; s0 < G; s0 += UNR) {
            Rows<VPL> rw[UNR];
            int tu_[UNR], ti_[UNR], tj_[UNR];
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                tu_[q] = __shfl_sync(0xffffffffu, u, gbase + s0 + q);
                ti_[q] = __shfl_sync(0xffffffffu, i, gbase + s0 + q);
                tj_[q] = __shfl_sync(0xffffffffu, j, gbase + s0 + q);
                load_rows(rw[q], tu_[q], ti_[q], tj_[q]);
            }
            if constexpr (ROUNDS) {
                // ---- read phase: scores and updates of this round's triples from the values the previous rounds left; each
                // triple's updates overwrite its rows in rw (registers: the rows are dead once the updates are formed)
#pragma unroll
                for (int q = 0; q < UNR; q++) {
                    Rows<VPL> &cur = rw[q];
                    float part = 0.f;
                    if (tu_[q] >= 0) {
#pragma unroll
                        for (int v = 0; v < VPL; v++) part += bpr_partial_dot(cur.u[v], cur.vi[v], cur.vj[v]);
                    }
                    part = group_sum<G>(part);
                    if (tu_[q] >= 0) {
                        const float z = bpr_sigmoid_loss(part + (cur.bi - cur.bj), loss_acc, gl);
#pragma unroll
                        for (int v = 0; v < VPL; v++) {
                            float4 du, di, dj;
                            bpr_row_deltas(cur.u[v], cur.vi[v], cur.vj[v], z, p.hp, du, di, dj);
                            cur.u[v] = du; cur.vi[v] = di; cur.vj[v] = dj;
                        }
                        float dbi, dbj;
                        bpr_bias_deltas(z, cur.bi, cur.bj, p.hp, dbi, dbj);
                        cur.bi = dbi; cur.bj = dbj;
                    }
                }
                cooperative_groups::this_grid().sync();      // every read of this round is done
                // ---- write phase
#pragma unroll
                for (int q = 0; q < UNR; q++) {
                    if (tu_[q] < 0) continue;
                    float *pu = p.U + (int64_t)tu_[q] * ld, *pi, *pj, *pbi, *pbj;
                    item_row<PEER>(p, ti_[q], pi, pbi); item_row<PEER>(p, tj_[q], pj, pbj);
#pragma unroll
                    for (int v = 0; v < VPL; v++) {
                        const int e = (v * G + gl) * 4;
                        red_add_v4(pu + e, rw[q].u[v]);
                        red_add_v4(pi + e, rw[q].vi[v]);
                        red_add_v4(pj + e, rw[q].vj[v]);
                    }
                    if (gl == 0) { red_add_f32(pbi, rw[q].bi); red_add_f32(pbj, rw[q].bj); }
                }
                cooperative_groups::this_grid().sync();      // every write of this round has landed before the next reads
                continue;
            }
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                const Rows<VPL> &cur = rw[q];
                const int cu = tu_[q], ci = ti_[q], cj = tj_[q];
                float part = 0.f;
                if (cu >= 0) {
#pragma unroll
                    for (int v = 0; v < VPL; v++) part += bpr_partial_dot(cur.u[v], cur.vi[v], cur.vj[v]);
                }
                part = group_sum<G>(part);
                if (cu >= 0) {
                    const float z = bpr_sigmoid_loss(part + (cur.bi - cur.bj), loss_acc, gl);
                    float *pu = p.U + (int64_t)cu * ld, *pi, *pj, *pbi, *pbj;
                    item_row<PEER>(p, ci, pi, pbi); item_row<PEER>(p, cj, pj, pbj);
#pragma unroll
                    for (int v = 0; v < VPL; v++) {
                        const float4 a = cur.u[v], vi = cur.vi[v], vj = cur.vj[v];
                        float4 du, di, dj;
                        bpr_row_deltas(a, vi, vj, z, p.hp, du, di, dj);
                        const int e = (v * G + gl) * 4;
                        if (PEER) {
                            red_add_v4(pu + e, du);
                            if (!p.no_item_updates) {
                                red_add_v4_sys(pi + e, di);
                                red_add_v4_sys(pj + e, dj);
                            }
                        } else if (ATOMIC) {
                            red_add_v4(pu + e, du);
                            red_add_v4(pi + e, di);
                            red_add_v4(pj + e, dj);
                        } else {
                            *reinterpret_cast<float4 *>(pu + e) = make_float4(a.x + du.x, a.y + du.y, a.z + du.z, a.w + du.w);
                            *reinterpret_cast<float4 *>(pi + e) = make_float4(vi.x + di.x, vi.y + di.y, vi.z + di.z, vi.w + di.w);
                            *reinterpret_cast<float4 *>(pj + e) = make_float4(vj.x + dj.x, vj.y + dj.y, vj.z + dj.z, vj.w + dj.w);
                        }
                    }
                    if (gl == 0) {
                        float dbi, dbj;
                        bpr_bias_deltas(z, cur.bi, cur.bj, p.hp, dbi, dbj);
                        if (PEER) { red_add_f32_sys(pbi, dbi); red_add_f32_sys(pbj, dbj); }
                        else if (ATOMIC) { red_add_f32(pbi, dbi); red_add_f32(pbj, dbj); }
                        else { *pbi = cur.bi + dbi; *pbj = cur.bj + dbj; }
                    }
                }
            }
        }
    }
    if (p.loss) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, off);
        if (lane == 0 && loss_acc != 0.f) atomicAdd(p.loss, (double)loss_acc);
    }
}

// ---------------------------------------------------------------- grouped sampled step (local tables, free-running)
// The sampled step on local tables applies its triples grouped by user.  user_key_kernel writes the user every triple will
// draw, a stable radix sort orders the triple indices by it, and bpr_grouped_kernel walks the sorted indices: a warp takes a
// window of 32 consecutive entries, each lane samples ITS triple t (same Philox draw as sample order, emitted at index t), and
// each lane group walks a contiguous slice of the window in order.  The group keeps the current user row in registers (`cur`,
// which triple k+1 of a run reads as triple k left it) and the run's summed update (`acc`), and adds acc to U once per run
// and slice.  So a visited user row is read and written about once per step instead of once per triple, in ascending
// address order, and the sampler's CSR row and indptr loads of one user are shared through L1.  Item rows and biases keep
// their per-triple vector atomics.  A run of one triple performs exactly the per-triple kernel's arithmetic.
__global__ void __launch_bounds__(256) user_key_kernel(const HogwildParams p, uint32_t *__restrict__ key, int32_t *__restrict__ val) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; t < p.n; t += stride) {
        uint32_t r[4];
        int u, len;
        int64_t beg;
        sample_user(p, t, r, u, beg, len);
        key[t] = (uint32_t)u; val[t] = (int32_t)t;
    }
}

template <int DP, bool ATOMIC>
__global__ void __launch_bounds__(256) bpr_grouped_kernel(const HogwildParams p) {
    constexpr int NV = DP / 4;                 // float4 per row
    constexpr int G = NV >= 32 ? 32 : NV;      // lanes per triple
    constexpr int VPL = NV / G;                // float4 per lane
    constexpr int UNR = G >= 4 ? 4 : G;        // triples of the slice whose rows are in flight at once
    const int lane = threadIdx.x & 31;
    const int gl = lane % G;
    const int gbase = lane - gl;
    const int64_t warp_id = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t ld = p.ld;
    float loss_acc = 0.f;

    const int64_t n_tiles = (p.n + 31) / 32;
    for (int64_t tile = warp_id; tile < n_tiles; tile += nwarps) {
        const int64_t pos = tile * 32 + lane;
        int u = -1, i = 0, j = 0;
        if (pos < p.n) fetch_triple<true>(p, __ldg(p.order + pos), u, i, j);
        // the group's run: user cu (-1: none yet), its row as the run left it, the run's summed update
        int cu = -1;
        float4 cur[VPL], acc[VPL];
        auto flush = [&]() {
            float *pu = p.U + (int64_t)cu * ld;
#pragma unroll
            for (int v = 0; v < VPL; v++) {
                float *e = pu + (v * G + gl) * 4;
                if (ATOMIC) red_add_v4(e, acc[v]);
                else *reinterpret_cast<float4 *>(e) = cur[v];
            }
        };
#pragma unroll 1
        for (int s0 = 0; s0 < G; s0 += UNR) {
            Rows<VPL> rw[UNR];
            int tu_[UNR], ti_[UNR], tj_[UNR];
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                tu_[q] = __shfl_sync(0xffffffffu, u, gbase + s0 + q);
                ti_[q] = __shfl_sync(0xffffffffu, i, gbase + s0 + q);
                tj_[q] = __shfl_sync(0xffffffffu, j, gbase + s0 + q);
                if (tu_[q] >= 0) {
                    // the user row only where a run starts: inside a run the row is `cur`
                    if (tu_[q] != (q == 0 ? cu : tu_[q - 1])) {
                        const float4 *pu = reinterpret_cast<const float4 *>(p.U + (int64_t)tu_[q] * ld);
#pragma unroll
                        for (int v = 0; v < VPL; v++) rw[q].u[v] = pu[v * G + gl];
                    }
                    const float4 *pi = reinterpret_cast<const float4 *>(p.V + (int64_t)ti_[q] * ld);
                    const float4 *pj = reinterpret_cast<const float4 *>(p.V + (int64_t)tj_[q] * ld);
#pragma unroll
                    for (int v = 0; v < VPL; v++) { rw[q].vi[v] = pi[v * G + gl]; rw[q].vj[v] = pj[v * G + gl]; }
                    rw[q].bi = p.b[ti_[q]];
                    rw[q].bj = p.b[tj_[q]];
                }
            }
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                const Rows<VPL> &nx = rw[q];
                const int qu = tu_[q], qi = ti_[q], qj = tj_[q];
                const bool start = qu != cu;                       // group-uniform
                if (start) {
                    if (cu >= 0) flush();
                    cu = qu;
#pragma unroll
                    for (int v = 0; v < VPL; v++) cur[v] = nx.u[v];
                }
                float part = 0.f;
                if (qu >= 0) {
#pragma unroll
                    for (int v = 0; v < VPL; v++) part += bpr_partial_dot(cur[v], nx.vi[v], nx.vj[v]);
                }
                part = group_sum<G>(part);
                if (qu >= 0) {
                    const float z = bpr_sigmoid_loss(part + (nx.bi - nx.bj), loss_acc, gl);
                    float *pi = p.V + (int64_t)qi * ld, *pj = p.V + (int64_t)qj * ld;
#pragma unroll
                    for (int v = 0; v < VPL; v++) {
                        const float4 a = cur[v], vi = nx.vi[v], vj = nx.vj[v];
                        float4 du, di, dj;
                        bpr_row_deltas(a, vi, vj, z, p.hp, du, di, dj);
                        cur[v] = make_float4(a.x + du.x, a.y + du.y, a.z + du.z, a.w + du.w);
                        acc[v] = start ? du : make_float4(acc[v].x + du.x, acc[v].y + du.y, acc[v].z + du.z, acc[v].w + du.w);
                        const int e = (v * G + gl) * 4;
                        if (ATOMIC) {
                            red_add_v4(pi + e, di);
                            red_add_v4(pj + e, dj);
                        } else {
                            *reinterpret_cast<float4 *>(pi + e) = make_float4(vi.x + di.x, vi.y + di.y, vi.z + di.z, vi.w + di.w);
                            *reinterpret_cast<float4 *>(pj + e) = make_float4(vj.x + dj.x, vj.y + dj.y, vj.z + dj.z, vj.w + dj.w);
                        }
                    }
                    if (gl == 0) {
                        float dbi, dbj;
                        bpr_bias_deltas(z, nx.bi, nx.bj, p.hp, dbi, dbj);
                        if (ATOMIC) { red_add_f32(p.b + qi, dbi); red_add_f32(p.b + qj, dbj); }
                        else { p.b[qi] = nx.bi + dbi; p.b[qj] = nx.bj + dbj; }
                    }
                }
            }
        }
        if (cu >= 0) flush();
    }
    if (p.loss) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, off);
        if (lane == 0 && loss_acc != 0.f) atomicAdd(p.loss, (double)loss_acc);
    }
}

// ---------------------------------------------------------------- staged variant of the Hogwild kernel (PEER mode only)
// Same update, same sampler, same atomics as bpr_hogwild_kernel<..., PEER = true>; the difference is HOW the three
// embedding rows of a triple reach the SM.  There every lane group loads "its" rows into registers (4 triples in flight per group, 118
// registers, 16 warps/SM) and the loads of a round cannot start before the previous round's arithmetic has retired.
// Here every lane, as soon as it has sampled its triple, hands the three rows to the copy engine
// (cp.async.bulk global -> shared, completion on a per-warp mbarrier): 3 x TT row copies per warp are in flight with NO
// register cost, the groups then read the rows from shared memory (conflict-free 128-bit loads).  That is the
// "128-bit row loads staged through shared memory" layout of the north_star, and it is what lets rows that live in a
// PEER GPU's memory (PEER mode: 2-3x the latency of local HBM) arrive without stalling the arithmetic.
// TT rows-triples per warp chunk: 12 KB of shared memory per warp whatever the row length (DP = 32/64/128 floats); halving the
// chunk to fit 4 CTAs per SM was measured SLOWER (1.32 vs 1.01 ms at C2): the step is not short of resident warps.
constexpr int STAGE_CHUNK_BYTES = 4096;
template <int DP, bool SAMPLE>
__global__ void __launch_bounds__(256) bpr_hogwild_stage_kernel(const HogwildParams p) {
    constexpr int NV = DP / 4;                 // float4 per row
    constexpr int G = NV >= 32 ? 32 : NV;      // lanes per triple
    constexpr int VPL = NV / G;                // float4 per lane
    constexpr int ROWB = DP * 4;
    constexpr int TT = STAGE_CHUNK_BYTES / ROWB;  // triples per chunk (32 / 16 / 8 at 4 KB of rows per row kind)
    constexpr int NGRP = 32 / G;               // triples processed side by side
    static_assert(TT >= NGRP && TT <= 32 && 32 % TT == 0, "chunk shape");
    extern __shared__ __align__(128) uint8_t stage_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int gl = lane % G, grp = lane / G;
    uint8_t *wbuf = stage_smem + (size_t)wib * (TT * 3 * ROWB);          // [TT][3][ROWB]
    uint64_t *bars = reinterpret_cast<uint64_t *>(stage_smem + (size_t)(blockDim.x >> 5) * (TT * 3 * ROWB));
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(bars + wib);
    const uint32_t wbuf_s = (uint32_t)__cvta_generic_to_shared(wbuf);
    if (lane == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(1) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    uint32_t phase = 0;
    const int64_t warp_id = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t ld = p.ld;
    float loss_acc = 0.f;

    for (int64_t tile = warp_id; tile * 32 < p.n; tile += nwarps) {
        const int64_t t = tile * 32 + lane;
        int u = -1, i = 0, j = 0;
        float bi = 0.f, bj = 0.f;
        float *pu = nullptr, *pi = nullptr, *pj = nullptr, *pbi = nullptr, *pbj = nullptr;
        if (t < p.n) {
            fetch_triple<SAMPLE>(p, t, u, i, j);
            pu = p.U + (int64_t)u * ld;
            item_row<true>(p, i, pi, pbi); item_row<true>(p, j, pj, pbj);
        }
        const bool valid = u >= 0;
#pragma unroll 1
        for (int c0 = 0; c0 < 32; c0 += TT) {
            const bool mine = valid && lane >= c0 && lane < c0 + TT;
            const uint32_t nmine = (uint32_t)__popc(__ballot_sync(0xffffffffu, mine));
            if (nmine == 0) continue;                                              // warp-uniform
            // the previous chunk's shared-memory reads (generic proxy) are done before the copy engine overwrites the buffer
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0)
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(nmine * 3u * (uint32_t)ROWB) : "memory");
            __syncwarp();
            if (mine) {
                const uint32_t dst = wbuf_s + (uint32_t)(lane - c0) * (3u * ROWB);
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(dst), "l"(pu), "r"(ROWB), "r"(bar) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(dst + ROWB), "l"(pi), "r"(ROWB), "r"(bar) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(dst + 2 * ROWB), "l"(pj), "r"(ROWB), "r"(bar) : "memory");
                bi = *pbi; bj = *pbj;                                              // biases ride in registers
            }
            {   // wait for the chunk's 3 * nmine rows
                uint32_t ok;
                do {
                    asm volatile("{\n\t.reg .pred q;\n\tmbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\n\tselp.u32 %0, 1, 0, q;\n\t}"
                                 : "=r"(ok) : "r"(bar), "r"(phase) : "memory");
                } while (!ok);
                phase ^= 1;
            }
#pragma unroll 1
            for (int s = 0; s < TT; s += NGRP) {
                const int q = s + grp;                                             // triple slot inside the chunk
                const int src = c0 + q;                                            // lane that sampled it
                const int cu = __shfl_sync(0xffffffffu, u, src), ci = __shfl_sync(0xffffffffu, i, src), cj = __shfl_sync(0xffffffffu, j, src);
                const float cbi = __shfl_sync(0xffffffffu, bi, src), cbj = __shfl_sync(0xffffffffu, bj, src);
                const bool on = cu >= 0;
                const float4 *su = reinterpret_cast<const float4 *>(wbuf + (size_t)q * (3 * ROWB));
                float4 a[VPL], vi[VPL], vj[VPL];
                float part = 0.f;
#pragma unroll
                for (int v = 0; v < VPL; v++) {
                    a[v] = su[v * G + gl]; vi[v] = su[NV + v * G + gl]; vj[v] = su[2 * NV + v * G + gl];
                    part += bpr_partial_dot(a[v], vi[v], vj[v]);
                }
                if (!on) part = 0.f;
                part = group_sum<G>(part);
                if (on) {
                    const float z = bpr_sigmoid_loss(part + (cbi - cbj), loss_acc, gl);
                    float *gu = p.U + (int64_t)cu * ld, *gi, *gj, *gbi, *gbj;
                    item_row<true>(p, ci, gi, gbi); item_row<true>(p, cj, gj, gbj);
#pragma unroll
                    for (int v = 0; v < VPL; v++) {
                        float4 du, di, dj;
                        bpr_row_deltas(a[v], vi[v], vj[v], z, p.hp, du, di, dj);
                        const int e = (v * G + gl) * 4;
                        red_add_v4(gu + e, du);
                        if (!p.no_item_updates) { red_add_v4_sys(gi + e, di); red_add_v4_sys(gj + e, dj); }
                    }
                    if (gl == 0) {
                        float dbi, dbj;
                        bpr_bias_deltas(z, cbi, cbj, p.hp, dbi, dbj);
                        red_add_f32_sys(gbi, dbi); red_add_f32_sys(gbj, dbj);
                    }
                }
            }
        }
    }
    if (p.loss) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) loss_acc += __shfl_xor_sync(0xffffffffu, loss_acc, off);
        if (lane == 0 && loss_acc != 0.f) atomicAdd(p.loss, (double)loss_acc);
    }
}

// Persistent grid of 256-thread CTAs: one CTA per 8 tiles of 32 triples (a tile per warp), at most what stays resident on the
// SMs left after `reserve_sms` (SMs left free for a concurrent collective (NCCL) kernel).
static int persistent_grid(const void *kern, int smem, int64_t n, int reserve_sms, unsigned &grid) {
    int per_sm = 0;
    EB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem));
    if (per_sm < 1) per_sm = 1;
    const int64_t tiles = (n + 31) / 32;
    const int64_t want = (tiles + 7) / 8;
    int sms = sm_count() - reserve_sms;
    if (sms < 1) sms = 1;
    int64_t g = (int64_t)sms * per_sm;
    if (want < g) g = want;
    grid = (unsigned)(g < 1 ? 1 : g);
    return EB_OK;
}

template <int DP, bool SAMPLE>
static int launch_stage_t(const HogwildParams &p, int reserve_sms, cudaStream_t st) {
    constexpr int SMEM = 8 * 3 * STAGE_CHUNK_BYTES + 64;   // 8 warps x 3 row kinds x chunk + mbarriers
    auto kern = bpr_hogwild_stage_kernel<DP, SAMPLE>;
    EB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    unsigned grid;
    if (int rc = persistent_grid((const void *)kern, SMEM, p.n, reserve_sms, grid)) return rc;
    kern<<<grid, 256, SMEM, st>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

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

__global__ void __launch_bounds__(256) philox_sample_kernel(const HogwildParams p) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; t < p.n; t += stride) {
        int u, i, j;
        sample_triple(p, t, u, i, j);
        p.out_u[t] = u; p.out_i[t] = i; p.out_j[t] = j;
    }
}

// pointwise_pos_neg_sampler.py:24-48: u uniform; one fair bit decides between a uniform train item of u (label 1) and a
// uniform non-train item (label 0).  The BPR sampler already draws both for u: keep one of them.
__global__ void __launch_bounds__(256) pointwise_sample_kernel(const HogwildParams p, float *__restrict__ out_label) {
    int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; t < p.n; t += stride) {
        int u, i, j;
        sample_triple(p, t, u, i, j);
        uint32_t r[4];
        Philox::gen(p.seed, p.first + (uint64_t)t, 0x20000000u, r);
        const bool pos = (r[0] >> 31) != 0;
        p.out_u[t] = u; p.out_i[t] = pos ? i : j; out_label[t] = pos ? 1.f : 0.f;
    }
}

template <int DP, bool SAMPLE, bool ATOMIC, bool PEER, bool ROUNDS>
static int launch_hogwild_t(const HogwildParams &p, int reserve_sms, cudaStream_t st) {
    auto kern = bpr_hogwild_kernel<DP, SAMPLE, ATOMIC, PEER, ROUNDS>;
    unsigned grid;
    if (int rc = persistent_grid((const void *)kern, 0, p.n, reserve_sms, grid)) return rc;
    if (ROUNDS) {
        // deterministic rounds (see bpr_hogwild_kernel): a cooperative launch, so every CTA is resident for the grid barriers
        void *args[] = {const_cast<HogwildParams *>(&p)};
        EB_CUDA(cudaLaunchCooperativeKernel((const void *)kern, dim3(grid), dim3(256), args, 0, st));
    } else {
        kern<<<grid, 256, 0, st>>>(p);
    }
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

// f(std::integral_constant<int, DP>{}) for the row stride DP == dp among the compiled ones (DPS), else EB_ERR_ARG
template <int... DPS, class F>
static int with_stride(int dp, const char *strides, F &&f) {
    int rc = EB_OK;
    const bool found = ((dp == DPS && (rc = f(std::integral_constant<int, DPS>{}), true)) || ...);
    return found ? rc : set_err(EB_ERR_ARG, "row stride ld=%d must be one of %s", dp, strides);
}

// EB_L2_PERSIST=1: mark the item table's address range as persisting in L2 for the launch's stream (cudaAccessPolicyWindow) when it
// fits the device's persisting carve-out — the table is hit by two of every triple's three row accesses, the user table and the
// CSR are streamed once.  An A/B switch, off by default.
static void item_table_l2_window(const HogwildParams &p, cudaStream_t st) {
    static const int env = [] { const char *e = getenv("EB_L2_PERSIST"); return e ? atoi(e) : 0; }();
    if (!env || !p.V) return;
    static int max_persist = -1, max_window = 0;
    if (max_persist < 0) {
        int dev = 0; cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, dev);
        cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, dev);
    }
    const size_t bytes = (size_t)p.n_items * (size_t)p.ld * sizeof(float);
    if (max_persist <= 0 || bytes > (size_t)max_persist || bytes > (size_t)max_window) return;
    static size_t carved = 0;                 // the carve-out is sized to the table, not to the device maximum
    if (carved != bytes) { cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, bytes); carved = bytes; }
    cudaStreamAttrValue attr{};
    attr.accessPolicyWindow.base_ptr = (void *)p.V;
    attr.accessPolicyWindow.num_bytes = bytes;
    attr.accessPolicyWindow.hitRatio = 1.0f;
    attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr.accessPolicyWindow.missProp = env == 2 ? cudaAccessPropertyNormal : cudaAccessPropertyStreaming;
    cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &attr);
}

template <int DP, bool ATOMIC>
static int launch_grouped_t(const HogwildParams &p, int reserve_sms, cudaStream_t st) {
    auto kern = bpr_grouped_kernel<DP, ATOMIC>;
    unsigned grid;
    if (int rc = persistent_grid((const void *)kern, 0, p.n, reserve_sms, grid)) return rc;
    kern<<<grid, 256, 0, st>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

static int bits_for(uint64_t v) { int b = 1; while ((v >> b) != 0) b++; return b; }

// The grouped step sorts the triple indices of at most GROUP_MAX triples at a time (int32 offsets); longer calls run as
// consecutive sub-steps of that size.
constexpr int64_t GROUP_MAX = (int64_t)INT32_MAX;

struct GroupLayout {
    size_t key_a, key_b, val_a, val_b, cub, cub_bytes, total;
};

// 16 B per triple (user keys and triple indices, each double-buffered for the sort) + cub's temporary storage
static GroupLayout group_layout(int64_t n, int32_t n_users) {
    const int64_t m = n < GROUP_MAX ? n : GROUP_MAX;
    GroupLayout L;
    size_t off = 0;
    L.key_a = off; off += align_up(sizeof(uint32_t) * (size_t)m);
    L.key_b = off; off += align_up(sizeof(uint32_t) * (size_t)m);
    L.val_a = off; off += align_up(sizeof(int32_t) * (size_t)m);
    L.val_b = off; off += align_up(sizeof(int32_t) * (size_t)m);
    cub::DoubleBuffer<uint32_t> keys(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> vals(nullptr, nullptr);
    size_t cb = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, cb, keys, vals, (int)m, 0, bits_for((uint64_t)n_users));
    L.cub_bytes = cb;
    L.cub = off; off += align_up(cb);
    L.total = off;
    return L;
}

// The schedule of one sub-step (p.n <= GROUP_MAX): the user keys and the stable sort of the triple indices by user.  Reads
// only seed, first, n, n_users, n_items and indptr, never the tables.  The ordered indices end up in one of the workspace's two
// index buffers (cub's double buffer decides which): `order` points at it.  The key pass leaves `reserve` SMs free; cub's
// sort kernels size their own grids.
static int schedule_grouped(const HogwildParams &p, int reserve, char *ws, const GroupLayout &L, cudaStream_t st,
                            const int32_t *&order) {
    int sms = sm_count() - reserve;
    if (sms < 1) sms = 1;
    cub::DoubleBuffer<uint32_t> keys((uint32_t *)(ws + L.key_a), (uint32_t *)(ws + L.key_b));
    cub::DoubleBuffer<int32_t> vals((int32_t *)(ws + L.val_a), (int32_t *)(ws + L.val_b));
    int64_t grid = (p.n + 255) / 256;
    if (grid > (int64_t)sms * 8) grid = (int64_t)sms * 8;
    user_key_kernel<<<(unsigned)grid, 256, 0, st>>>(p, keys.Current(), vals.Current());
    EB_CUDA(cudaGetLastError());
    size_t cb = L.cub_bytes;
    EB_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.cub, cb, keys, vals, (int)p.n, 0, bits_for((uint64_t)p.n_users), st));
    order = vals.Current();
    return EB_OK;
}

// Sampled step on local tables, free-running: per sub-step, the schedule above, then the grouped update (which leaves
// `reserve` SMs free).
template <int DP, bool ATOMIC>
static int launch_grouped(HogwildParams p, int reserve, char *ws, const GroupLayout &L, cudaStream_t st) {
    const int64_t n = p.n;
    const uint64_t first = p.first;
    int32_t *out_u = p.out_u, *out_i = p.out_i, *out_j = p.out_j;
    for (int64_t c0 = 0; c0 < n; c0 += GROUP_MAX) {
        p.n = n - c0 < GROUP_MAX ? n - c0 : GROUP_MAX;
        p.first = first + (uint64_t)c0;
        if (out_u) { p.out_u = out_u + c0; p.out_i = out_i + c0; p.out_j = out_j + c0; }
        if (int rc = schedule_grouped(p, reserve, ws, L, st, p.order)) return rc;
        if (int rc = launch_grouped_t<DP, ATOMIC>(p, reserve, st)) return rc;
    }
    return EB_OK;
}

// SAMPLE: the sampled step; free-running on local tables it runs grouped by user (ws: eb_bpr_step_sampled_workspace_bytes)
template <bool SAMPLE>
static int launch_hogwild(const HogwildParams &p, int dp, int flags, cudaStream_t st, void *ws = nullptr, size_t ws_bytes = 0) {
    const bool atomic = !(flags & 1);
    const bool rounds = (flags & 64) != 0;
    const int reserve = (flags >> 8) & 0xff;
    EB_ARG(!(flags & 32), "the shared-memory-staged kernel exists for sharded item tables only");
    EB_ARG(atomic || !rounds, "deterministic rounds run with atomic updates");
    if constexpr (SAMPLE) {
        if (!rounds) {
            const GroupLayout L = group_layout(p.n, p.n_users);
            if (!ws || ws_bytes < L.total) return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", ws ? ws_bytes : 0, L.total);
            // the row stride is checked before anything is launched
            return with_stride<8, 16, 32, 64, 128, 256>(dp, "8,16,32,64,128,256 floats", [&](auto dpc) {
                constexpr int DP = decltype(dpc)::value;
                item_table_l2_window(p, st);
                return atomic ? launch_grouped<DP, true>(p, reserve, (char *)ws, L, st)
                              : launch_grouped<DP, false>(p, reserve, (char *)ws, L, st);
            });
        }
    }
    item_table_l2_window(p, st);
    return with_stride<8, 16, 32, 64, 128, 256>(dp, "8,16,32,64,128,256 floats", [&](auto dpc) {
        constexpr int DP = decltype(dpc)::value;
        if constexpr (!SAMPLE) {
            if (!rounds) return atomic ? launch_hogwild_t<DP, false, true, false, false>(p, reserve, st)
                                       : launch_hogwild_t<DP, false, false, false, false>(p, reserve, st);
        }
        return launch_hogwild_t<DP, SAMPLE, true, false, true>(p, reserve, st);   // deterministic rounds
    });
}

// The grouped update alone, on an order the caller scheduled (p.order, p.n <= GROUP_MAX)
static int launch_apply(const HogwildParams &p, int dp, int flags, cudaStream_t st) {
    const bool atomic = !(flags & 1);
    const int reserve = (flags >> 8) & 0xff;
    EB_ARG(!(flags & (32 | 64)), "the grouped update runs free-running on local tables (no rounds, no staged kernel)");
    return with_stride<8, 16, 32, 64, 128, 256>(dp, "8,16,32,64,128,256 floats", [&](auto dpc) {
        constexpr int DP = decltype(dpc)::value;
        item_table_l2_window(p, st);
        return atomic ? launch_grouped_t<DP, true>(p, reserve, st) : launch_grouped_t<DP, false>(p, reserve, st);
    });
}

// PEER mode: atomics only (other GPUs update the same rows), strides the sharded configurations use.  The shared-memory-staged
// kernel is the default (its row copies are in flight without holding registers while the rows cross NVLink); flags bit 4 (16),
// or bit 0, selects the register kernel (whose peer updates stay atomic).
template <bool SAMPLE>
static int launch_hogwild_peer(const HogwildParams &p, int dp, int flags, cudaStream_t st) {
    const int reserve = (flags >> 8) & 0xff;
    EB_ARG(!(flags & 64), "deterministic rounds exist for local tables only (other GPUs update peer rows concurrently)");
    const bool stage = !(flags & (1 | 16));
    return with_stride<32, 64, 128>(dp, "32,64,128 floats for sharded item tables", [&](auto dpc) {
        constexpr int DP = decltype(dpc)::value;
        return stage ? launch_stage_t<DP, SAMPLE>(p, reserve, st) : launch_hogwild_t<DP, SAMPLE, true, true, false>(p, reserve, st);
    });
}

static int fill_peer(HogwildParams &p, float *const *V_shards, float *const *b_shards, int n_shards, int32_t shard_rows,
                     int32_t n_items) {
    EB_ARG(V_shards && b_shards && n_shards >= 1 && n_shards <= EB_MAX_PEERS, "1 <= n_shards <= %d", EB_MAX_PEERS);
    EB_ARG(shard_rows >= 1 && (int64_t)shard_rows * n_shards >= n_items, "shards do not cover the item range");
    for (int s = 0; s < n_shards; s++) {
        EB_ARG(V_shards[s] && b_shards[s] && ((uintptr_t)V_shards[s] % 16) == 0, "null / misaligned shard pointer %d", s);
        p.Vp[s] = V_shards[s]; p.bp[s] = b_shards[s];
    }
    for (int s = n_shards; s < EB_MAX_PEERS; s++) { p.Vp[s] = V_shards[0]; p.bp[s] = b_shards[0]; }
    p.shards = shard_map(shard_rows);
    return EB_OK;
}

static int check_tables(const void *U, const void *V, const void *b, int d, int ld) {
    EB_ARG(U && V && b, "null table pointer");
    EB_ARG(d >= 1 && ld >= d, "need 1 <= d <= ld (d=%d ld=%d)", d, ld);
    EB_ARG(((uintptr_t)U % 16) == 0 && ((uintptr_t)V % 16) == 0, "tables must be 16-byte aligned");
    return EB_OK;
}

// ---------------------------------------------------------------- exact mode (fp64)
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

extern "C" int eb_bpr_step_f32(float *U, float *V, float *item_bias, int d, int ld, const int32_t *tu,
                               const int32_t *ti, const int32_t *tj, int64_t n, float lr, float reg_u, float reg_b,
                               float reg_pos, float reg_neg, double *loss, int flags, void *stream) {
    if (int rc = check_tables(U, V, item_bias, d, ld)) return rc;
    EB_ARG(n >= 0, "n < 0");
    if (n == 0) return EB_OK;
    EB_ARG(tu && ti && tj, "null triple arrays");
    HogwildParams p{};
    p.U = U; p.V = V; p.b = item_bias; p.ld = ld; p.tu = tu; p.ti = ti; p.tj = tj; p.n = n;
    p.hp = {lr, reg_u, reg_b, reg_pos, reg_neg}; p.loss = loss;
    return launch_hogwild<false>(p, ld, flags, (cudaStream_t)stream);
}

static int set_filter(HogwildParams &p, const uint32_t *filter, int filter_words) {
    if (!filter) return EB_OK;
    EB_ARG(filter_words >= 1 && filter_words <= 1024 && (filter_words & (filter_words - 1)) == 0,
           "filter_words must be a power of two in [1, 1024] (got %d)", filter_words);
    int lb = 5;
    while ((1 << (lb - 5)) < filter_words) lb++;
    p.filter = filter; p.filter_log2bits = lb;
    return EB_OK;
}

extern "C" int eb_bloom_build(const int64_t *csr_indptr, const int32_t *csr_indices, int32_t n_users, int filter_words,
                              uint32_t *out, void *stream) {
    EB_ARG(csr_indptr && csr_indices && out && n_users >= 1, "bad argument");
    HogwildParams p{};
    if (int rc = set_filter(p, out, filter_words)) return rc;
    int64_t grid = ((int64_t)n_users * 32 + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    bloom_build_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(csr_indptr, csr_indices, n_users, p.filter_log2bits, out);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_bpr_step_sampled_f32(float *U, float *V, float *item_bias, int d, int ld, int32_t n_users,
                                       int32_t n_items, const int64_t *csr_indptr, const int32_t *csr_indices,
                                       int64_t n, uint64_t seed, uint64_t first_triple, float lr, float reg_u,
                                       float reg_b, float reg_pos, float reg_neg, double *loss, int32_t *out_u,
                                       int32_t *out_i, int32_t *out_j, void *workspace, size_t workspace_bytes, int flags,
                                       void *stream) {
    return eb_bpr_step_sampled_filter_f32(U, V, item_bias, d, ld, n_users, n_items, csr_indptr, csr_indices, nullptr, 0, n, seed,
                                          first_triple, lr, reg_u, reg_b, reg_pos, reg_neg, loss, out_u, out_i, out_j, workspace,
                                          workspace_bytes, flags, stream);
}

extern "C" size_t eb_bpr_step_sampled_workspace_bytes(int64_t n, int32_t n_users) {
    if (n <= 0 || n_users <= 0) return 256;
    return group_layout(n, n_users).total;
}

extern "C" int eb_bpr_step_sampled_filter_f32(float *U, float *V, float *item_bias, int d, int ld, int32_t n_users,
                                              int32_t n_items, const int64_t *csr_indptr, const int32_t *csr_indices,
                                              const uint32_t *filter, int filter_words, int64_t n, uint64_t seed,
                                              uint64_t first_triple, float lr, float reg_u, float reg_b, float reg_pos,
                                              float reg_neg, double *loss, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                                              void *workspace, size_t workspace_bytes, int flags, void *stream) {
    if (int rc = check_tables(U, V, item_bias, d, ld)) return rc;
    EB_ARG(n >= 0 && n_users > 0 && n_items > 1, "bad sizes");
    EB_ARG(csr_indptr && csr_indices, "null CSR");
    EB_ARG((!out_u && !out_i && !out_j) || (out_u && out_i && out_j), "out_u/out_i/out_j: all or none");
    if (n == 0) return EB_OK;
    HogwildParams p{};
    p.U = U; p.V = V; p.b = item_bias; p.ld = ld; p.n = n;
    p.hp = {lr, reg_u, reg_b, reg_pos, reg_neg}; p.loss = loss;
    p.n_users = n_users; p.n_items = n_items; p.indptr = csr_indptr; p.indices = csr_indices;
    p.seed = seed; p.first = first_triple; p.out_u = out_u; p.out_i = out_i; p.out_j = out_j;
    if (int rc = set_filter(p, filter, filter_words)) return rc;
    return launch_hogwild<true>(p, ld, flags, (cudaStream_t)stream, workspace, workspace_bytes);
}

extern "C" int eb_bpr_schedule_sampled(int32_t n_users, int32_t n_items, const int64_t *csr_indptr, int64_t n, uint64_t seed,
                                       uint64_t first_triple, void *workspace, size_t workspace_bytes, size_t *order_offset,
                                       int flags, void *stream) {
    EB_ARG(n >= 1 && n <= GROUP_MAX && n_users > 0 && n_items > 1, "bad sizes (a schedule covers 1..%lld triples)",
           (long long)GROUP_MAX);
    EB_ARG(csr_indptr && order_offset, "null pointer");
    const GroupLayout L = group_layout(n, n_users);
    if (!workspace || workspace_bytes < L.total)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace ? workspace_bytes : 0, L.total);
    HogwildParams p{};
    p.n = n; p.n_users = n_users; p.n_items = n_items; p.indptr = csr_indptr; p.seed = seed; p.first = first_triple;
    const int32_t *order = nullptr;
    if (int rc = schedule_grouped(p, (flags >> 8) & 0xff, (char *)workspace, L, (cudaStream_t)stream, order)) return rc;
    *order_offset = (size_t)((const char *)order - (const char *)workspace);
    return EB_OK;
}

extern "C" int eb_bpr_apply_sampled_filter_f32(float *U, float *V, float *item_bias, int d, int ld, int32_t n_users,
                                               int32_t n_items, const int64_t *csr_indptr, const int32_t *csr_indices,
                                               const uint32_t *filter, int filter_words, int64_t n, uint64_t seed,
                                               uint64_t first_triple, float lr, float reg_u, float reg_b, float reg_pos,
                                               float reg_neg, double *loss, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                                               const int32_t *order, int flags, void *stream) {
    if (int rc = check_tables(U, V, item_bias, d, ld)) return rc;
    EB_ARG(n >= 1 && n <= GROUP_MAX && n_users > 0 && n_items > 1, "bad sizes (an apply covers 1..%lld triples)",
           (long long)GROUP_MAX);
    EB_ARG(csr_indptr && csr_indices && order, "null CSR or order");
    EB_ARG((!out_u && !out_i && !out_j) || (out_u && out_i && out_j), "out_u/out_i/out_j: all or none");
    HogwildParams p{};
    p.U = U; p.V = V; p.b = item_bias; p.ld = ld; p.n = n;
    p.hp = {lr, reg_u, reg_b, reg_pos, reg_neg}; p.loss = loss;
    p.n_users = n_users; p.n_items = n_items; p.indptr = csr_indptr; p.indices = csr_indices;
    p.seed = seed; p.first = first_triple; p.out_u = out_u; p.out_i = out_i; p.out_j = out_j;
    p.order = order;
    if (int rc = set_filter(p, filter, filter_words)) return rc;
    return launch_apply(p, ld, flags, (cudaStream_t)stream);
}

extern "C" int eb_bpr_step_peer_f32(float *U, float *const *V_shards, float *const *b_shards, int n_shards, int32_t shard_rows,
                                    int d, int ld, int32_t n_items, const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n,
                                    float lr, float reg_u, float reg_b, float reg_pos, float reg_neg, double *loss, int flags,
                                    void *stream) {
    EB_ARG(U && d >= 1 && ld >= d && ((uintptr_t)U % 16) == 0, "bad user table");
    EB_ARG(n >= 0, "n < 0");
    HogwildParams p{};
    if (int rc = fill_peer(p, V_shards, b_shards, n_shards, shard_rows, n_items)) return rc;
    if (n == 0) return EB_OK;
    EB_ARG(tu && ti && tj, "null triple arrays");
    p.U = U; p.ld = ld; p.tu = tu; p.ti = ti; p.tj = tj; p.n = n;
    p.hp = {lr, reg_u, reg_b, reg_pos, reg_neg}; p.loss = loss;
    return launch_hogwild_peer<false>(p, ld, flags, (cudaStream_t)stream);
}

extern "C" int eb_bpr_step_sampled_peer_f32(float *U, float *const *V_shards, float *const *b_shards, int n_shards, int32_t shard_rows,
                                            int d, int ld, int32_t n_users, int32_t n_items, const int64_t *csr_indptr,
                                            const int32_t *csr_indices, const uint32_t *filter, int filter_words, int64_t n,
                                            uint64_t seed, uint64_t first_triple, float lr,
                                            float reg_u, float reg_b, float reg_pos, float reg_neg, double *loss, int32_t *out_u,
                                            int32_t *out_i, int32_t *out_j, int flags, void *stream) {
    EB_ARG(U && d >= 1 && ld >= d && ((uintptr_t)U % 16) == 0, "bad user table");
    EB_ARG(n >= 0 && n_users > 0 && n_items > 1, "bad sizes");
    EB_ARG(csr_indptr && csr_indices, "null CSR");
    EB_ARG((!out_u && !out_i && !out_j) || (out_u && out_i && out_j), "out_u/out_i/out_j: all or none");
    HogwildParams p{};
    if (int rc = fill_peer(p, V_shards, b_shards, n_shards, shard_rows, n_items)) return rc;
    if (n == 0) return EB_OK;
    p.U = U; p.ld = ld; p.n = n;
    p.hp = {lr, reg_u, reg_b, reg_pos, reg_neg}; p.loss = loss;
    p.n_users = n_users; p.n_items = n_items; p.indptr = csr_indptr; p.indices = csr_indices;
    p.seed = seed; p.first = first_triple; p.out_u = out_u; p.out_i = out_i; p.out_j = out_j;
    p.no_item_updates = (flags >> 2) & 1;
    if (int rc = set_filter(p, filter, filter_words)) return rc;
    return launch_hogwild_peer<true>(p, ld, flags, (cudaStream_t)stream);
}

extern "C" int eb_bpr_sample_philox(int32_t n_users, int32_t n_items, const int64_t *csr_indptr,
                                    const int32_t *csr_indices, int64_t n, uint64_t seed, uint64_t first_triple,
                                    int32_t *out_u, int32_t *out_i, int32_t *out_j, void *stream) {
    return eb_bpr_sample_philox_filter(n_users, n_items, csr_indptr, csr_indices, nullptr, 0, n, seed, first_triple, out_u, out_i,
                                       out_j, stream);
}

extern "C" int eb_bpr_sample_philox_filter(int32_t n_users, int32_t n_items, const int64_t *csr_indptr,
                                           const int32_t *csr_indices, const uint32_t *filter, int filter_words, int64_t n,
                                           uint64_t seed, uint64_t first_triple, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                                           void *stream) {
    EB_ARG(n >= 0 && n_users > 0 && n_items > 1, "bad sizes");
    EB_ARG(csr_indptr && csr_indices && out_u && out_i && out_j, "null pointer");
    if (n == 0) return EB_OK;
    HogwildParams p{};
    p.n = n; p.n_users = n_users; p.n_items = n_items; p.indptr = csr_indptr; p.indices = csr_indices;
    p.seed = seed; p.first = first_triple; p.out_u = out_u; p.out_i = out_i; p.out_j = out_j;
    if (int rc = set_filter(p, filter, filter_words)) return rc;
    int64_t grid = (n + 255) / 256;
    int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    philox_sample_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_pointwise_sample_philox(int32_t n_users, int32_t n_items, const int64_t *csr_indptr, const int32_t *csr_indices,
                                          const uint32_t *filter, int filter_words, int64_t n, uint64_t seed, uint64_t first,
                                          int32_t *out_u, int32_t *out_i, float *out_label, void *stream) {
    EB_ARG(n >= 0 && n_users > 0 && n_items > 1, "bad sizes");
    EB_ARG(csr_indptr && csr_indices && out_u && out_i && out_label, "null pointer");
    if (n == 0) return EB_OK;
    HogwildParams p{};
    p.n = n; p.n_users = n_users; p.n_items = n_items; p.indptr = csr_indptr; p.indices = csr_indices;
    p.seed = seed; p.first = first; p.out_u = out_u; p.out_i = out_i;
    if (int rc = set_filter(p, filter, filter_words)) return rc;
    int64_t grid = (n + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    pointwise_sample_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(p, out_label);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_bpr_step_host_f32(float *U, float *V, float *item_bias, int d, int ld, const int32_t *tu_host,
                                    const int32_t *ti_host, const int32_t *tj_host, int64_t n, float lr, float reg_u,
                                    float reg_b, float reg_pos, float reg_neg, int32_t *staging, double *loss_dev,
                                    double *loss_host, int flags, void *stream) {
    EB_ARG(staging && tu_host && ti_host && tj_host, "null host/staging pointer");
    cudaStream_t st = (cudaStream_t)stream;
    EB_CUDA(cudaMemcpyAsync(staging, tu_host, sizeof(int32_t) * n, cudaMemcpyHostToDevice, st));
    EB_CUDA(cudaMemcpyAsync(staging + n, ti_host, sizeof(int32_t) * n, cudaMemcpyHostToDevice, st));
    EB_CUDA(cudaMemcpyAsync(staging + 2 * n, tj_host, sizeof(int32_t) * n, cudaMemcpyHostToDevice, st));
    if (loss_dev) EB_CUDA(cudaMemsetAsync(loss_dev, 0, sizeof(double), st));
    if (int rc = eb_bpr_step_f32(U, V, item_bias, d, ld, staging, staging + n, staging + 2 * n, n, lr, reg_u, reg_b,
                                 reg_pos, reg_neg, loss_dev, flags, stream))
        return rc;
    if (loss_dev && loss_host)
        EB_CUDA(cudaMemcpyAsync(loss_host, loss_dev, sizeof(double), cudaMemcpyDeviceToHost, st));
    if (!(flags & 2)) EB_CUDA(cudaStreamSynchronize(st));
    return EB_OK;
}

extern "C" int eb_bpr_step_host_packed_f32(float *U, float *V, float *item_bias, int d, int ld, const uint64_t *packed_host, int64_t n,
                                           int bits_u, int bits_i, float lr, float reg_u, float reg_b, float reg_pos, float reg_neg,
                                           uint64_t *staging, double *loss_dev, double *loss_host, int flags, void *stream) {
    if (int rc = check_tables(U, V, item_bias, d, ld)) return rc;
    EB_ARG(staging && packed_host && n >= 0, "null host/staging pointer");
    EB_ARG(bits_u >= 1 && bits_i >= 1 && bits_u + 2 * bits_i <= 64, "need bits_u + 2*bits_i <= 64 (got %d, %d)", bits_u, bits_i);
    cudaStream_t st = (cudaStream_t)stream;
    if (loss_dev) EB_CUDA(cudaMemsetAsync(loss_dev, 0, sizeof(double), st));
    if (n > 0) {
        EB_CUDA(cudaMemcpyAsync(staging, packed_host, sizeof(uint64_t) * n, cudaMemcpyHostToDevice, st));   // ONE copy, 8 B / triple
        HogwildParams p{};
        p.U = U; p.V = V; p.b = item_bias; p.ld = ld; p.n = n; p.packed = staging; p.bits_u = bits_u; p.bits_i = bits_i;
        p.hp = {lr, reg_u, reg_b, reg_pos, reg_neg}; p.loss = loss_dev;
        if (int rc = launch_hogwild<false>(p, ld, flags, st)) return rc;
    }
    if (loss_dev && loss_host) EB_CUDA(cudaMemcpyAsync(loss_host, loss_dev, sizeof(double), cudaMemcpyDeviceToHost, st));
    if (!(flags & 2)) EB_CUDA(cudaStreamSynchronize(st));
    return EB_OK;
}

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
