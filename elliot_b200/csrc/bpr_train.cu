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
//  * bpr_rounds_kernel   — the same update in deterministic rounds (flags bit 6).
//  * bpr_grouped_kernel  — the free-running sampled step on local tables: the same update, applied to the triples
//    grouped by user (user_key_kernel + a stable radix sort first), the user row kept in registers across a run.
//  * bpr_hogwild_stage_kernel — the update on peer item tables with the rows staged through shared memory.
// Exact mode (fp64) is in bpr_exact.cu, the sampler in bpr_sampler.cuh and its stand-alone kernels in bpr_sample.cu.
#include <cooperative_groups.h>
#include <cub/cub.cuh>

#include <type_traits>

#include "bpr_sampler.cuh"
#include "bpr_update.cuh"

namespace eb {

struct HogwildParams {
    float *U, *V, *b;
    int ld;
    const int32_t *tu, *ti, *tj;
    int64_t n;
    BprHyper hp;
    double *loss;
    SamplerParams sampler;
    int32_t *out_u, *out_i, *out_j;
    // PEER mode (item table row-sharded over the GPUs of one NVSwitch box, SURVEY.md §8e): shard s holds item rows
    // [s*shards.rows, (s+1)*shards.rows) at Vp[s] / bp[s] — local memory for this rank's shard, peer-mapped memory
    // (cudaIpcOpenMemHandle, peer.cu) for the others; loads and vector atomics go straight over NVLink.
    float *Vp[EB_MAX_PEERS], *bp[EB_MAX_PEERS];
    ShardMap shards;
    // optional PACKED triples (host boundary: 8 B instead of 12 B per triple over PCIe): u | i << bits_u | j << (bits_u + bits_i)
    const uint64_t *packed;
    int bits_u, bits_i;
    // grouped sampled step: the call's triple indices ordered by user (ascending u, then ascending t)
    const int32_t *order;
};

// triple t: sampled (and written to out_* when asked), unpacked from the 8-byte host format, or read from three arrays
template <bool SAMPLE>
__device__ __forceinline__ void fetch_triple(const HogwildParams &p, int64_t t, int &u, int &i, int &j) {
    if (SAMPLE) {
        sample_triple(p.sampler, t, u, i, j);
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

// the lane's share of the rows and the biases of triple (u, i, j), nothing for u < 0; peer rows with system-scope loads
template <int DP, bool PEER>
__device__ __forceinline__ void load_rows(const HogwildParams &p, int gl, Rows<LaneGroup<DP>::VPL> &r, int u, int i, int j) {
    constexpr int G = LaneGroup<DP>::G, VPL = LaneGroup<DP>::VPL;
    if (u >= 0) {
        float *ri, *rj, *bi, *bj;
        item_row<PEER>(p, i, ri, bi); item_row<PEER>(p, j, rj, bj);
        const float4 *pu = reinterpret_cast<const float4 *>(p.U + (int64_t)u * p.ld);
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
}

// W: how the item rows and biases are written.  Write::AtomicSys is the peer-table kernel (item rows in the owner shard's
// memory); the user row, always local, takes GPU-scope atomics unless the step is the racy plain-store one.
template <int DP, bool SAMPLE, Write W>
__global__ void __launch_bounds__(256) bpr_hogwild_kernel(const HogwildParams p) {
    using LG = LaneGroup<DP>;
    constexpr int G = LG::G, VPL = LG::VPL, UNR = LG::UNR;
    constexpr bool PEER = W == Write::AtomicSys;
    constexpr Write WU = W == Write::Store ? Write::Store : Write::Atomic;
    const LG lg;
    const int64_t ld = p.ld;
    float loss_acc = 0.f;

    const int64_t n_tiles = (p.n + 31) / 32;
    for (int64_t tile = lg.warp; tile < n_tiles; tile += lg.nwarps) {
        const int64_t t = tile * 32 + lg.lane;
        int u = -1, i = 0, j = 0;
        if (t < p.n) fetch_triple<SAMPLE>(p, t, u, i, j);
        // UNR triples of the group in flight at once: all their row loads are issued before the first reduction
#pragma unroll 1
        for (int s0 = 0; s0 < G; s0 += UNR) {
            Rows<VPL> rw[UNR];
            int tu_[UNR], ti_[UNR], tj_[UNR];
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                bcast_triple(u, i, j, lg.gbase + s0 + q, tu_[q], ti_[q], tj_[q]);
                load_rows<DP, PEER>(p, lg.gl, rw[q], tu_[q], ti_[q], tj_[q]);
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
                    const float z = bpr_sigmoid_loss(part + (cur.bi - cur.bj), loss_acc, lg.gl);
                    float *pu = p.U + (int64_t)cu * ld, *pi, *pj, *pbi, *pbj;
                    item_row<PEER>(p, ci, pi, pbi); item_row<PEER>(p, cj, pj, pbj);
#pragma unroll
                    for (int v = 0; v < VPL; v++) {
                        const float4 a = cur.u[v], vi = cur.vi[v], vj = cur.vj[v];
                        float4 du, di, dj;
                        bpr_row_deltas(a, vi, vj, z, p.hp, du, di, dj);
                        const int e = (v * G + lg.gl) * 4;
                        write_row<WU>(pu + e, a, du);
                        write_row<W>(pi + e, vi, di);
                        write_row<W>(pj + e, vj, dj);
                    }
                    if (lg.gl == 0) {
                        float dbi, dbj;
                        bpr_bias_deltas(z, cur.bi, cur.bj, p.hp, dbi, dbj);
                        write_bias<W>(pbi, cur.bi, dbi);
                        write_bias<W>(pbj, cur.bj, dbj);
                    }
                }
            }
        }
    }
    flush_loss(loss_acc, p.loss, lg.lane);
}

// Deterministic rounds (opt-in, flags bit 6 / deterministic=True in ops) make the step deterministic.  The launch is
// cooperative and runs in rounds: every warp loads the rows of UNR triples per lane group, computes their updates from those
// values, the whole grid waits, every warp adds its updates, the grid waits again.  A triple therefore reads exactly the
// values left by the previous rounds — which round a triple falls into is fixed by its index and the grid size, not by
// timing — so the same inputs give the same tables on every run (up to the order in which one round's atomic adds to a
// shared row land, i.e. fp32 rounding).  Staleness stays bounded by one round (the grid's lane groups x UNR triples).  The
// barriers cost throughput (the row loads of one round no longer overlap the previous round's atomics), so the default is
// free-running Hogwild; rounds exist for local tables with atomic updates only.
template <int DP, bool SAMPLE>
__global__ void __launch_bounds__(256) bpr_rounds_kernel(const HogwildParams p) {
    using LG = LaneGroup<DP>;
    constexpr int G = LG::G, VPL = LG::VPL, UNR = LG::UNR;
    const LG lg;
    const int64_t ld = p.ld;
    float loss_acc = 0.f;

    // every warp runs the same number of iterations (idle ones with u = -1), so all of them reach every grid barrier
    const int64_t n_tiles = (p.n + 31) / 32;
    const int64_t tile_end = (n_tiles + lg.nwarps - 1) / lg.nwarps * lg.nwarps;
    for (int64_t tile = lg.warp; tile < tile_end; tile += lg.nwarps) {
        const int64_t t = tile * 32 + lg.lane;
        int u = -1, i = 0, j = 0;
        if (t < p.n) fetch_triple<SAMPLE>(p, t, u, i, j);
#pragma unroll 1
        for (int s0 = 0; s0 < G; s0 += UNR) {
            Rows<VPL> rw[UNR];
            int tu_[UNR], ti_[UNR], tj_[UNR];
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                bcast_triple(u, i, j, lg.gbase + s0 + q, tu_[q], ti_[q], tj_[q]);
                load_rows<DP, false>(p, lg.gl, rw[q], tu_[q], ti_[q], tj_[q]);
            }
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
                    const float z = bpr_sigmoid_loss(part + (cur.bi - cur.bj), loss_acc, lg.gl);
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
                item_row<false>(p, ti_[q], pi, pbi); item_row<false>(p, tj_[q], pj, pbj);
#pragma unroll
                for (int v = 0; v < VPL; v++) {
                    const int e = (v * G + lg.gl) * 4;
                    red_add_v4(pu + e, rw[q].u[v]);
                    red_add_v4(pi + e, rw[q].vi[v]);
                    red_add_v4(pj + e, rw[q].vj[v]);
                }
                if (lg.gl == 0) { red_add_f32(pbi, rw[q].bi); red_add_f32(pbj, rw[q].bj); }
            }
            cooperative_groups::this_grid().sync();      // every write of this round has landed before the next reads
        }
    }
    flush_loss(loss_acc, p.loss, lg.lane);
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
        sample_user(p.sampler, t, r, u, beg, len);
        key[t] = (uint32_t)u; val[t] = (int32_t)t;
    }
}

// W: Write::Atomic, or Write::Store for the racy step (the run's row `cur` is stored instead of acc added)
template <int DP, Write W>
__global__ void __launch_bounds__(256) bpr_grouped_kernel(const HogwildParams p) {
    using LG = LaneGroup<DP>;
    constexpr int G = LG::G, VPL = LG::VPL, UNR = LG::UNR;
    const LG lg;
    const int64_t ld = p.ld;
    float loss_acc = 0.f;

    const int64_t n_tiles = (p.n + 31) / 32;
    for (int64_t tile = lg.warp; tile < n_tiles; tile += lg.nwarps) {
        const int64_t pos = tile * 32 + lg.lane;
        int u = -1, i = 0, j = 0;
        if (pos < p.n) fetch_triple<true>(p, __ldg(p.order + pos), u, i, j);
        // the group's run: user cu (-1: none yet), its row as the run left it, the run's summed update
        int cu = -1;
        float4 cur[VPL], acc[VPL];
        auto flush = [&]() {
            float *pu = p.U + (int64_t)cu * ld;
#pragma unroll
            for (int v = 0; v < VPL; v++) {
                float *e = pu + (v * G + lg.gl) * 4;
                if (W == Write::Atomic) red_add_v4(e, acc[v]);
                else *reinterpret_cast<float4 *>(e) = cur[v];
            }
        };
#pragma unroll 1
        for (int s0 = 0; s0 < G; s0 += UNR) {
            Rows<VPL> rw[UNR];
            int tu_[UNR], ti_[UNR], tj_[UNR];
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                bcast_triple(u, i, j, lg.gbase + s0 + q, tu_[q], ti_[q], tj_[q]);
                if (tu_[q] >= 0) {
                    // the user row only where a run starts: inside a run the row is `cur`
                    if (tu_[q] != (q == 0 ? cu : tu_[q - 1])) {
                        const float4 *pu = reinterpret_cast<const float4 *>(p.U + (int64_t)tu_[q] * ld);
#pragma unroll
                        for (int v = 0; v < VPL; v++) rw[q].u[v] = pu[v * G + lg.gl];
                    }
                    const float4 *pi = reinterpret_cast<const float4 *>(p.V + (int64_t)ti_[q] * ld);
                    const float4 *pj = reinterpret_cast<const float4 *>(p.V + (int64_t)tj_[q] * ld);
#pragma unroll
                    for (int v = 0; v < VPL; v++) { rw[q].vi[v] = pi[v * G + lg.gl]; rw[q].vj[v] = pj[v * G + lg.gl]; }
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
                    const float z = bpr_sigmoid_loss(part + (nx.bi - nx.bj), loss_acc, lg.gl);
                    float *pi = p.V + (int64_t)qi * ld, *pj = p.V + (int64_t)qj * ld;
#pragma unroll
                    for (int v = 0; v < VPL; v++) {
                        const float4 a = cur[v], vi = nx.vi[v], vj = nx.vj[v];
                        float4 du, di, dj;
                        bpr_row_deltas(a, vi, vj, z, p.hp, du, di, dj);
                        cur[v] = make_float4(a.x + du.x, a.y + du.y, a.z + du.z, a.w + du.w);
                        acc[v] = start ? du : make_float4(acc[v].x + du.x, acc[v].y + du.y, acc[v].z + du.z, acc[v].w + du.w);
                        const int e = (v * G + lg.gl) * 4;
                        write_row<W>(pi + e, vi, di);
                        write_row<W>(pj + e, vj, dj);
                    }
                    if (lg.gl == 0) {
                        float dbi, dbj;
                        bpr_bias_deltas(z, nx.bi, nx.bj, p.hp, dbi, dbj);
                        write_bias<W>(p.b + qi, nx.bi, dbi);
                        write_bias<W>(p.b + qj, nx.bj, dbj);
                    }
                }
            }
        }
        if (cu >= 0) flush();
    }
    flush_loss(loss_acc, p.loss, lg.lane);
}

// ---------------------------------------------------------------- staged variant of the Hogwild kernel (PEER mode only)
// Same update, same sampler, same atomics as bpr_hogwild_kernel<..., Write::AtomicSys>; the difference is HOW the three
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
    using LG = LaneGroup<DP>;
    constexpr int NV = LG::NV, G = LG::G, VPL = LG::VPL;
    constexpr int ROWB = DP * 4;
    constexpr int TT = STAGE_CHUNK_BYTES / ROWB;  // triples per chunk (32 / 16 / 8 at 4 KB of rows per row kind)
    constexpr int NGRP = 32 / G;               // triples processed side by side
    static_assert(TT >= NGRP && TT <= 32 && 32 % TT == 0, "chunk shape");
    extern __shared__ __align__(128) uint8_t stage_smem[];
    const LG lg;
    const int lane = lg.lane, gl = lg.gl, wib = threadIdx.x >> 5, grp = lane / G;
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
    const int64_t ld = p.ld;
    float loss_acc = 0.f;

    for (int64_t tile = lg.warp; tile * 32 < p.n; tile += lg.nwarps) {
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
                int cu, ci, cj;
                bcast_triple(u, i, j, src, cu, ci, cj);
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
                        red_add_v4_sys(gi + e, di);
                        red_add_v4_sys(gj + e, dj);
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
    flush_loss(loss_acc, p.loss, lane);
}

// ---------------------------------------------------------------- host side
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

using StepKernel = void (*)(HogwildParams);

// kern on the persistent grid; the rounds kernel is launched cooperatively, so every CTA is resident for its grid barriers
static int launch_persistent(StepKernel kern, const HogwildParams &p, int reserve_sms, cudaStream_t st, int smem = 0,
                             bool cooperative = false) {
    unsigned grid;
    if (int rc = persistent_grid((const void *)kern, smem, p.n, reserve_sms, grid)) return rc;
    if (cooperative) {
        void *args[] = {const_cast<HogwildParams *>(&p)};
        EB_CUDA(cudaLaunchCooperativeKernel((const void *)kern, dim3(grid), dim3(256), args, smem, st));
    } else {
        kern<<<grid, 256, smem, st>>>(p);
    }
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

// The flags word of the eb_bpr_step_* entry points (include/elliot_b200.h)
struct StepFlags {
    bool racy;      // bit 0: plain stores instead of atomics
    bool no_sync;   // bit 1: the host-triple step returns without synchronising its stream
    bool reg;       // bit 4: peer tables: the register kernel instead of the shared-memory-staged one
    bool stage;     // bit 5: the shared-memory-staged kernel (peer tables only)
    bool rounds;    // bit 6: deterministic rounds
    int reserve;    // bits 8..15: SMs the grids leave free
};

static int decode_flags(int flags, StepFlags &f) {
    EB_ARG(!(flags & 4), "flags bit 2 is not a BPR step option (item-row updates cannot be switched off)");
    f = StepFlags{(flags & 1) != 0, (flags & 2) != 0, (flags & 16) != 0, (flags & 32) != 0, (flags & 64) != 0, (flags >> 8) & 0xff};
    return EB_OK;
}

// The compiled row strides of each table kind
template <int... DPS>
struct Strides {};
using LocalStrides = Strides<8, 16, 32, 64, 128, 256>;
using PeerStrides = Strides<32, 64, 128>;            // sharded item tables

// f(std::integral_constant<int, DP>{}) for the row stride DP == dp among the compiled ones, else EB_ERR_ARG
template <int... DPS, class F>
static int with_stride(Strides<DPS...>, int dp, F &&f) {
    int rc = EB_OK;
    if (((dp == DPS && (rc = f(std::integral_constant<int, DPS>{}), true)) || ...)) return rc;
    char list[64];
    int len = 0;
    ((len += snprintf(list + len, sizeof list - len, len ? ",%d" : "%d", DPS)), ...);
    return set_err(EB_ERR_ARG, "row stride ld=%d must be one of %s floats", dp, list);
}

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
// only n and the sampler's seed, first, n_users, n_items and indptr, never the tables.  The ordered indices end up in one of
// the workspace's two index buffers (cub's double buffer decides which): `order` points at it.  The key pass leaves
// `reserve` SMs free; cub's sort kernels size their own grids.
static int schedule_grouped(const HogwildParams &p, int reserve, char *ws, const GroupLayout &L, cudaStream_t st,
                            const int32_t *&order) {
    cub::DoubleBuffer<uint32_t> keys((uint32_t *)(ws + L.key_a), (uint32_t *)(ws + L.key_b));
    cub::DoubleBuffer<int32_t> vals((int32_t *)(ws + L.val_a), (int32_t *)(ws + L.val_b));
    user_key_kernel<<<capped_grid(p.n, reserve), 256, 0, st>>>(p, keys.Current(), vals.Current());
    EB_CUDA(cudaGetLastError());
    size_t cb = L.cub_bytes;
    EB_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.cub, cb, keys, vals, (int)p.n, 0, bits_for((uint64_t)p.sampler.n_users), st));
    order = vals.Current();
    return EB_OK;
}

template <int DP>
static StepKernel grouped_kernel(bool racy) {
    return racy ? bpr_grouped_kernel<DP, Write::Store> : bpr_grouped_kernel<DP, Write::Atomic>;
}

// Sampled step on local tables, free-running: per sub-step, the schedule above, then the grouped update (which leaves
// `reserve` SMs free).
static int launch_grouped(StepKernel kern, HogwildParams p, int reserve, char *ws, const GroupLayout &L, cudaStream_t st) {
    const int64_t n = p.n;
    const uint64_t first = p.sampler.first;
    int32_t *out_u = p.out_u, *out_i = p.out_i, *out_j = p.out_j;
    for (int64_t c0 = 0; c0 < n; c0 += GROUP_MAX) {
        p.n = n - c0 < GROUP_MAX ? n - c0 : GROUP_MAX;
        p.sampler.first = first + (uint64_t)c0;
        if (out_u) { p.out_u = out_u + c0; p.out_i = out_i + c0; p.out_j = out_j + c0; }
        if (int rc = schedule_grouped(p, reserve, ws, L, st, p.order)) return rc;
        if (int rc = launch_persistent(kern, p, reserve, st)) return rc;
    }
    return EB_OK;
}

// One table.  SAMPLE: the sampled step; free-running it runs grouped by user (ws: eb_bpr_step_sampled_workspace_bytes).
// Deterministic rounds run bpr_rounds_kernel, materialised triples free-running bpr_hogwild_kernel.
template <bool SAMPLE>
static int launch_local(const HogwildParams &p, int flags, cudaStream_t st, void *ws = nullptr, size_t ws_bytes = 0) {
    StepFlags f;
    if (int rc = decode_flags(flags, f)) return rc;
    EB_ARG(!f.stage, "the shared-memory-staged kernel exists for sharded item tables only");
    EB_ARG(!f.racy || !f.rounds, "deterministic rounds run with atomic updates");
    GroupLayout L{};
    if (SAMPLE && !f.rounds) {
        L = group_layout(p.n, p.sampler.n_users);
        if (!ws || ws_bytes < L.total) return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", ws ? ws_bytes : 0, L.total);
    }
    return with_stride(LocalStrides{}, p.ld, [&](auto dpc) {
        constexpr int DP = decltype(dpc)::value;
        if (f.rounds) return launch_persistent(bpr_rounds_kernel<DP, SAMPLE>, p, f.reserve, st, 0, true);
        if constexpr (SAMPLE) return launch_grouped(grouped_kernel<DP>(f.racy), p, f.reserve, (char *)ws, L, st);
        else return launch_persistent(f.racy ? bpr_hogwild_kernel<DP, false, Write::Store> : bpr_hogwild_kernel<DP, false, Write::Atomic>,
                                      p, f.reserve, st);
    });
}

// The grouped update alone, on an order the caller scheduled (p.order, p.n <= GROUP_MAX)
static int launch_apply(const HogwildParams &p, int flags, cudaStream_t st) {
    StepFlags f;
    if (int rc = decode_flags(flags, f)) return rc;
    EB_ARG(!f.stage && !f.rounds, "the grouped update runs free-running on local tables (no rounds, no staged kernel)");
    return with_stride(LocalStrides{}, p.ld, [&](auto dpc) {
        return launch_persistent(grouped_kernel<decltype(dpc)::value>(f.racy), p, f.reserve, st);
    });
}

// PEER mode: atomics only (other GPUs update the same rows), strides the sharded configurations use.  The shared-memory-staged
// kernel is the default (its row copies are in flight without holding registers while the rows cross NVLink); flags bit 4 (16),
// or bit 0, selects the register kernel (whose peer updates stay atomic).
template <bool SAMPLE>
static int launch_peer(const HogwildParams &p, int flags, cudaStream_t st) {
    StepFlags f;
    if (int rc = decode_flags(flags, f)) return rc;
    EB_ARG(!f.rounds, "deterministic rounds exist for local tables only (other GPUs update peer rows concurrently)");
    return with_stride(PeerStrides{}, p.ld, [&](auto dpc) {
        constexpr int DP = decltype(dpc)::value;
        if (f.racy || f.reg) return launch_persistent(bpr_hogwild_kernel<DP, SAMPLE, Write::AtomicSys>, p, f.reserve, st);
        constexpr int SMEM = 8 * 3 * STAGE_CHUNK_BYTES + 64;   // 8 warps x 3 row kinds x chunk + mbarriers
        EB_CUDA(cudaFuncSetAttribute(bpr_hogwild_stage_kernel<DP, SAMPLE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        return launch_persistent(bpr_hogwild_stage_kernel<DP, SAMPLE>, p, f.reserve, st, SMEM);
    });
}

// the fields every step fills
static HogwildParams step_params(float *U, float *V, float *b, int ld, int64_t n, BprHyper hp, double *loss) {
    HogwildParams p{};
    p.U = U; p.V = V; p.b = b; p.ld = ld; p.n = n; p.hp = hp; p.loss = loss;
    return p;
}

// the optional sampled-triple outputs: all three or none
static int set_out(HogwildParams &p, int32_t *out_u, int32_t *out_i, int32_t *out_j) {
    EB_ARG((!out_u && !out_i && !out_j) || (out_u && out_i && out_j), "out_u/out_i/out_j: all or none");
    p.out_u = out_u; p.out_i = out_i; p.out_j = out_j;
    return EB_OK;
}

// the user table (p.U, row stride p.ld) and the item shards of a peer step
static int fill_peer(HogwildParams &p, int d, float *const *V_shards, float *const *b_shards, int n_shards, int32_t shard_rows,
                     int32_t n_items) {
    EB_ARG(p.U && d >= 1 && p.ld >= d && ((uintptr_t)p.U % 16) == 0, "bad user table");
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

}  // namespace eb

using namespace eb;

extern "C" int eb_bpr_step_f32(float *U, float *V, float *item_bias, int d, int ld, const int32_t *tu,
                               const int32_t *ti, const int32_t *tj, int64_t n, float lr, float reg_u, float reg_b,
                               float reg_pos, float reg_neg, double *loss, int flags, void *stream) {
    if (int rc = check_tables(U, V, item_bias, d, ld)) return rc;
    EB_ARG(n >= 0, "n < 0");
    if (n == 0) return EB_OK;
    EB_ARG(tu && ti && tj, "null triple arrays");
    HogwildParams p = step_params(U, V, item_bias, ld, n, {lr, reg_u, reg_b, reg_pos, reg_neg}, loss);
    p.tu = tu; p.ti = ti; p.tj = tj;
    return launch_local<false>(p, flags, (cudaStream_t)stream);
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
    EB_ARG(n >= 0, "n < 0");
    HogwildParams p = step_params(U, V, item_bias, ld, n, {lr, reg_u, reg_b, reg_pos, reg_neg}, loss);
    if (int rc = sampler_params(p.sampler, n_users, n_items, csr_indptr, csr_indices, filter, filter_words, seed, first_triple))
        return rc;
    if (int rc = set_out(p, out_u, out_i, out_j)) return rc;
    if (n == 0) return EB_OK;
    return launch_local<true>(p, flags, (cudaStream_t)stream, workspace, workspace_bytes);
}

extern "C" int eb_bpr_schedule_sampled(int32_t n_users, int32_t n_items, const int64_t *csr_indptr, int64_t n, uint64_t seed,
                                       uint64_t first_triple, void *workspace, size_t workspace_bytes, size_t *order_offset,
                                       int flags, void *stream) {
    EB_ARG(n >= 1 && n <= GROUP_MAX && n_users > 0 && n_items > 1, "bad sizes (a schedule covers 1..%lld triples)",
           (long long)GROUP_MAX);
    EB_ARG(csr_indptr && order_offset, "null pointer");
    StepFlags f;
    if (int rc = decode_flags(flags, f)) return rc;
    const GroupLayout L = group_layout(n, n_users);
    if (!workspace || workspace_bytes < L.total)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace ? workspace_bytes : 0, L.total);
    HogwildParams p{};
    p.n = n; p.sampler = SamplerParams{n_users, n_items, csr_indptr, nullptr, seed, first_triple, nullptr, 0};
    const int32_t *order = nullptr;
    if (int rc = schedule_grouped(p, f.reserve, (char *)workspace, L, (cudaStream_t)stream, order)) return rc;
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
    EB_ARG(n >= 1 && n <= GROUP_MAX, "bad sizes (an apply covers 1..%lld triples)", (long long)GROUP_MAX);
    EB_ARG(order, "null order");
    HogwildParams p = step_params(U, V, item_bias, ld, n, {lr, reg_u, reg_b, reg_pos, reg_neg}, loss);
    if (int rc = sampler_params(p.sampler, n_users, n_items, csr_indptr, csr_indices, filter, filter_words, seed, first_triple))
        return rc;
    if (int rc = set_out(p, out_u, out_i, out_j)) return rc;
    p.order = order;
    return launch_apply(p, flags, (cudaStream_t)stream);
}

extern "C" int eb_bpr_step_peer_f32(float *U, float *const *V_shards, float *const *b_shards, int n_shards, int32_t shard_rows,
                                    int d, int ld, int32_t n_items, const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n,
                                    float lr, float reg_u, float reg_b, float reg_pos, float reg_neg, double *loss, int flags,
                                    void *stream) {
    EB_ARG(n >= 0, "n < 0");
    HogwildParams p = step_params(U, nullptr, nullptr, ld, n, {lr, reg_u, reg_b, reg_pos, reg_neg}, loss);
    if (int rc = fill_peer(p, d, V_shards, b_shards, n_shards, shard_rows, n_items)) return rc;
    if (n == 0) return EB_OK;
    EB_ARG(tu && ti && tj, "null triple arrays");
    p.tu = tu; p.ti = ti; p.tj = tj;
    return launch_peer<false>(p, flags, (cudaStream_t)stream);
}

extern "C" int eb_bpr_step_sampled_peer_f32(float *U, float *const *V_shards, float *const *b_shards, int n_shards, int32_t shard_rows,
                                            int d, int ld, int32_t n_users, int32_t n_items, const int64_t *csr_indptr,
                                            const int32_t *csr_indices, const uint32_t *filter, int filter_words, int64_t n,
                                            uint64_t seed, uint64_t first_triple, float lr,
                                            float reg_u, float reg_b, float reg_pos, float reg_neg, double *loss, int32_t *out_u,
                                            int32_t *out_i, int32_t *out_j, int flags, void *stream) {
    EB_ARG(n >= 0, "n < 0");
    HogwildParams p = step_params(U, nullptr, nullptr, ld, n, {lr, reg_u, reg_b, reg_pos, reg_neg}, loss);
    if (int rc = sampler_params(p.sampler, n_users, n_items, csr_indptr, csr_indices, filter, filter_words, seed, first_triple))
        return rc;
    if (int rc = set_out(p, out_u, out_i, out_j)) return rc;
    if (int rc = fill_peer(p, d, V_shards, b_shards, n_shards, shard_rows, n_items)) return rc;
    if (n == 0) return EB_OK;
    return launch_peer<true>(p, flags, (cudaStream_t)stream);
}

extern "C" int eb_bpr_step_host_packed_f32(float *U, float *V, float *item_bias, int d, int ld, const uint64_t *packed_host, int64_t n,
                                           int bits_u, int bits_i, float lr, float reg_u, float reg_b, float reg_pos, float reg_neg,
                                           uint64_t *staging, double *loss_dev, double *loss_host, int flags, void *stream) {
    if (int rc = check_tables(U, V, item_bias, d, ld)) return rc;
    EB_ARG(staging && packed_host && n >= 0, "null host/staging pointer");
    EB_ARG(bits_u >= 1 && bits_i >= 1 && bits_u + 2 * bits_i <= 64, "need bits_u + 2*bits_i <= 64 (got %d, %d)", bits_u, bits_i);
    StepFlags f;
    if (int rc = decode_flags(flags, f)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (loss_dev) EB_CUDA(cudaMemsetAsync(loss_dev, 0, sizeof(double), st));
    if (n > 0) {
        EB_CUDA(cudaMemcpyAsync(staging, packed_host, sizeof(uint64_t) * n, cudaMemcpyHostToDevice, st));   // ONE copy, 8 B / triple
        HogwildParams p = step_params(U, V, item_bias, ld, n, {lr, reg_u, reg_b, reg_pos, reg_neg}, loss_dev);
        p.packed = staging; p.bits_u = bits_u; p.bits_i = bits_i;
        if (int rc = launch_local<false>(p, flags, st)) return rc;
    }
    if (loss_dev && loss_host) EB_CUDA(cudaMemcpyAsync(loss_host, loss_dev, sizeof(double), cudaMemcpyDeviceToHost, st));
    if (!f.no_sync) EB_CUDA(cudaStreamSynchronize(st));
    return EB_OK;
}
