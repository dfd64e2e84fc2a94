// score_topk_tc.cu — full-catalogue U·Vᵀ on the Hopper tensor cores (wgmma + TMA + mbarrier)
// with the per-user masked top-k fused into the epilogue and an exact fp32 re-rank.
//
// Replaces BPRMF_batch_model.predict/get_top_k (BPRMF_batch_model.py:82-88) /
// MFModel.get_user_predictions (BPRMF_model.py:70-85) at catalogue scale: the (users x items)
// score matrix is never materialised.
//
// Pipeline per CTA (persistent, one CTA per SM, NG consumer warpgroups + one TMA warp; NG = 2 by default):
//   last warp     TMA producer : A tile (128 users x KP, bf16, once per user block) and a ring of
//                                B tiles (BN items x KP) via cp.async.bulk.tensor, 128B swizzle (+ a narrower-swizzle K tail)
//   warpgroup g   consumer     : takes every NG-th item tile; issues wgmma.m64nBNk16 twice per K step (users 0-63 and
//                                64-127) into fp32 register accumulators, hands the B stage back, moves its accumulators
//                                through a per-warp shared-memory tile so that every thread holds ONE user row, then a
//                                running threshold filters all but the group's current top-16 approximate scores (max-tree
//                                fast path), survivors are checked against the train CSR (block's mask rows cached in shared
//                                memory) and kept in a per-row candidate list.
// While one warpgroup scans its tile the other one's MMAs run on the tensor cores.  Variants behind template switches (TcCfg):
// one consumer warpgroup (NG = 1), CTA pairs sharing every item tile through TMA multicast (PAIR), the user block held in
// registers as the wgmma A operand (ATM), instrumentation (DBG).
// After the last item tile each warp re-scores its rows' <= 32 candidates (16 per group) EXACTLY in fp32
// (same summation order as score_topk.cu), sorts them with a 32-lane bitonic network
// (score desc, index asc) and certifies the result:
//      every item not in the list has approx score <= tau (final threshold), so its exact
//      score is <= tau + eps_u with eps_u = c * ||u|| * max_i ||v_i|| (bf16 rounding bound);
//      if the k-th exact score exceeds tau + eps_u the list is provably the exact top-k.
// Users that cannot be certified are appended to a list and re-done by the exact kernel.
#include <cuda.h>
#include <cuda_bf16.h>
#include <math_constants.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace eb {

constexpr int TC_BM = 128;        // users per block (two wgmma M = 64 halves)
constexpr int TC_KC = 32;         // candidates kept per user (one per lane in the re-rank)


// ---------------------------------------------------------------- parameters
// ---------------------------------------------------------------- parameters
struct TcParams {
    // exact-side inputs
    const float *U, *V, *bias;   // fp32 tables (row stride ld), bias may be null
    int d, ld;
    int32_t n_items;
    const int64_t *mask_indptr;
    const int32_t *mask_indices; // sorted rows
    int32_t user_begin;
    int32_t n_sel;
    int k;
    // prepared by tc_prep kernels
    const __nv_bfloat16 *ubf;    // bf16 user rows [n_sel][KP] (the A operand), read directly by the users-in-registers kernel
    const float *unorm;          // ||u|| per selected user
    const float *vstat;          // [0] = max ||v||, [1] = max |bias|
    const float *bmax_chunk;     // max bias per 32-item chunk (null if no bias)
    // outputs
    int32_t *out_idx;
    float *out_val;
    int32_t *flag_count;         // number of uncertified users
    int32_t *flag_list;          // their positions q in [0, n_sel)
    float *dump;                 // optional dense n_sel x n_items approximate scores (tests)
    float eps_scale;             // c in eps_u = c * ||u|| * max||v|| + 1e-6 * (...)
    long long *prof;             // optional per-kernel cycle counters (8 values), profiling only
    int bias_folded;             // 1: bias already inside the accumulators (extra K columns); the re-rank still adds it exactly
    int debug_mode;              // profiling only: 1 = accumulator read + max only, 2 = no compaction (results invalid)
};

constexpr int TC_BUF = 64;        // append-buffer slots per user row over all epilogue groups (top-KC kept + pending)

// KP = padded K (multiple of 16): KB full 64-wide blocks (one 128-byte swizzle atom each) + a tail of KT = 0, 16 or 32
// columns in its own narrower-swizzle block.  (A 48-column tail is rounded up to a full block by the host.)  Padding K
// to a multiple of 64 instead costs 2.0x the MMA work at d = 64 + 2 bias columns (128 vs 80) and 1.33x at d = 128 + 2
// (192 vs 144).
// NG = number of consumer warpgroups.  NG = 1: warpgroup 0 takes every tile, 32 kept candidates in a 64-slot buffer per row.
// NG = 2: warpgroup 0 takes the even tiles, warpgroup 1 the odd ones (global tile counter), so the MMAs of one overlap the
// scan of the other.  Each group keeps KC/2 = 16 candidates in a 32-slot buffer per row: the 16th best of half the stream
// sits at the same level as the 32nd best of the whole stream, so the insert rate per item is that of NG = 1, the shared
// memory is the same 64 KB, and the re-rank reads the two lists side by side (16 + 16 lanes) with tau = max of the two.
// BN = items per tile (wgmma N).  A warpgroup's accumulators are 128 x BN fp32; they pass through a per-warp shared-memory
// tile (32 rows x BN) on their way from the wgmma fragment layout to one row per thread, so BN also sets that tile's size:
// 64 up to KP = 128, 32 above (so that four B stages still fit beside the 64 KB user block).
// PAIR: two CTAs of a cluster (two SMs) score their own user blocks against the same item tiles; each CTA fetches HALF of
// every item tile and multicasts it into both shared memories, so the item table crosses the L2 -> SM fabric once per 256
// users instead of once per 128.  A stage is refilled only after the consumers of BOTH CTAs have released it.
// ATM: the user block (the operand that stays for the whole item stream) is held in the consumer warpgroups' registers as
// the wgmma A operand instead of being re-read from shared memory by every MMA; only the item tile is read from shared
// memory.  (The historical name: the Blackwell kernel kept it in tensor memory.)  Built for KP <= 144 (KP / 2 registers).
template <int KP, int NG_, bool PAIR_ = false, bool ATM_ = false> struct TcCfg {
    static constexpr int KB = KP / 64;                       // full 64-wide K blocks
    static constexpr int KT = KP % 64;                       // tail columns
    static_assert(KT == 0 || KT == 16 || KT == 32, "K tail must be 0, 16 or 32 columns");
    static constexpr int NG = NG_;
    static constexpr bool PAIR = PAIR_, ATM = ATM_;
    static_assert(!(PAIR && ATM) && (!(PAIR || ATM) || NG_ == 2), "CTA pairs / users in registers: two-group kernel only");
    static_assert(!ATM || KP <= 144, "users in registers: KP <= 144");
    static constexpr int BN = KP <= 128 ? 64 : 32;
    static_assert(BN == 32 || BN == 64, "tiles of 32 or 64 items");
    static constexpr int NCH = BN / 4;                       // 16-byte chunks per staged row
    static constexpr int KCG = TC_KC / NG;                   // candidates kept per row and group
    static constexpr int BUFG = TC_BUF / NG;                 // buffer slots per row and group
    static constexpr int ROWB = BUFG * 4;                    // bytes per buffer row (keys; the ids follow in a second array)
    static constexpr int THREADS = 128 * NG + 32;            // NG consumer warpgroups + the TMA warp
    static constexpr int A_BYTES = TC_BM * KP * 2;
    static constexpr int B_BYTES = BN * KP * 2;
    static constexpr int STG_WARP = 32 * BN * 4;             // accumulator staging per warp
    static constexpr int STG_BYTES = 4 * NG * STG_WARP;
    static constexpr int CAND_BYTES = TC_BM * TC_BUF * 8;    // all groups together
    static constexpr int MRG_BYTES = 2048;                   // per-row {cnt, thresh} of every group after the last tile
    static constexpr int FIXED = A_BYTES + STG_BYTES + CAND_BYTES + MRG_BYTES + 256;
    static constexpr int ROOM = (232448 - FIXED) / B_BYTES;  // 227 KB of dynamic shared memory per CTA
    static constexpr int STAGES = ROOM >= 4 ? 4 : ROOM;
    static_assert(STAGES >= 2, "B ring needs two stages");
    static constexpr int USED = FIXED + STAGES * B_BYTES;
    static constexpr int SMEM = 232448;                      // everything: what is left caches the user block's train-mask rows
    static constexpr int MASKC = (SMEM - USED) / 4;          // cached mask entries (int32) per user block
};

// The user row a thread owns: warp q of a warpgroup holds the accumulators of rows 16 q .. 16 q + 15 of both 64-row halves
// (wgmma fragment layout), so it takes exactly those 32 rows — lane l < 16 row 16 q + l, lane l >= 16 row 64 + 16 q + l - 16 —
// and the fragment-to-row transposition stays inside the warp.
__device__ __forceinline__ int tc_row(int quad, int l) { return (l < 16 ? 0 : 48) + quad * 16 + l; }


__device__ __forceinline__ bool cand_better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__device__ __forceinline__ float lds_f32(uint32_t a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a)); return v; }
__device__ __forceinline__ int lds_s32(uint32_t a) { int v; asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts_f32(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void sts_s32(uint32_t a, int v) { asm volatile("st.shared.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

// binary search for `key` in the sorted int32 row at shared-memory address `a` (the cached copy of a train-mask row)
__device__ __forceinline__ bool contains_sorted_smem(uint32_t a, int len, int32_t key) {
    int lo = 0, hi = len;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (lds_s32(a + 4u * (uint32_t)mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo < len && lds_s32(a + 4u * (uint32_t)lo) == key;
}

constexpr uint32_t TC_KEY_NEG = 0x007FFFC0u;     // sortable key of -inf with the tie-break bits cleared

__device__ __forceinline__ uint32_t tc_key_of(float f, int pos) {   // order-preserving float->uint, low 6 bits = tie-break
    const uint32_t b = __float_as_uint(f);
    const uint32_t k = b ^ ((uint32_t)((int32_t)b >> 31) | 0x80000000u);
    return (k & ~63u) | (uint32_t)(63 - pos);
}
__device__ __forceinline__ float tc_upper_of(uint32_t key) {       // largest float whose key could be `key`
    const uint32_t k = key | 63u;
    const uint32_t b = (k & 0x80000000u) ? (k ^ 0x80000000u) : ~k;
    return __uint_as_float(b);
}

// Warp-cooperative compaction of ONE row of the candidate buffer (all 32 lanes call it together): rank the row's BUFG keys
// by counting (broadcast reads, no shuffles), keep ranks < KCG in sorted order, refill the rest with -inf.  BUFG = 64: two
// keys per lane; BUFG = 32: one.  Returns (number of valid kept entries, bits of the new threshold).
// Deliberately NOT inlined: it is called from every 8-column group of the unrolled scan and the
// kernel must stay inside the instruction cache.
template <int BUFG, int KCG>
__device__ __noinline__ uint2 tc_compact_row(uint32_t bk, uint32_t bi, int rrow, int lane, int rl, const int32_t *mrow,
                                             uint32_t mrow_smem, int n_items) {
    constexpr int PM = BUFG - 1;
    constexpr bool TWO = BUFG == 64;
    const int p0 = (lane + rrow) & PM, p1 = (lane + 32 + rrow) & PM;
    uint32_t k0 = (uint32_t)lds_s32(bk + 4u * p0), k1 = TWO ? (uint32_t)lds_s32(bk + 4u * p1) : 0u;
    int i0 = lds_s32(bi + 4u * p0), i1 = TWO ? lds_s32(bi + 4u * p1) : 0;
    // train items (-inf in the reference) and the zero rows TMA pads past the catalogue
    bool d0 = false, d1 = false;
    // (the row's mask entries are read from the block's shared-memory copy when they fit: the search is a chain of
    // dependent loads, ~30 cycles each there against an L2 round trip each from global memory)
    if (mrow_smem) {
        if (k0 > (TC_KEY_NEG | 63u)) d0 = i0 >= n_items || (rl > 0 && contains_sorted_smem(mrow_smem, rl, i0));
        if (TWO && k1 > (TC_KEY_NEG | 63u)) d1 = i1 >= n_items || (rl > 0 && contains_sorted_smem(mrow_smem, rl, i1));
    } else {
        if (k0 > (TC_KEY_NEG | 63u)) d0 = i0 >= n_items || (rl > 0 && contains_sorted(mrow, rl, i0));
        if (TWO && k1 > (TC_KEY_NEG | 63u)) d1 = i1 >= n_items || (rl > 0 && contains_sorted(mrow, rl, i1));
    }
    if (d0) { k0 = TC_KEY_NEG | (uint32_t)(63 - p0); sts_s32(bk + 4u * p0, (int)k0); }
    if (TWO && d1) { k1 = TC_KEY_NEG | (uint32_t)(63 - p1); sts_s32(bk + 4u * p1, (int)k1); }
    __syncwarp();
    int r0 = 0, r1 = 0;
#pragma unroll
    for (int j = 0; j < BUFG; j += 4) {
        uint32_t x0, x1, x2, x3;
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0), "=r"(x1), "=r"(x2), "=r"(x3) : "r"(bk + 4u * j));
        r0 += (x0 > k0) + (x1 > k0) + (x2 > k0) + (x3 > k0);
        if (TWO) r1 += (x0 > k1) + (x1 > k1) + (x2 > k1) + (x3 > k1);
    }
    __syncwarp();                     // all reads done before the row is rewritten
    const int n0 = (r0 + rrow) & PM, n1 = (r1 + rrow) & PM;
    const bool keep0 = r0 < KCG && k0 > (TC_KEY_NEG | 63u), keep1 = TWO && r1 < KCG && k1 > (TC_KEY_NEG | 63u);
    // without the second key, ranks >= 32 never occur and every physical slot gets exactly one writer (its rank is unique)
    sts_s32(bk + 4u * n0, (int)(keep0 ? ((k0 & ~63u) | (uint32_t)(63 - n0)) : (TC_KEY_NEG | (uint32_t)(63 - n0))));
    if (TWO) sts_s32(bk + 4u * n1, (int)(keep1 ? ((k1 & ~63u) | (uint32_t)(63 - n1)) : (TC_KEY_NEG | (uint32_t)(63 - n1))));
    if (keep0) sts_s32(bi + 4u * n0, i0);
    if (keep1) sts_s32(bi + 4u * n1, i1);
    const int nvalid = __popc(__ballot_sync(0xffffffffu, keep0)) + (TWO ? __popc(__ballot_sync(0xffffffffu, keep1)) : 0);
    __syncwarp();
    const float th = nvalid == KCG ? tc_upper_of((uint32_t)lds_s32(bk + 4u * ((KCG - 1 + rrow) & PM))) : -CUDART_INF_F;
    return make_uint2((uint32_t)nvalid, __float_as_uint(th));
}

// compaction of all rows of this warp selected by `todo`; returns the calling lane's new (cnt, thresh)
template <int BUFG, int KCG>
__device__ __noinline__ uint2 tc_compact_rows(uint32_t todo, uint32_t ckey, uint32_t cidx, int quad, int lane, int mlen,
                                              int64_t mbeg, const int32_t *mask_indices, int64_t seg_beg, int n_cached,
                                              uint32_t mcache, int n_items, int cnt, float thresh) {
    constexpr uint32_t ROWB = BUFG * 4;
    __syncwarp();
    while (todo) {
        const int r = __ffs(todo) - 1;
        todo &= todo - 1;
        const int rrow = tc_row(quad, r);
        const int rl = __shfl_sync(0xffffffffu, mlen, r);
        const int64_t rb = __shfl_sync(0xffffffffu, mbeg, r);
        const int64_t rel = rb - seg_beg;                       // the row's offset inside the block's cached segment
        const uint32_t ms = (rl > 0 && rel + rl <= (int64_t)n_cached) ? mcache + 4u * (uint32_t)rel : 0u;
        const uint2 res = tc_compact_row<BUFG, KCG>(ckey + ROWB * (uint32_t)rrow, cidx + ROWB * (uint32_t)rrow, rrow, lane, rl,
                                                    mask_indices + rb, ms, n_items);
        if (lane == r) {
            cnt = (int)res.x;
            if (res.x == KCG) thresh = __uint_as_float(res.y);
        }
    }
    __syncwarp();
    return make_uint2((uint32_t)cnt, __float_as_uint(thresh));
}

// DBG = false compiles the instrumentation out (cycle counters, dense score dump, EB_TC_DEBUG modes); the launcher picks
// DBG = true only when one of them is requested.
template <int KP, bool HAS_BIAS, int NGT, bool PAIR, bool ATM, bool DBG>
__global__ void __launch_bounds__(TcCfg<KP, NGT, PAIR, ATM>::THREADS, 1)
score_topk_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmAt, const __grid_constant__ CUtensorMap tmBt, const TcParams p) {
    using C = TcCfg<KP, NGT, PAIR, ATM>;
    constexpr int KB = C::KB, KT = C::KT, BN = C::BN, S = C::STAGES, NG = C::NG, NCH = C::NCH;
    constexpr int KCG = C::KCG, BUFG = C::BUFG;
    constexpr uint32_t ROWB = C::ROWB, GRPB = TC_BM * BUFG * 8;           // bytes per buffer row / per group (keys + ids)
    const bool DUMP = DBG && p.dump != nullptr;
    const int debug_mode = DBG ? p.debug_mode : 0;
    extern __shared__ __align__(1024) uint8_t sm[];
    uint8_t *sA = sm;                                   // KB blocks of [128 rows x 128 B] + the tail block
    uint8_t *sB = sA + C::A_BYTES;                      // S stages of KB blocks of [BN rows x 128 B] + tail
    const uint32_t stg = smem_u32(sB + S * C::B_BYTES);                      // per warp: fp32 [32 rows][BN], chunk-swizzled
    const uint32_t cval = stg + C::STG_BYTES;                                // keys / ids [BUF][128]
    const uint32_t mrg = cval + C::CAND_BYTES;                               // per group: {cnt[128], thresh[128]}
    uint64_t *bars = reinterpret_cast<uint64_t *>(sB + S * C::B_BYTES + C::STG_BYTES + C::CAND_BYTES + C::MRG_BYTES);
    const uint32_t bar0 = smem_u32(bars);
    auto B_FULL = [&](int s) { return bar0 + 8u * (uint32_t)s; };
    auto B_EMPTY = [&](int s) { return bar0 + 8u * (uint32_t)(S + s); };
    const uint32_t A_FULL = bar0 + 8u * (2 * S), A_EMPTY = bar0 + 8u * (2 * S + 1);
    const uint32_t mcache = smem_u32(sm + C::USED);                          // int32 [MASKC]: the user block's train-mask rows

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // provably warp-uniform: role branches do not diverge
    const int lane = threadIdx.x & 31;
    const int n_tiles = (p.n_items + BN - 1) / BN;
    const int n_mblocks = (p.n_sel + TC_BM - 1) / TC_BM;
    // work units: user blocks, or (PAIR) pairs of user blocks — CTA rank r of the cluster takes block 2 * unit + r; with an
    // odd number of blocks the last unit's second CTA runs a phantom block (TMA zero-fills its A tile, every row invalid)
    const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
    const int n_units = PAIR ? (n_mblocks + 1) / 2 : n_mblocks;
    const int unit0 = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x, unit_step = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;
    if (threadIdx.x == 0) {
        if (smem_u32(sm) & 1023u) __trap();             // SWIZZLE_128B tiles need 1024-byte alignment
        for (int s = 0; s < S; s++) { mbar_init(B_FULL(s), 1); mbar_init(B_EMPTY(s), PAIR ? 2 : 1); }
        mbar_init(A_FULL, 1); mbar_init(A_EMPTY, NG);
        fence_barrier_init();
    }
    if (PAIR) cluster_sync_all(); else __syncthreads();   // PAIR: the peer's barriers exist before anything is multicast to it

    if (warp == 4 * NG) {
        // ===================== TMA producer =====================
        if (elect_one_sync()) {
            tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
            if (KT) { tma_prefetch_desc(&tmAt); tma_prefetch_desc(&tmBt); }
            int s = 0; uint32_t ph = 0; uint32_t it = 0;
            const bool prof = DBG && p.prof != nullptr && blockIdx.x == 0;
            long long w_bempty = 0;
            for (int un = unit0; un < n_units; un += unit_step, it++) {
                const int mb = PAIR ? 2 * un + (int)rank : un;
                if (!ATM) {                           // ATM: the consumers read the user rows into registers themselves
                    mbar_wait(A_EMPTY, (it & 1) ^ 1);
                    mbar_expect_tx(A_FULL, C::A_BYTES);
                    for (int kb = 0; kb < KB; kb++) tma_load_2d(smem_u32(sA + kb * (TC_BM * 128)), &tmA, A_FULL, kb * 64, mb * TC_BM);
                    if (KT) tma_load_2d(smem_u32(sA + KB * (TC_BM * 128)), &tmAt, A_FULL, KB * 64, mb * TC_BM);
                }
                for (int t = 0; t < n_tiles; t++) {
                    const long long t0 = prof ? clock64() : 0;
                    mbar_wait(B_EMPTY(s), ph ^ 1);
                    if (prof) w_bempty += clock64() - t0;
                    mbar_expect_tx(B_FULL(s), C::B_BYTES);       // PAIR: half from this CTA, half multicast by the peer
                    if (PAIR) {
                        constexpr int H = BN / 2;                    // item rows of a tile this CTA fetches for both
                        for (int kb = 0; kb < KB; kb++)
                            tma_load_2d_mc(smem_u32(sB + s * C::B_BYTES + kb * (BN * 128) + rank * (H * 128)), &tmB, B_FULL(s), kb * 64,
                                           t * BN + (int)rank * H, (uint16_t)3);
                        if (KT) tma_load_2d_mc(smem_u32(sB + s * C::B_BYTES + KB * (BN * 128) + rank * (H * KT * 2)), &tmBt, B_FULL(s),
                                               KB * 64, t * BN + (int)rank * H, (uint16_t)3);
                    } else {
                        for (int kb = 0; kb < KB; kb++)
                            tma_load_2d(smem_u32(sB + s * C::B_BYTES + kb * (BN * 128)), &tmB, B_FULL(s), kb * 64, t * BN);
                        if (KT) tma_load_2d(smem_u32(sB + s * C::B_BYTES + KB * (BN * 128)), &tmBt, B_FULL(s), KB * 64, t * BN);
                    }
                    if (++s == S) { s = 0; ph ^= 1; }
                }
            }
            if (prof) p.prof[12] = w_bempty;
        }
    } else if (warp < 4 * NG) {
        // ===================== consumers: warpgroup 0 (warps 0-3) and, if NG == 2, warpgroup 1 (warps 4-7) =====================
        // Group g owns the tiles with (global tile counter % NG) == g and its own candidate buffers; the re-rank at the end of
        // every user block reads the groups' lists side by side.
        const int grp = NG == 2 ? (warp >> 2) : 0;
        const int quad = warp & 3;                    // warp inside the warpgroup
        const int row = tc_row(quad, lane);           // row inside the 128-user block
        const float NEG = -CUDART_INF_F;
        // candidate buffer: row-major [128 rows][BUFG slots] of sortable keys + item ids; logical slot s of row r
        // lives at physical position (s + r) & (BUFG - 1) (rotation: conflict-free appends AND conflict-free row reads)
        const uint32_t ckey = cval + (uint32_t)grp * GRPB;                    // uint32 keys [128][BUFG], then ids [128][BUFG]
        const uint32_t cidx = ckey + TC_BM * BUFG * 4;
        const uint32_t stw = stg + (uint32_t)(warp * C::STG_WARP);            // this warp's accumulator staging tile
        uint32_t tile = 0;
        long long c_wait = 0, c_ld = 0, c_scan = 0, c_comp = 0, c_rank = 0, n_comp = 0, n_slow = 0, n_grp = 0;
        const bool prof = DBG && p.prof != nullptr && warp == 0;
        constexpr int EPI_THREADS = 128 * NG;
        uint32_t ublk = 0;                            // user blocks this CTA has started
        for (int un = unit0; un < n_units; un += unit_step, ublk++) {
            const int mb = PAIR ? 2 * un + (int)rank : un;
            const int q = mb * TC_BM + row;           // position in the selected user range
            const bool valid = q < p.n_sel;
            const int u = p.user_begin + (valid ? q : 0);
            int64_t mbeg = 0; int mlen = 0;
            if (valid && p.mask_indptr) { mbeg = p.mask_indptr[u]; mlen = (int)(p.mask_indptr[u + 1] - mbeg); }
            // the CSR rows of the block's 128 consecutive users are ONE contiguous segment: copy as much of it as fits
            int64_t seg_beg = 0; int n_cached = 0;
            if (p.mask_indptr && C::MASKC > 0 && mb < n_mblocks) {
                const int q1 = min(mb * TC_BM + TC_BM, p.n_sel);
                seg_beg = p.mask_indptr[p.user_begin + mb * TC_BM];
                n_cached = (int)min(p.mask_indptr[p.user_begin + q1] - seg_beg, (int64_t)C::MASKC);
                for (int e = (int)threadIdx.x; e < n_cached; e += EPI_THREADS) sts_s32(mcache + 4u * (uint32_t)e, __ldg(p.mask_indices + seg_beg + e));
            }
            named_bar_sync(3, EPI_THREADS);
            // ATM: this thread's A fragments of both 64-row halves for every K = 16 step, straight from the bf16 user rows
            uint32_t afr[ATM ? 2 : 1][ATM ? KP / 16 : 1][4];
            if (ATM) {
#pragma unroll
                for (int h = 0; h < 2; h++) {
#pragma unroll
                    for (int hf = 0; hf < 2; hf++) {
                        const int rq = mb * TC_BM + h * 64 + quad * 16 + (lane >> 2) + 8 * hf;
                        const uint32_t *src = reinterpret_cast<const uint32_t *>(p.ubf + (int64_t)(rq < p.n_sel ? rq : 0) * KP) + (lane & 3);
#pragma unroll
                        for (int ks = 0; ks < (ATM ? KP / 16 : 1); ks++) {
                            afr[h][ks][hf] = rq < p.n_sel ? __ldg(src + ks * 8) : 0u;
                            afr[h][ks][2 + hf] = rq < p.n_sel ? __ldg(src + ks * 8 + 4) : 0u;
                        }
                    }
                }
            } else {
                mbar_wait(A_FULL, ublk & 1);          // the block's user rows are in shared memory
            }
            int cnt = 0;                              // filled logical slots of my row
            float thresh = (valid && debug_mode != 1) ? NEG : CUDART_INF_F;   // upper bound of everything dropped so far
            const uint32_t my_key = ckey + ROWB * (uint32_t)row, my_idx = cidx + ROWB * (uint32_t)row;
            // invariant: logical slots >= cnt hold -inf keys
#pragma unroll 8
            for (int sl = 0; sl < BUFG; sl++) sts_s32(my_key + 4u * (uint32_t)sl, (int)(TC_KEY_NEG | (uint32_t)(63 - sl)));
            __syncwarp();

            auto compact = [&](uint32_t todo) {
                const uint2 res = tc_compact_rows<BUFG, KCG>(todo, ckey, cidx, quad, lane, mlen, mbeg, p.mask_indices, seg_beg, n_cached,
                                                             mcache, p.n_items, cnt, thresh);
                cnt = (int)res.x; thresh = __uint_as_float(res.y);
            };

            for (int t = 0; t < n_tiles; t++, tile++) {
                if (NG == 2 && (int)(tile & 1u) != grp) continue;
                const int s = (int)(tile % (uint32_t)S);
                long long t0 = prof ? clock64() : 0;
                named_bar_sync(4 + grp, 128);         // the warpgroup issues its wgmma together
                mbar_wait(B_FULL(s), (tile / (uint32_t)S) & 1);
                long long t1 = prof ? clock64() : 0;
                if (prof) c_wait += t1 - t0;
                // ---- 128 users x BN items: two wgmma M = 64 halves per K = 16 step
                float acc0[BN / 2], acc1[BN / 2];
                {
                    const uint32_t a_addr = smem_u32(sA), b_addr = smem_u32(sB + s * C::B_BYTES);
                    wgmma_fence();
                    if constexpr (ATM) {
#pragma unroll
                        for (int ks = 0; ks < KP / 16; ks++) {
                            const int kb = ks / 4, k = ks % 4;
                            const uint64_t db = kb < KB ? gmma_desc_sw128(b_addr + kb * (BN * 128) + k * 32)
                                                        : gmma_desc_tail<KT ? KT : 16>(b_addr + KB * (BN * 128) + k * 32);
                            if (BN == 64) {
                                wgmma_m64n64k16_rs(acc0, afr[0][ks], db, ks != 0);
                                wgmma_m64n64k16_rs(acc1, afr[ATM ? 1 : 0][ks], db, ks != 0);
                            } else {
                                wgmma_m64n32k16_rs(acc0, afr[0][ks], db, ks != 0);
                                wgmma_m64n32k16_rs(acc1, afr[ATM ? 1 : 0][ks], db, ks != 0);
                            }
                        }
                    }
#pragma unroll
                    for (int kb = 0; kb < (ATM ? 0 : KB); kb++) {
#pragma unroll
                        for (int k = 0; k < 4; k++) {     // K = 16 bf16 = 32 B inside the 128-B swizzle atom
                            const uint64_t db = gmma_desc_sw128(b_addr + kb * (BN * 128) + k * 32);
                            const uint32_t aa = a_addr + kb * (TC_BM * 128) + k * 32;
                            const bool accum = (kb | k) != 0;
                            if (BN == 64) {
                                wgmma_m64n64k16<0, 0>(acc0, gmma_desc_sw128(aa), db, accum);
                                wgmma_m64n64k16<0, 0>(acc1, gmma_desc_sw128(aa + 64 * 128), db, accum);
                            } else {
                                wgmma_m64n32k16<0, 0>(acc0, gmma_desc_sw128(aa), db, accum);
                                wgmma_m64n32k16<0, 0>(acc1, gmma_desc_sw128(aa + 64 * 128), db, accum);
                            }
                        }
                    }
                    if (KT && !ATM) {                     // K tail: one (16 columns) or two (32) more K = 16 steps
                        constexpr int KTT = KT ? KT : 16;
#pragma unroll
                        for (int k = 0; k < KT / 16; k++) {
                            const uint64_t db = gmma_desc_tail<KTT>(b_addr + KB * (BN * 128) + k * 32);
                            const uint32_t aa = a_addr + KB * (TC_BM * 128) + k * 32;
                            const bool accum = (KB | k) != 0;
                            if (BN == 64) {
                                wgmma_m64n64k16<0, 0>(acc0, gmma_desc_tail<KTT>(aa), db, accum);
                                wgmma_m64n64k16<0, 0>(acc1, gmma_desc_tail<KTT>(aa + 64 * KTT * 2), db, accum);
                            } else {
                                wgmma_m64n32k16<0, 0>(acc0, gmma_desc_tail<KTT>(aa), db, accum);
                                wgmma_m64n32k16<0, 0>(acc1, gmma_desc_tail<KTT>(aa + 64 * KTT * 2), db, accum);
                            }
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_acc_fence<BN / 2>(acc0);
                    wgmma_acc_fence<BN / 2>(acc1);
                }
                if (threadIdx.x % 128 == 0) {         // B stage reusable: this group's MMAs have retired (PAIR: in both CTAs)
                    mbar_arrive(B_EMPTY(s));
                    if (PAIR) mbar_arrive_cluster(mapa_cluster(B_EMPTY(s), rank ^ 1u));
                }
                // ---- fragments -> one row per thread through this warp's staging tile: 16-byte chunk c of staged row r sits
                // at chunk c ^ (r % NCH) (conflict-free row-per-lane reads)
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const float *a = h ? acc1 : acc0;
#pragma unroll
                    for (int j = 0; j < BN / 8; j++) {
#pragma unroll
                        for (int hf = 0; hf < 2; hf++) {
                            const int lr = h * 16 + (lane >> 2) + 8 * hf;
                            const int col = 8 * j + 2 * (lane & 3);
                            const uint32_t dst = stw + (uint32_t)(lr * BN * 4) + (uint32_t)((((col >> 2) ^ (lr & (NCH - 1))) << 4) | ((col & 3) << 2));
                            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(dst), "f"(a[4 * j + 2 * hf]), "f"(a[4 * j + 2 * hf + 1]) : "memory");
                        }
                    }
                }
                __syncwarp();
                float v[BN];
#pragma unroll
                for (int c = 0; c < NCH; c++) {
                    const uint32_t src = stw + (uint32_t)(lane * BN * 4) + (uint32_t)((c ^ (lane & (NCH - 1))) << 4);
                    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                                 : "=f"(v[4 * c]), "=f"(v[4 * c + 1]), "=f"(v[4 * c + 2]), "=f"(v[4 * c + 3]) : "r"(src) : "memory");
                }
                if (prof) c_ld += clock64() - t1;
                long long t2 = prof ? clock64() : 0;
                const int col0 = t * BN;
                if (DUMP) {
                    if (valid)
                        for (int c = 0; c < BN; c++)
                            if (col0 + c < p.n_items) p.dump[(int64_t)q * p.n_items + col0 + c] = v[c];
                }
                // max of each group of 8 columns (fast reject), 3-input max trees
                constexpr int NS8 = BN / 8;
                float g[NS8];
#pragma unroll
                for (int s8 = 0; s8 < NS8; s8++) {
                    const float *w = v + s8 * 8;
                    g[s8] = fmaxf(fmaxf(fmaxf(w[0], w[1]), w[2]), fmaxf(fmaxf(fmaxf(w[3], w[4]), w[5]), fmaxf(w[6], w[7])));
                }
                // bias bound per 32-item chunk (bm1: the second chunk of a 64-item tile)
                float bm0 = 0.f, bm1 = 0.f;
                if (HAS_BIAS) {
                    bm0 = __ldg(p.bmax_chunk + (col0 >> 5));
                    if (BN == 64) bm1 = __ldg(p.bmax_chunk + min((col0 >> 5) + 1, (p.n_items - 1) >> 5));
                }
                float m64;
                if (BN == 64)
                    m64 = HAS_BIAS ? fmaxf(fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3])) + bm0, fmaxf(fmaxf(g[NS8 - 4], g[NS8 - 3]), fmaxf(g[NS8 - 2], g[NS8 - 1])) + bm1)
                                   : fmaxf(fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3])), fmaxf(fmaxf(g[NS8 - 4], g[NS8 - 3]), fmaxf(g[NS8 - 2], g[NS8 - 1])));
                else
                    m64 = fmaxf(fmaxf(g[0], g[1]), fmaxf(g[2], g[3])) + (HAS_BIAS ? bm0 : 0.f);
                if (__any_sync(0xffffffffu, m64 > thresh)) {
                    if (DBG) n_slow++;
#pragma unroll
                    for (int s8 = 0; s8 < NS8; s8++) {
                        const float bm = s8 < 4 ? bm0 : bm1;
                        if (!__any_sync(0xffffffffu, (HAS_BIAS ? g[s8] + bm : g[s8]) > thresh)) continue;
                        if (DBG) n_grp++;
                        // Append survivors one at a time, largest first: locate the group's max with static
                        // compares, append it (branch-free), knock it out and re-evaluate the group max.  Almost
                        // always one round: ~45 instructions instead of ~150 for 8 unconditional append slots.
                        float w8[8];
#pragma unroll
                        for (int c = 0; c < 8; c++)
                            w8[c] = HAS_BIAS ? v[s8 * 8 + c] + __ldg(p.bias + min(col0 + s8 * 8 + c, p.n_items - 1)) : v[s8 * 8 + c];
                        float gm = fmaxf(fmaxf(fmaxf(w8[0], w8[1]), w8[2]), fmaxf(fmaxf(fmaxf(w8[3], w8[4]), w8[5]), fmaxf(w8[6], w8[7])));
#pragma unroll 1
                        for (int round = 0; round < 8; round++) {
                            if (!__any_sync(0xffffffffu, gm > thresh)) break;
                            // a row is compacted only when an append finds its buffer FULL (not 8 slots early): with 32 slots
                            // and 16 kept that is 16 appends per compaction instead of 9-16
                            const uint32_t todo = __ballot_sync(0xffffffffu, gm > thresh && cnt >= BUFG);
                            if (todo) {
                                long long t3 = prof ? clock64() : 0;
                                if (DBG) n_comp += __popc(todo);
                                if (debug_mode == 2) { if (cnt >= BUFG) { cnt = 0; thresh = 0.3f; } } else compact(todo);
                                if (prof) { long long dt = clock64() - t3; c_comp += dt; c_scan -= dt; }
                                if (!__any_sync(0xffffffffu, gm > thresh)) break;       // the thresholds just rose
                            }
                            int am = 7;
#pragma unroll
                            for (int c = 6; c >= 0; c--) am = (w8[c] == gm) ? c : am;      // first position holding the max
                            const uint32_t take = gm > thresh ? 1u : 0u;
                            const int pos = (cnt + row) & (BUFG - 1);
                            const uint32_t key = tc_key_of(gm, pos);
                            asm volatile(
                                "{\n\t.reg .pred p;\n\t"
                                "setp.ne.u32 p, %0, 0;\n\t"
                                "@p st.shared.u32 [%1], %2;\n\t"
                                "@p st.shared.s32 [%3], %4;\n\t}"
                                ::"r"(take), "r"(my_key + 4u * (uint32_t)pos), "r"(key), "r"(my_idx + 4u * (uint32_t)pos),
                                  "r"(col0 + s8 * 8 + am)
                                : "memory");
                            cnt += (int)take;
#pragma unroll
                            for (int c = 0; c < 8; c++) w8[c] = (take && c == am) ? -CUDART_INF_F : w8[c];
                            gm = fmaxf(fmaxf(fmaxf(w8[0], w8[1]), w8[2]), fmaxf(fmaxf(fmaxf(w8[3], w8[4]), w8[5]), fmaxf(w8[6], w8[7])));
                        }
                    }
                }
                if (prof) c_scan += clock64() - t2;
            }
            if (!ATM && threadIdx.x % 128 == 0) mbar_arrive(A_EMPTY);  // this group's MMAs of the block have all retired
            // final compaction: every row ends with its <= KC best unmasked candidates in logical slots 0..cnt-1
            __syncwarp();
            long long t4 = prof ? clock64() : 0;
            compact(__ballot_sync(0xffffffffu, valid));
            sts_s32(mrg + 1024u * (uint32_t)grp + 4u * (uint32_t)row, cnt);
            sts_f32(mrg + 1024u * (uint32_t)grp + 512u + 4u * (uint32_t)row, thresh);
            if (NG == 2) named_bar_sync(1, EPI_THREADS);      // both groups' lists are final
            else __syncwarp();

            const float vmax_n = p.vstat[0], bmax_a = p.vstat[1];
            const float my_unorm = valid ? p.unorm[q] : 0.f;
            // ---- exact re-rank (rows split between the groups): lane l re-scores candidate l of the row in fp32 with the
            // SAME operation order as score_topk.cu (32 strided partial sums, then the xor-butterfly tree)
            for (int r = (NG == 2 ? grp * 16 : 0); r < (NG == 2 ? grp * 16 + 16 : 32); r++) {
                const int rrow = tc_row(quad, r);
                const int rq = mb * TC_BM + rrow;
                if (rq >= p.n_sel) continue;                                 // warp-uniform
                const int ru = p.user_begin + rq;
                // lanes [g * KCG, g * KCG + cnt_g) take group g's list; everything either group dropped is <= the larger tau
                const int lg = NG == 2 ? lane / KCG : 0, ls = lane - lg * KCG;
                const int c0 = lds_s32(mrg + 4u * (uint32_t)rrow), c1 = NG == 2 ? lds_s32(mrg + 1024u + 4u * (uint32_t)rrow) : 0;
                const int rcount = c0 + c1;
                float rthresh = lds_f32(mrg + 512u + 4u * (uint32_t)rrow);
                if (NG == 2) rthresh = fmaxf(rthresh, lds_f32(mrg + 1024u + 512u + 4u * (uint32_t)rrow));
                const bool have = ls < (lg ? c1 : c0);
                const int my_i = have ? lds_s32(cval + (uint32_t)lg * GRPB + TC_BM * BUFG * 4 + ROWB * (uint32_t)rrow +
                                                4u * (uint32_t)((ls + rrow) & (BUFG - 1)))
                                      : 0x7fffffff;
                float my_v = NEG;
                if (have) {
                    const float *ur = p.U + (int64_t)ru * p.ld;
                    const float *vr = p.V + (int64_t)my_i * p.ld;
                    float ps[32];
#pragma unroll
                    for (int tt = 0; tt < 32; tt++) ps[tt] = 0.f;
                    for (int base = 0; base < p.d; base += 32) {
#pragma unroll
                        for (int tt = 0; tt < 32; tt += 4) {
                            if (base + tt + 3 < p.d) {
                                const float4 a4 = __ldg(reinterpret_cast<const float4 *>(ur + base + tt));
                                const float4 b4 = *reinterpret_cast<const float4 *>(vr + base + tt);
                                ps[tt] = fmaf(a4.x, b4.x, ps[tt]); ps[tt + 1] = fmaf(a4.y, b4.y, ps[tt + 1]);
                                ps[tt + 2] = fmaf(a4.z, b4.z, ps[tt + 2]); ps[tt + 3] = fmaf(a4.w, b4.w, ps[tt + 3]);
                            } else {
#pragma unroll
                                for (int e = 0; e < 4; e++)
                                    if (base + tt + e < p.d) ps[tt + e] = fmaf(__ldg(ur + base + tt + e), vr[base + tt + e], ps[tt + e]);
                            }
                        }
                    }
#pragma unroll
                    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
                        for (int tt = 0; tt < off; tt++) ps[tt] = ps[tt] + ps[tt + off];
                    my_v = (p.bias ? p.bias[my_i] : 0.f) + ps[0];
                }
                // bitonic sort over 32 lanes: (score desc, index asc)
                float sv = my_v; int si = my_i;
#pragma unroll
                for (int kk = 2; kk <= 32; kk <<= 1) {
#pragma unroll
                    for (int j = kk >> 1; j > 0; j >>= 1) {
                        const float ov = __shfl_xor_sync(0xffffffffu, sv, j);
                        const int oi = __shfl_xor_sync(0xffffffffu, si, j);
                        const bool up = ((lane & kk) == 0);
                        const bool lower = ((lane & j) == 0);
                        const bool other_first = cand_better(ov, oi, sv, si);
                        const bool take = (up == lower) ? other_first : !other_first;
                        if (take) { sv = ov; si = oi; }
                    }
                }
                // certification: the k-th exact score must clear tau + eps_u (tau = -inf if nothing was ever dropped)
                const float un = __shfl_sync(0xffffffffu, my_unorm, r);
                const float eps = p.eps_scale * un * vmax_n + 1e-6f * un * vmax_n + 4e-5f * bmax_a;   // bias: hi+lo bf16 split, 2^-17 rel
                const float kth = __shfl_sync(0xffffffffu, sv, p.k - 1);
                const bool certified = !(rthresh > NEG) || (kth > rthresh + eps) || debug_mode != 0;
                if (lane < p.k) {
                    const bool ok = lane < rcount && sv > NEG;
                    p.out_idx[(int64_t)rq * p.k + lane] = ok ? si : -1;
                    p.out_val[(int64_t)rq * p.k + lane] = ok ? sv : NEG;
                }
                if (!certified && lane == 0) {
                    const int slot = atomicAdd(p.flag_count, 1);
                    p.flag_list[slot] = rq;
                }
            }
            __syncwarp();
            named_bar_sync(2, EPI_THREADS);      // every list has been read: buffers and mask cache are free for the next user block
            if (prof) c_rank += clock64() - t4;
        }
        if (prof && lane == 0 && blockIdx.x == 0) {
            p.prof[0] = c_wait; p.prof[1] = c_ld; p.prof[2] = c_scan; p.prof[3] = c_comp; p.prof[4] = c_rank;
            p.prof[5] = n_comp; p.prof[6] = n_slow; p.prof[7] = n_grp;
        }
    }
    if (PAIR) cluster_sync_all();     // no CTA leaves while its peer may still multicast into it or signal its barriers
}

// ---------------------------------------------------------------- preparation kernels
// fp32 rows [n, ld] (first d valid) -> bf16 rows [n, KP] zero padded; row norms; optional max
// fold: 0 none; 1 (user side) columns d, d+1 = 1.0; 2 (item side) columns d, d+1 = bf16 hi / lo parts of bias[row]
__global__ void tc_convert_kernel(const float *src, int64_t n, int d, int ld, int row0, __nv_bfloat16 *dst, int KP,
                                  float *norms, float *norm_max, int fold, const float *bias) {
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    float wmax = 0.f;
    for (; w < n; w += nw) {
        const float *r = src + (row0 + w) * (int64_t)ld;
        float ss = 0.f;
        for (int k = lane; k < KP; k += 32) {
            const float x = k < d ? r[k] : 0.f;
            ss += x * x;
            __nv_bfloat16 o = __float2bfloat16_rn(x);
            if (fold == 1 && (k == d || k == d + 1)) o = __float2bfloat16_rn(1.f);
            if (fold == 2 && (k == d || k == d + 1)) {
                const float b = bias[row0 + w];
                const __nv_bfloat16 hi = __float2bfloat16_rn(b);
                o = k == d ? hi : __float2bfloat16_rn(b - __bfloat162float(hi));
            }
            dst[w * KP + k] = o;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, off);
        const float nr = sqrtf(ss) * (1.f + 1e-6f);
        if (norms && lane == 0) norms[w] = nr;
        wmax = fmaxf(wmax, nr);
    }
    if (norm_max && lane == 0 && wmax > 0.f) atomicMax(reinterpret_cast<int *>(norm_max), __float_as_int(wmax));
}

__global__ void tc_bias_kernel(const float *bias, int32_t n_items, float *bmax_chunk, float *babs_max) {
    const int chunk = blockIdx.x * blockDim.x + threadIdx.x;
    const int nchunks = (n_items + 31) / 32;
    if (chunk >= nchunks) return;
    float m = -CUDART_INF_F, a = 0.f;
    for (int c = chunk * 32; c < min(chunk * 32 + 32, n_items); c++) { m = fmaxf(m, bias[c]); a = fmaxf(a, fabsf(bias[c])); }
    bmax_chunk[chunk] = m;
    atomicMax(reinterpret_cast<int *>(babs_max), __float_as_int(a));
}

// ---------------------------------------------------------------- host side
extern "C" size_t eb_score_recheck_workspace_bytes(int64_t n_sel_max, int32_t n_items);    // score_topk.cu

typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                             const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn get_encode() {
    static EncodeFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = (EncodeFn)p;
    }
    return fn;
}

// {box_cols bf16, box_rows} boxes starting at any column of a [rows, KP] bf16 matrix; box_cols 64 -> SWIZZLE_128B,
// 32 -> SWIZZLE_64B, 16 -> SWIZZLE_32B (the box's inner extent is exactly the swizzle span)
static int make_map(CUtensorMap *m, void *base, uint64_t rows, int KP, uint32_t box_cols, uint32_t box_rows) {
    EncodeFn enc = get_encode();
    if (!enc) return set_err(EB_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[2] = {(cuuint64_t)KP, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)KP * 2};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapSwizzle sw = box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : (box_cols == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_err(EB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return EB_OK;
}

static inline size_t al(size_t x) { return (x + 1023) / 1024 * 1024; }

struct TcLayout {
    size_t ubf, vbf, unorm, vstat, bmax, flag_count, flag_list, exact_ws, total, exact_bytes;
    int KP;
};

// fold = the item bias travels through the MMA as two extra K columns (bf16 hi + lo) against ones on the user side
static TcLayout tc_layout(int64_t n_sel, int32_t n_items, int d, bool fold) {
    TcLayout L;
    L.KP = (d + (fold ? 2 : 0) + 15) / 16 * 16;          // K padded to the MMA's K = 16 ...
    if (L.KP % 64 == 48) L.KP += 16;                     // ... except that a 48-column tail becomes a full 64-wide block
    size_t off = 0;
    L.ubf = off; off += al((size_t)n_sel * L.KP * 2);
    L.vbf = off; off += al((size_t)n_items * L.KP * 2);
    L.unorm = off; off += al((size_t)n_sel * 4);
    L.vstat = off; off += al(64);
    L.bmax = off; off += al(((size_t)n_items + 31) / 32 * 4);
    L.flag_count = off; off += al(256);
    L.flag_list = off; off += al((size_t)n_sel * 4);
    L.exact_bytes = eb_score_recheck_workspace_bytes(n_sel, n_items);
    L.exact_ws = off; off += al(L.exact_bytes);
    L.total = off;
    return L;
}

struct TcMaps { CUtensorMap a, b, at, bt; };

template <int KP, bool HAS_BIAS, int NG, bool PAIR, bool ATM, bool DBG>
static int launch_tc3(const TcMaps &m, const TcParams &p, int n_mblocks, cudaStream_t st) {
    using C = TcCfg<KP, NG, PAIR, ATM>;
    auto kern = score_topk_tc_kernel<KP, HAS_BIAS, NG, PAIR, ATM, DBG>;
    EB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    if (!PAIR) {
        int grid = sm_count();
        if (grid > n_mblocks) grid = n_mblocks;
        kern<<<grid, C::THREADS, C::SMEM, st>>>(m.a, m.b, m.at, m.bt, p);
    } else {
        // clusters of two CTAs: a cluster scores two user blocks against every item tile
        int clusters = sm_count() / 2;
        if (clusters > (n_mblocks + 1) / 2) clusters = (n_mblocks + 1) / 2;
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(2 * clusters); cfg.blockDim = dim3(C::THREADS); cfg.dynamicSmemBytes = C::SMEM; cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        EB_CUDA(cudaLaunchKernelEx(&cfg, kern, m.a, m.b, m.at, m.bt, p));
    }
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

template <int KP, int NG, bool PAIR, bool ATM>
static int launch_tc(void *ubf, void *vbf, const TcParams &p, int n_mblocks, cudaStream_t st) {
    using C = TcCfg<KP, NG, PAIR, ATM>;
    constexpr int BL = PAIR ? C::BN / 2 : C::BN;           // item rows per TMA box (PAIR: each CTA fetches half a tile)
    TcMaps m;
    // a tile without full blocks (KP = 16 / 32) still needs valid descriptors in the unused slots
    const uint32_t bc = C::KB ? 64 : C::KT, tc = C::KT ? C::KT : 64;
    if (int rc = make_map(&m.a, ubf, (uint64_t)p.n_sel, KP, bc, TC_BM)) return rc;
    if (int rc = make_map(&m.b, vbf, (uint64_t)p.n_items, KP, bc, BL)) return rc;
    if (int rc = make_map(&m.at, ubf, (uint64_t)p.n_sel, KP, tc, TC_BM)) return rc;
    if (int rc = make_map(&m.bt, vbf, (uint64_t)p.n_items, KP, tc, BL)) return rc;
    const bool hb = p.bias != nullptr && !p.bias_folded;    // epilogue adds the bias only when it is not folded into the MMA
    // the lean kernel exists for the default layout only; the others always carry the instrumentation
    constexpr bool LEAN = NG == 2 && !PAIR && !ATM;
    const bool dbg = p.dump != nullptr || p.prof != nullptr || p.debug_mode != 0;
    if (LEAN && !dbg)
        return hb ? launch_tc3<KP, true, NG, PAIR, ATM, !LEAN>(m, p, n_mblocks, st) : launch_tc3<KP, false, NG, PAIR, ATM, !LEAN>(m, p, n_mblocks, st);
    return hb ? launch_tc3<KP, true, NG, PAIR, ATM, true>(m, p, n_mblocks, st) : launch_tc3<KP, false, NG, PAIR, ATM, true>(m, p, n_mblocks, st);
}

}  // namespace eb

using namespace eb;

extern "C" size_t eb_score_topk_tc_workspace_bytes(int64_t n_sel, int32_t n_items, int d) {
    if (n_sel < 1) n_sel = 1;
    return tc_layout(n_sel, n_items, d, d + 2 <= 256).total;    // sized for the bias-folded layout (the larger one)
}

// internal entry of score_topk.cu with an output-row map (re-check of uncertified users)
extern "C" int eb_score_topk_f32_mapped(const float *U, const float *V, const float *item_bias, int32_t n_items, int d,
                                        int ld, const int64_t *mask_indptr, const int32_t *mask_indices,
                                        const int32_t *positions, int32_t user_begin, int64_t n_sel, int k,
                                        int32_t *out_idx, float *out_val, void *workspace, size_t workspace_bytes,
                                        void *stream);
// the same with the number of rows read from device memory at kernel start (n_rows_dev[0] <= n_sel_max)
extern "C" int eb_score_topk_f32_mapped_dev(const float *U, const float *V, const float *item_bias, int32_t n_items, int d,
                                            int ld, const int64_t *mask_indptr, const int32_t *mask_indices,
                                            const int32_t *positions, const int32_t *n_rows_dev, int32_t user_begin,
                                            int64_t n_sel_max, int k, int32_t *out_idx, float *out_val, void *workspace,
                                            size_t workspace_bytes, void *stream);

extern "C" int eb_score_topk_tc_f32(const float *U, const float *V, const float *item_bias, int32_t n_items, int d, int ld,
                                    const int64_t *mask_indptr, const int32_t *mask_indices, int32_t user_begin,
                                    int64_t n_sel, int k, int32_t *out_idx, float *out_val, float *dump,
                                    void *workspace, size_t workspace_bytes, int64_t *stats_host, void *stream) {
    EB_ARG(U && V && out_idx && out_val && workspace, "null pointer");
    EB_ARG(d >= 1 && d <= 256 && ld >= d, "tensor-core scoring supports 1 <= d <= 256 (d=%d ld=%d)", d, ld);
    EB_ARG(k >= 1 && k <= 16, "tensor-core scoring keeps 32 candidates per user: k must be <= 16 (k=%d); "
                              "use eb_score_topk_f32 for longer lists", k);
    EB_ARG(n_items >= 1 && n_sel >= 0 && n_sel < (1ll << 31), "bad sizes");
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel == 0) return EB_OK;
    int cc = 0;
    if (int rc = eb_device_info(nullptr, &cc)) return rc;
    if (cc != 90) return set_err(EB_ERR_CUDA, "the wgmma scoring kernel is built for compute capability 9.0 (got %d)", cc);
    const bool fold = item_bias != nullptr && d + 2 <= 256;
    const TcLayout L = tc_layout(n_sel, n_items, d, fold);
    if (workspace_bytes < L.total) return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace_bytes, L.total);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    __nv_bfloat16 *ubf = (__nv_bfloat16 *)(ws + L.ubf), *vbf = (__nv_bfloat16 *)(ws + L.vbf);
    float *unorm = (float *)(ws + L.unorm), *vstat = (float *)(ws + L.vstat), *bmax = (float *)(ws + L.bmax);
    int32_t *flag_count = (int32_t *)(ws + L.flag_count), *flag_list = (int32_t *)(ws + L.flag_list);
    EB_CUDA(cudaMemsetAsync(vstat, 0, 64, st));
    EB_CUDA(cudaMemsetAsync(flag_count, 0, 256, st));
    const int cgrid = sm_count() * 8;
    tc_convert_kernel<<<cgrid, 256, 0, st>>>(U, n_sel, d, ld, user_begin, ubf, L.KP, unorm, nullptr, fold ? 1 : 0, nullptr);
    tc_convert_kernel<<<cgrid, 256, 0, st>>>(V, n_items, d, ld, 0, vbf, L.KP, nullptr, vstat, fold ? 2 : 0, item_bias);
    if (item_bias) tc_bias_kernel<<<((n_items + 31) / 32 + 255) / 256, 256, 0, st>>>(item_bias, n_items, bmax, vstat + 1);
    EB_CUDA(cudaGetLastError());
    TcParams p{};
    p.U = U; p.V = V; p.bias = item_bias; p.d = d; p.ld = ld; p.n_items = n_items;
    p.mask_indptr = mask_indptr; p.mask_indices = mask_indices; p.user_begin = user_begin; p.n_sel = (int32_t)n_sel; p.k = k;
    p.ubf = ubf; p.unorm = unorm; p.vstat = vstat; p.bmax_chunk = item_bias ? bmax : nullptr; p.bias_folded = fold ? 1 : 0;
    p.out_idx = out_idx; p.out_val = out_val; p.flag_count = flag_count; p.flag_list = flag_list; p.dump = dump;
    // bf16 RN: |x~-x| <= 2^-9|x|  =>  |u~.v~ - u.v| <= (2^-8 + 2^-18) ||u|| ||v||; +2% for fp32 accumulation and re-rank rounding
    p.eps_scale = 1.02f * (1.f / 256.f);
    { const char *dbg = getenv("EB_TC_DEBUG"); p.debug_mode = dbg ? atoi(dbg) : 0; }
    p.prof = (stats_host && getenv("EB_TC_PROF")) ? (long long *)(flag_count + 16) : nullptr;
    const int n_mblocks = (int)((n_sel + TC_BM - 1) / TC_BM);
    // consumer warpgroups: two by default (see TcCfg); EB_TC_NG=1 selects the single-group kernel for A/B measurements
    int ng = 2;
    { const char *e = getenv("EB_TC_NG"); if (e && atoi(e) == 1) ng = 1; }
    // CTA pairs sharing every item tile through TMA multicast (see TcCfg): EB_TC_PAIR=1 (two consumer groups only)
    bool pair = false;
    { const char *e = getenv("EB_TC_PAIR"); if (e && atoi(e) == 1 && ng == 2) pair = true; }
    // the user block in registers instead of shared memory (see TcCfg): EB_TC_ATM=1
    bool atm = false;
    { const char *e = getenv("EB_TC_ATM"); if (e && atoi(e) == 1 && ng == 2 && !pair) atm = true; }
    int rc;
    switch (L.KP) {
#define EB_TC_CASE(K) case K: rc = ng == 2 ? launch_tc<K, 2, false, false>(ubf, vbf, p, n_mblocks, st)                           \
                                          : launch_tc<K, 1, false, false>(ubf, vbf, p, n_mblocks, st); break;
        // the measured variants (CTA pairs, users in registers) exist for d = 64 and 128 with and without bias
#define EB_TC_CASE_X(K) case K: rc = pair ? launch_tc<K, 2, true, false>(ubf, vbf, p, n_mblocks, st)                            \
                                         : (atm ? launch_tc<K, 2, false, true>(ubf, vbf, p, n_mblocks, st)                     \
                                                : (ng == 2 ? launch_tc<K, 2, false, false>(ubf, vbf, p, n_mblocks, st)         \
                                                           : launch_tc<K, 1, false, false>(ubf, vbf, p, n_mblocks, st))); break;
        EB_TC_CASE(16) EB_TC_CASE(32) EB_TC_CASE_X(64) EB_TC_CASE_X(80) EB_TC_CASE(96) EB_TC_CASE_X(128) EB_TC_CASE_X(144)
        EB_TC_CASE(160) EB_TC_CASE(192) EB_TC_CASE(208) EB_TC_CASE(224) EB_TC_CASE(256)
#undef EB_TC_CASE
#undef EB_TC_CASE_X
        default: return set_err(EB_ERR_ARG, "internal: unsupported padded K %d", L.KP);
    }
    if (rc) return rc;
    // provably-exact re-check of the users the bound could not certify: launched unconditionally over the DEVICE-side
    // count (no host round trip per call; with nothing flagged the CTAs exit at once)
    rc = eb_score_topk_f32_mapped_dev(U, V, item_bias, n_items, d, ld, mask_indptr, mask_indices, flag_list, flag_count, user_begin,
                                      n_sel, k, out_idx, out_val, ws + L.exact_ws, L.exact_bytes, stream);
    if (rc) return rc;
    if (stats_host) {                                   // statistics are the only reason to synchronise
        int32_t flagged = 0;
        EB_CUDA(cudaMemcpyAsync(&flagged, flag_count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        EB_CUDA(cudaStreamSynchronize(st));
        stats_host[0] = flagged; stats_host[1] = L.KP;
        if (p.prof) EB_CUDA(cudaMemcpy(stats_host + 2, p.prof, 14 * sizeof(long long), cudaMemcpyDeviceToHost));
    }
    return EB_OK;
}
