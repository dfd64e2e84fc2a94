// mt_sampler.cu — bit-exact device replay of the reference's negative sampler stream.
//
// Replaces Sampler.__init__/step (elliot/dataset/samplers/custom_sampler.py:14-46): the
// reference draws every (u, i, j) from ONE legacy numpy MT19937 stream seeded with 42,
// with a data-dependent number of 32-bit draws per triple (masked rejection in randint,
// redraw while j is a train item).  The stream is serial by construction; it is replayed
// on the GPU in four data-parallel steps:
//   1. mt_generate_kernel : one CTA regenerates the MT19937 state 624 words at a time
//      (three dependent waves of 227 words + the last word) and writes the tempered
//      outputs;
//   2. mt_parse_kernel    : EVERY stream position speculatively parses the triple that
//      would start there and records where the next triple would start;
//   3. chain_*_kernel     : the true triple starts are the chain 0 -> next(0) -> ...;
//      it is resolved per block of positions (backward DP inside a block, one short
//      serial walk across blocks);
//   4. emit_kernel        : blocks write their triples at their global offsets; the
//      position after the last triple advances the persistent state.
#include "common.cuh"

namespace eb {

constexpr int MT_N = 624, MT_M = 397;
constexpr int CHAIN_L = 512;          // positions per chain block
constexpr int32_t INCOMPLETE = 0x7fffffff;

struct MtStatus {
    int64_t produced;   // triples emitted
    int64_t consumed;   // raw draws consumed by them
    int32_t error;      // 1: user owning every item / empty user
    int32_t pad;
};

__device__ __forceinline__ uint32_t mt_mix(uint32_t a, uint32_t b) {
    const uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
    return (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}
__device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
}

// mt[] in shared memory, all threads of the CTA participate
__device__ void mt_twist_cta(uint32_t *mt) {
    const int tid = threadIdx.x;
    uint32_t v = 0;
    // wave A: k in [0,227) uses old k, k+1, k+397
    if (tid < MT_N - MT_M) v = mt[tid + MT_M] ^ mt_mix(mt[tid], mt[tid + 1]);
    __syncthreads();
    if (tid < MT_N - MT_M) mt[tid] = v;
    __syncthreads();
    // wave B: k in [227,454) uses new k-227, old k, k+1
    if (tid < 227) { const int k = tid + 227; v = mt[k - 227] ^ mt_mix(mt[k], mt[k + 1]); }
    __syncthreads();
    if (tid < 227) mt[tid + 227] = v;
    __syncthreads();
    // wave C: k in [454,623) uses new k-227, old k, k+1
    if (tid < 169) { const int k = tid + 454; v = mt[k - 227] ^ mt_mix(mt[k], mt[k + 1]); }
    __syncthreads();
    if (tid < 169) mt[tid + 454] = v;
    __syncthreads();
    if (tid == 0) mt[MT_N - 1] = mt[MT_M - 1] ^ mt_mix(mt[MT_N - 1], mt[0]);
    __syncthreads();
}

// Generates `n` tempered outputs starting at the state's position.  If `out` is null the
// outputs are discarded.  If `commit` the advanced state is written back.
// n_ptr (optional, device) overrides n (used to advance by a count computed on device).
__global__ void __launch_bounds__(256) mt_generate_kernel(uint32_t *state, uint32_t *out, int64_t n,
                                                          const int64_t *n_ptr, int commit) {
    __shared__ uint32_t mt[MT_N];
    __shared__ int s_pos;
    for (int k = threadIdx.x; k < MT_N; k += blockDim.x) mt[k] = state[k];
    if (threadIdx.x == 0) s_pos = (int)state[MT_N];
    __syncthreads();
    if (n_ptr) n = *n_ptr;
    int pos = s_pos;
    int64_t done = 0;
    while (done < n) {
        if (pos == MT_N) { mt_twist_cta(mt); pos = 0; }
        int64_t take = MT_N - pos;
        if (take > n - done) take = n - done;
        if (out)
            for (int k = threadIdx.x; k < take; k += blockDim.x) out[done + k] = mt_temper(mt[pos + k]);
        pos += (int)take;
        done += take;
    }
    __syncthreads();
    if (commit) {
        for (int k = threadIdx.x; k < MT_N; k += blockDim.x) state[k] = mt[k];
        if (threadIdx.x == 0) state[MT_N] = (uint32_t)pos;
    }
}

__global__ void mt_seed_kernel(uint32_t *state, uint32_t seed) {
    // init_genrand (serial recurrence, 624 steps)
    uint32_t x = seed;
    state[0] = x;
    for (int i = 1; i < MT_N; i++) {
        x = 1812433253u * (x ^ (x >> 30)) + (uint32_t)i;
        state[i] = x;
    }
    state[MT_N] = MT_N;
}

__device__ __forceinline__ uint32_t mask_for(uint32_t rng) {
    uint32_t m = rng;
    m |= m >> 1; m |= m >> 2; m |= m >> 4; m |= m >> 8; m |= m >> 16;
    return m;
}

struct ParseParams {
    const uint32_t *raw;
    int64_t n_raw;
    int32_t n_users, n_items;
    const int64_t *indptr;
    const int32_t *set_indices, *sorted_indices;
    int4 *parsed;   // (u, i, j, next)
    MtStatus *status;
};

// legacy randint(n): rng = n-1; rng == 0 -> 0 without a draw; else masked rejection
__device__ __forceinline__ bool draw_bounded(const uint32_t *raw, int64_t n_raw, int64_t &q, uint32_t rng, uint32_t mask,
                                             uint32_t &val) {
    if (rng == 0) { val = 0; return true; }
    while (q < n_raw) {
        const uint32_t v = __ldg(raw + q) & mask;
        q++;
        if (v <= rng) { val = v; return true; }
    }
    return false;
}

__global__ void __launch_bounds__(256) mt_parse_kernel(const ParseParams p) {
    const int64_t pos = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= p.n_raw) return;
    int64_t q = pos;
    int4 res = make_int4(-1, -1, -1, INCOMPLETE);
    uint32_t u, pi, j;
    const uint32_t rng_u = (uint32_t)(p.n_users - 1), rng_i = (uint32_t)(p.n_items - 1);
    if (draw_bounded(p.raw, p.n_raw, q, rng_u, mask_for(rng_u), u)) {       // custom_sampler.py:32
        const int64_t beg = __ldg(p.indptr + u);
        const int lui = (int)(__ldg(p.indptr + u + 1) - beg);
        if (lui <= 0 || lui >= p.n_items) {
            // custom_sampler.py:35-41 recurses/spins forever here; only an error if this
            // position is really on the chain -> recorded lazily by the emitter (u = -2)
            res.x = -2;
        } else if (draw_bounded(p.raw, p.n_raw, q, (uint32_t)(lui - 1), mask_for((uint32_t)(lui - 1)), pi)) {
            const int32_t it = __ldg(p.set_indices + beg + pi);               // custom_sampler.py:37
            const int32_t *row = p.sorted_indices + beg;
            const uint32_t mask_i = mask_for(rng_i);
            bool ok = false;
            while (draw_bounded(p.raw, p.n_raw, q, rng_i, mask_i, j)) {     // custom_sampler.py:39-41
                if (!contains_sorted(row, lui, (int32_t)j)) { ok = true; break; }
                if (rng_i == 0) break;
            }
            if (ok) res = make_int4((int)u, it, (int)j, (int)(q - pos));
        }
    }
    p.parsed[pos] = res;
}

// backward DP inside each block of CHAIN_L positions: exit position + number of triples
__global__ void __launch_bounds__(128) chain_block_kernel(const int4 *parsed, int64_t n_raw, int64_t *exit_pos,
                                                          int32_t *cnt) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t start = b * CHAIN_L;
    if (start >= n_raw) return;
    const int64_t end = (start + CHAIN_L < n_raw) ? start + CHAIN_L : n_raw;
    for (int64_t pos = end - 1; pos >= start; pos--) {
        const int4 r = parsed[pos];
        if (r.w == INCOMPLETE) { exit_pos[pos] = -1; cnt[pos] = 0; continue; }
        const int64_t nx = pos + r.w;
        if (nx >= end) { exit_pos[pos] = nx; cnt[pos] = 1; }
        else if (r.w == 0) { exit_pos[pos] = -1; cnt[pos] = 0; }  // zero-length triple (all ranges 1): degenerate
        else { exit_pos[pos] = exit_pos[nx]; cnt[pos] = cnt[nx] + 1; }
    }
}

// serial walk over blocks: entry position and first triple index of each visited block
__global__ void chain_walk_kernel(const int64_t *exit_pos, const int32_t *cnt, int64_t n_raw, int64_t events,
                                  int64_t *entry, int64_t *base, int64_t n_blocks) {
    int64_t pos = 0, off = 0;
    while (pos >= 0 && pos < n_raw && off < events) {
        const int64_t b = pos / CHAIN_L;
        entry[b] = pos;
        base[b] = off;
        off += cnt[pos];
        pos = exit_pos[pos];
    }
}

__global__ void __launch_bounds__(128) emit_kernel(const int4 *parsed, const int64_t *entry, const int64_t *base,
                                                   int64_t n_blocks, int64_t n_raw, int64_t events, int32_t *out_u,
                                                   int32_t *out_i, int32_t *out_j, MtStatus *status) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    int64_t pos = entry[b];
    if (pos < 0) return;
    const int64_t end = ((b + 1) * CHAIN_L < n_raw) ? (b + 1) * CHAIN_L : n_raw;
    int64_t t = base[b];
    while (pos < end && t < events) {
        const int4 r = parsed[pos];
        if (r.w == INCOMPLETE) {
            if (r.x == -2) status->error = 1;
            // stream ran out before `events` triples: report how far we got
            atomicMin((unsigned long long *)&status->produced, (unsigned long long)t);
            return;
        }
        out_u[t] = r.x; out_i[t] = r.y; out_j[t] = r.z;
        pos += r.w;
        t++;
        if (t == events) status->consumed = pos;
    }
}

__global__ void init_chain_kernel(int64_t *entry, int64_t n_blocks, MtStatus *status, int64_t events) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n_blocks) entry[b] = -1;
    if (b == 0) { status->produced = events; status->consumed = -1; status->error = 0; status->pad = 0; }
}

struct SamplerLayout {
    size_t raw, parsed, exit_pos, cnt, entry, base, status, total;
    int64_t n_raw_max, n_blocks_max;
};

static SamplerLayout sampler_layout(int64_t events) {
    SamplerLayout L;
    L.n_raw_max = 8 * events + 16384;
    L.n_blocks_max = (L.n_raw_max + CHAIN_L - 1) / CHAIN_L;
    size_t off = 0;
    L.raw = off; off += align_up(sizeof(uint32_t) * (size_t)L.n_raw_max);
    L.parsed = off; off += align_up(sizeof(int4) * (size_t)L.n_raw_max);
    L.exit_pos = off; off += align_up(sizeof(int64_t) * (size_t)L.n_raw_max);
    L.cnt = off; off += align_up(sizeof(int32_t) * (size_t)L.n_raw_max);
    L.entry = off; off += align_up(sizeof(int64_t) * (size_t)L.n_blocks_max);
    L.base = off; off += align_up(sizeof(int64_t) * (size_t)L.n_blocks_max);
    L.status = off; off += align_up(sizeof(MtStatus));
    L.total = off;
    return L;
}


// ---------------------------------------------------------------- pointwise ratio sampler
// Replays dataset/samplers/pointwise_pos_neg_ratio_ratings_sampler.py (DMF, and FISM / NAIS later) on the same four
// steps.  Each sample draws u = randint(n_users), then np.random.shuffle of the list [0]*neg_ratio + [1] (legacy
// untyped path: for i = n-1 .. 1, j = random_interval(i) by masked rejection, swap), then a positive ui[randint(lui)]
// with its rating if list[0] == 1, else negatives randint(n_items) redrawn while they are train items.  The list's
// permutation carries from sample to sample, so the branch depends on the state s = position of the 1: the parse stores,
// per stream position, the shuffle's permutation pi (s -> pi(s), nibble-packed, n <= 16) and BOTH branch outcomes, and
// the chain is resolved over (position, state) pairs.
constexpr int PW_MAX_STATES = 16;

struct PwRec {
    int32_t u;         // -1: incomplete head; -2: the user owns every item or none (the reference never terminates)
    int32_t pos_item, pos_len;   // positive branch: item, draws from the sample's start (INCOMPLETE: ran out)
    int32_t neg_item, neg_len;   // negative branch
    float pos_r;
    uint64_t perm;     // nibble s holds pi(s)
};

struct PwStatus {
    int64_t produced, consumed;
    int32_t error, final_state;
};

struct PwParams {
    const uint32_t *raw;
    int64_t n_raw;
    int32_t n_users, n_items, n_states;
    const int64_t *indptr;
    const int32_t *set_indices, *sorted_indices;
    const float *set_ratings;
    PwRec *rec;
};

__global__ void __launch_bounds__(256) pw_parse_kernel(const PwParams p) {
    const int64_t pos = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pos >= p.n_raw) return;
    PwRec r{-1, -1, INCOMPLETE, -1, INCOMPLETE, 0.f, 0};
    int64_t q = pos;
    uint32_t u, v;
    const uint32_t rng_u = (uint32_t)(p.n_users - 1);
    if (!draw_bounded(p.raw, p.n_raw, q, rng_u, mask_for(rng_u), u)) { p.rec[pos] = r; return; }
    const int64_t beg = __ldg(p.indptr + u);
    const int lui = (int)(__ldg(p.indptr + u + 1) - beg);
    if (lui <= 0 || lui >= p.n_items) { r.u = -2; p.rec[pos] = r; return; }
    uint64_t arr = 0;                                   // arr nibble k: which incoming slot the list's slot k now holds
    for (int k = 0; k < p.n_states; k++) arr |= (uint64_t)k << (4 * k);
    for (int i = p.n_states - 1; i >= 1; i--) {
        if (!draw_bounded(p.raw, p.n_raw, q, (uint32_t)i, mask_for((uint32_t)i), v)) { p.rec[pos] = r; return; }
        const uint64_t a = (arr >> (4 * i)) & 15u, b = (arr >> (4 * v)) & 15u;
        arr &= ~((15ull << (4 * i)) | (15ull << (4 * v)));
        arr |= (b << (4 * i)) | (a << (4 * v));
    }
    uint64_t perm = 0;
    for (int k = 0; k < p.n_states; k++) perm |= (uint64_t)k << (4 * ((arr >> (4 * k)) & 15u));
    r.u = (int32_t)u;
    r.perm = perm;
    int64_t q1 = q;
    if (draw_bounded(p.raw, p.n_raw, q1, (uint32_t)(lui - 1), mask_for((uint32_t)(lui - 1)), v)) {
        r.pos_item = __ldg(p.set_indices + beg + v);
        r.pos_r = __ldg(p.set_ratings + beg + v);
        r.pos_len = (int32_t)(q1 - pos);
    }
    if (p.n_states > 1) {                               // neg_ratio = 0: the list is [1] and every sample is positive
        const uint32_t rng_i = (uint32_t)(p.n_items - 1), mask_i = mask_for(rng_i);
        const int32_t *row = p.sorted_indices + beg;
        int64_t q2 = q;
        while (draw_bounded(p.raw, p.n_raw, q2, rng_i, mask_i, v)) {
            if (!contains_sorted(row, lui, (int32_t)v)) {
                r.neg_item = (int32_t)v;
                r.neg_len = (int32_t)(q2 - pos);
                break;
            }
        }
    }
    p.rec[pos] = r;
}

__device__ __forceinline__ int pw_next_state(uint64_t perm, int s) { return (int)((perm >> (4 * s)) & 15u); }

// backward DP inside each block of CHAIN_L positions, one warp per block and one lane per list state: from (pos, s),
// the block's exit (position, state) and the number of samples up to it
__global__ void __launch_bounds__(128) pw_chain_block_kernel(const PwRec *rec, int64_t n_raw, int n_states,
                                                             int32_t *exit_pos, uint8_t *exit_st, int32_t *cnt) {
    const int64_t b = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int s = threadIdx.x & 31;
    const int64_t start = b * CHAIN_L;
    if (start >= n_raw) return;
    const int64_t end = (start + CHAIN_L < n_raw) ? start + CHAIN_L : n_raw;
    for (int64_t pos = end - 1; pos >= start; pos--) {
        if (s < n_states) {
            const PwRec r = rec[pos];
            const int64_t o = pos * n_states + s;
            int32_t len = INCOMPLETE;
            int ns = 0;
            if (r.u >= 0) {
                ns = pw_next_state(r.perm, s);
                len = ns == 0 ? r.pos_len : r.neg_len;
            }
            if (len == INCOMPLETE || len == 0) { exit_pos[o] = -1; exit_st[o] = 0; cnt[o] = 0; }  // 0: degenerate
            else if (pos + len >= end) { exit_pos[o] = (int32_t)(pos + len); exit_st[o] = (uint8_t)ns; cnt[o] = 1; }
            else {
                const int64_t on = (pos + len) * n_states + ns;
                exit_pos[o] = exit_pos[on]; exit_st[o] = exit_st[on]; cnt[o] = cnt[on] + 1;
            }
        }
        __syncwarp();
    }
}

__global__ void pw_chain_walk_kernel(const int32_t *exit_pos, const uint8_t *exit_st, const int32_t *cnt, int n_states,
                                     int64_t n_raw, int64_t events, const int32_t *list_pos, int64_t *entry,
                                     int32_t *entry_st, int64_t *base) {
    int64_t pos = 0, off = 0;
    int s = *list_pos;
    while (pos >= 0 && pos < n_raw && off < events) {
        const int64_t b = pos / CHAIN_L, o = pos * n_states + s;
        entry[b] = pos;
        entry_st[b] = s;
        base[b] = off;
        off += cnt[o];
        s = exit_st[o];
        pos = exit_pos[o];
    }
}

__global__ void __launch_bounds__(128) pw_emit_kernel(const PwRec *rec, const int64_t *entry, const int32_t *entry_st,
                                                      const int64_t *base, int64_t n_blocks, int64_t n_raw, int64_t events,
                                                      int32_t *out_u, int32_t *out_i, float *out_r, PwStatus *status) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    int64_t pos = entry[b];
    if (pos < 0) return;
    int s = entry_st[b];
    const int64_t end = ((b + 1) * CHAIN_L < n_raw) ? (b + 1) * CHAIN_L : n_raw;
    int64_t t = base[b];
    while (pos < end && t < events) {
        const PwRec r = rec[pos];
        const int ns = r.u >= 0 ? pw_next_state(r.perm, s) : 0;
        const int32_t len = r.u < 0 ? INCOMPLETE : (ns == 0 ? r.pos_len : r.neg_len);
        if (len == INCOMPLETE || len == 0) {
            if (r.u == -2) status->error = 1;
            atomicMin((unsigned long long *)&status->produced, (unsigned long long)t);
            return;
        }
        out_u[t] = r.u;
        out_i[t] = ns == 0 ? r.pos_item : r.neg_item;
        out_r[t] = ns == 0 ? r.pos_r : 0.f;
        pos += len;
        s = ns;
        t++;
        if (t == events) { status->consumed = pos; status->final_state = s; }
    }
}

__global__ void pw_init_kernel(int64_t *entry, int64_t n_blocks, PwStatus *status, int64_t events) {
    const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n_blocks) entry[b] = -1;
    if (b == 0) { status->produced = events; status->consumed = -1; status->error = 0; status->final_state = -1; }
}

struct PwLayout {
    size_t raw, rec, exit_pos, exit_st, cnt, entry, entry_st, base, status, total;
    int64_t n_raw_first, n_raw_max, n_blocks_max;
};

// Raw-draw budget: the expected draws of one sample are (mask(m-1) + 1) / m for each bounded draw over m values — the
// user, the n - 1 shuffle swaps — plus at most 2 for the positive and 2 / (1 - density) for a negative; the first attempt
// allows 1.25x that with 2.5 for the branch, the second twice as much.
static PwLayout pw_layout(int64_t events, int n_users, int n_states) {
    auto expect = [](uint32_t m) {            // draws per bounded draw over m >= 1 values
        uint32_t r = m - 1, k = r;
        k |= k >> 1; k |= k >> 2; k |= k >> 4; k |= k >> 8; k |= k >> 16;
        return r == 0 ? 0.0 : ((double)k + 1.0) / (double)m;
    };
    double per = expect((uint32_t)(n_users < 1 ? 1 : n_users)) + 2.5;
    for (int i = 1; i < n_states; i++) per += expect((uint32_t)i + 1);
    PwLayout L;
    L.n_raw_first = (int64_t)(1.25 * per * (double)events) + 8192;
    L.n_raw_max = 2 * L.n_raw_first;
    L.n_blocks_max = (L.n_raw_max + CHAIN_L - 1) / CHAIN_L;
    const size_t ns = (size_t)L.n_raw_max * n_states;
    size_t off = 0;
    L.raw = off; off += align_up(sizeof(uint32_t) * (size_t)L.n_raw_max);
    L.rec = off; off += align_up(sizeof(PwRec) * (size_t)L.n_raw_max);
    L.exit_pos = off; off += align_up(sizeof(int32_t) * ns);
    L.exit_st = off; off += align_up(ns);
    L.cnt = off; off += align_up(sizeof(int32_t) * ns);
    L.entry = off; off += align_up(sizeof(int64_t) * (size_t)L.n_blocks_max);
    L.entry_st = off; off += align_up(sizeof(int32_t) * (size_t)L.n_blocks_max);
    L.base = off; off += align_up(sizeof(int64_t) * (size_t)L.n_blocks_max);
    L.status = off; off += align_up(sizeof(PwStatus));
    L.total = off;
    return L;
}

}  // namespace eb

using namespace eb;

extern "C" int eb_mt_seed(uint32_t *state, uint32_t seed, void *stream) {
    EB_ARG(state, "null state");
    mt_seed_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state, seed);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_mt_raw(uint32_t *state, uint32_t *out, int64_t n, void *stream) {
    EB_ARG(state && out && n >= 0, "bad argument");
    if (n == 0) return EB_OK;
    mt_generate_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(state, out, n, nullptr, 1);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" size_t eb_mt_sampler_workspace_bytes(int64_t events) {
    return sampler_layout(events < 1 ? 1 : events).total;
}

extern "C" int eb_mt_sampler_step(uint32_t *state, int32_t n_users, int32_t n_items, const int64_t *indptr,
                                  const int32_t *set_indices, const int32_t *sorted_indices, int64_t events,
                                  int32_t *out_u, int32_t *out_i, int32_t *out_j, void *workspace,
                                  size_t workspace_bytes, void *stream) {
    EB_ARG(state && indptr && set_indices && sorted_indices && out_u && out_i && out_j, "null pointer");
    EB_ARG(n_users >= 1 && n_items >= 2 && events >= 0, "bad sizes");
    if (events == 0) return EB_OK;
    const SamplerLayout L = sampler_layout(events);
    if (!workspace || workspace_bytes < L.total)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace_bytes, L.total);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    uint32_t *raw = (uint32_t *)(ws + L.raw);
    int4 *parsed = (int4 *)(ws + L.parsed);
    int64_t *exit_pos = (int64_t *)(ws + L.exit_pos);
    int32_t *cnt = (int32_t *)(ws + L.cnt);
    int64_t *entry = (int64_t *)(ws + L.entry), *base = (int64_t *)(ws + L.base);
    MtStatus *status = (MtStatus *)(ws + L.status);

    int64_t n_raw = 4 * events + 8192;
    for (int attempt = 0; attempt < 2; attempt++) {
        if (n_raw > L.n_raw_max) n_raw = L.n_raw_max;
        const int64_t n_blocks = (n_raw + CHAIN_L - 1) / CHAIN_L;
        // 1. raw stream from the current state (state itself not advanced yet)
        mt_generate_kernel<<<1, 256, 0, st>>>(state, raw, n_raw, nullptr, 0);
        init_chain_kernel<<<(unsigned)((n_blocks + 255) / 256), 256, 0, st>>>(entry, n_blocks, status, events);
        // 2. speculative parse at every position
        ParseParams pp{raw, n_raw, n_users, n_items, indptr, set_indices, sorted_indices, parsed, status};
        mt_parse_kernel<<<(unsigned)((n_raw + 255) / 256), 256, 0, st>>>(pp);
        // 3. chain resolution
        chain_block_kernel<<<(unsigned)((n_blocks + 127) / 128), 128, 0, st>>>(parsed, n_raw, exit_pos, cnt);
        chain_walk_kernel<<<1, 1, 0, st>>>(exit_pos, cnt, n_raw, events, entry, base, n_blocks);
        // 4. emit
        emit_kernel<<<(unsigned)((n_blocks + 127) / 128), 128, 0, st>>>(parsed, entry, base, n_blocks, n_raw, events,
                                                                        out_u, out_i, out_j, status);
        EB_CUDA(cudaGetLastError());
        MtStatus h;
        EB_CUDA(cudaMemcpyAsync(&h, status, sizeof(h), cudaMemcpyDeviceToHost, st));
        EB_CUDA(cudaStreamSynchronize(st));
        if (h.error) return set_err(EB_ERR_DATA, "a sampled user has no train item or owns every item "
                                                 "(custom_sampler.py:35-41 never terminates)");
        if (h.consumed >= 0 && h.produced == events) {
            // advance the persistent state by exactly the consumed draws
            mt_generate_kernel<<<1, 256, 0, st>>>(state, nullptr, h.consumed, nullptr, 1);
            EB_CUDA(cudaGetLastError());
            return EB_OK;
        }
        if (n_raw == L.n_raw_max) break;
        n_raw = L.n_raw_max;
    }
    return set_err(EB_ERR_DATA, "sampler needed more than %lld raw draws for %lld triples (rejection rate too high)",
                   (long long)L.n_raw_max, (long long)events);
}

extern "C" size_t eb_mt_pointwise_ratio_workspace_bytes(int64_t events, int32_t n_users, int32_t neg_ratio) {
    if (neg_ratio < 0 || neg_ratio >= PW_MAX_STATES) return 0;
    return pw_layout(events < 1 ? 1 : events, n_users, neg_ratio + 1).total;
}

extern "C" int eb_mt_pointwise_ratio_step(uint32_t *state, int32_t *list_pos, int32_t n_users, int32_t n_items,
                                          const int64_t *indptr, const int32_t *set_indices, const float *set_ratings,
                                          const int32_t *sorted_indices, int32_t neg_ratio, int64_t events, int32_t *out_u,
                                          int32_t *out_i, float *out_r, void *workspace, size_t workspace_bytes,
                                          void *stream) {
    EB_ARG(state && list_pos && indptr && set_indices && set_ratings && sorted_indices && out_u && out_i && out_r,
           "null pointer");
    EB_ARG(n_users >= 1 && n_items >= 2 && events >= 0, "bad sizes");
    EB_ARG(neg_ratio >= 0 && neg_ratio < PW_MAX_STATES, "neg_ratio=%d must lie in [0, %d]", neg_ratio, PW_MAX_STATES - 1);
    if (events == 0) return EB_OK;
    const int n_states = neg_ratio + 1;
    const PwLayout L = pw_layout(events, n_users, n_states);
    EB_ARG(L.n_raw_max < INT32_MAX, "events=%lld need more raw draws than one call can index; call in windows",
           (long long)events);
    if (!workspace || workspace_bytes < L.total)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace_bytes, L.total);
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    uint32_t *raw = (uint32_t *)(ws + L.raw);
    PwRec *rec = (PwRec *)(ws + L.rec);
    int32_t *exit_pos = (int32_t *)(ws + L.exit_pos), *cnt = (int32_t *)(ws + L.cnt);
    uint8_t *exit_st = (uint8_t *)(ws + L.exit_st);
    int64_t *entry = (int64_t *)(ws + L.entry), *base = (int64_t *)(ws + L.base);
    int32_t *entry_st = (int32_t *)(ws + L.entry_st);
    PwStatus *status = (PwStatus *)(ws + L.status);

    int64_t n_raw = L.n_raw_first;
    for (int attempt = 0; attempt < 2; attempt++) {
        const int64_t n_blocks = (n_raw + CHAIN_L - 1) / CHAIN_L;
        mt_generate_kernel<<<1, 256, 0, st>>>(state, raw, n_raw, nullptr, 0);
        pw_init_kernel<<<(unsigned)((n_blocks + 255) / 256), 256, 0, st>>>(entry, n_blocks, status, events);
        PwParams pp{raw, n_raw, n_users, n_items, n_states, indptr, set_indices, sorted_indices, set_ratings, rec};
        pw_parse_kernel<<<(unsigned)((n_raw + 255) / 256), 256, 0, st>>>(pp);
        pw_chain_block_kernel<<<(unsigned)((n_blocks + 3) / 4), 128, 0, st>>>(rec, n_raw, n_states, exit_pos, exit_st, cnt);
        pw_chain_walk_kernel<<<1, 1, 0, st>>>(exit_pos, exit_st, cnt, n_states, n_raw, events, list_pos, entry, entry_st,
                                              base);
        pw_emit_kernel<<<(unsigned)((n_blocks + 127) / 128), 128, 0, st>>>(rec, entry, entry_st, base, n_blocks, n_raw,
                                                                            events, out_u, out_i, out_r, status);
        EB_CUDA(cudaGetLastError());
        PwStatus h;
        EB_CUDA(cudaMemcpyAsync(&h, status, sizeof(h), cudaMemcpyDeviceToHost, st));
        EB_CUDA(cudaStreamSynchronize(st));
        if (h.error) return set_err(EB_ERR_DATA, "a sampled user has no train item or owns every item "
                                                 "(the reference's negative draw never terminates)");
        if (h.consumed >= 0 && h.produced == events) {
            mt_generate_kernel<<<1, 256, 0, st>>>(state, nullptr, h.consumed, nullptr, 1);
            EB_CUDA(cudaGetLastError());
            EB_CUDA(cudaMemcpyAsync(list_pos, &status->final_state, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
            return EB_OK;
        }
        n_raw = L.n_raw_max;
    }
    return set_err(EB_ERR_DATA, "sampler needed more than %lld raw draws for %lld samples (rejection rate too high)",
                   (long long)L.n_raw_max, (long long)events);
}
