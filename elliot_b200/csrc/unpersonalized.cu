// unpersonalized.cu — the reference's MostPop and Random lists (recommender/unpersonalized/).
//
// MostPop: pop[i] = train users of item i (integer atomics: reruns give the same counts), one global order (pop desc,
// item asc; the host sorts the n_items keys), and per user the first k entries of that order outside the user's train
// row: one warp per user walks the order 32 entries at a time, tests them by binary search in the sorted row, and places
// the accepted ones with a ballot and a popc prefix.
//
// Random: the reference draws, per user in private order, local_k = min(k, n_u) values r = np.random.randint(n_u)
// (n_u = items outside the train row) from one legacy MT19937 stream, and lists the r-th such item.  The stream words
// come from mt_sampler.cu's generator; one warp walks them in user order (the masked rejection of randint makes every
// user's start depend on every earlier user's draws, so this walk is serial by construction), and a data-parallel pass
// maps each r to its item.
#include "common.cuh"

namespace eb {

// the smallest 2^b - 1 >= v (numpy's mask for randint's masked rejection)
__device__ __forceinline__ uint32_t rand_mask(uint32_t v) {
    v |= v >> 1; v |= v >> 2; v |= v >> 4; v |= v >> 8; v |= v >> 16;
    return v;
}

__global__ void item_pop_kernel(const int32_t *__restrict__ indices, int64_t nnz, int32_t *__restrict__ pop) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x)
        atomicAdd(pop + __ldg(indices + e), 1);
}

constexpr int MP_WARPS = 8;

__global__ void __launch_bounds__(MP_WARPS * 32) mostpop_lists_kernel(
    const int32_t *__restrict__ order, const int32_t *__restrict__ pop, int32_t n_items, const int64_t *__restrict__ indptr,
    const int32_t *__restrict__ train, const int32_t *__restrict__ users, int32_t user_begin, int64_t n_sel, int k,
    int32_t *__restrict__ out_idx, int32_t *__restrict__ out_val, int32_t *__restrict__ skipped) {
    const int lane = threadIdx.x & 31;
    for (int64_t q = (int64_t)blockIdx.x * MP_WARPS + threadIdx.x / 32; q < n_sel; q += (int64_t)gridDim.x * MP_WARPS) {
        const int64_t u = users ? (int64_t)__ldg(users + q) : (int64_t)user_begin + q;
        const int64_t a = __ldg(indptr + u);
        const int len = (int)(__ldg(indptr + u + 1) - a);
        int32_t *oi = out_idx + q * k, *ov = out_val + q * k;
        int cur = 0;
        if ((int64_t)len + k >= n_items) {
            // most_popular.py: `if lui + k >= n_items: r[u] = []` -- no list; the host rebuilds the reference's dict
            if (lane == 0) atomicAdd(skipped, 1);
        } else {
            for (int base = 0; base < n_items && cur < k; base += 32) {
                const int p = base + lane;
                const int32_t it = p < n_items ? __ldg(order + p) : -1;
                const bool ok = it >= 0 && !contains_sorted(train + a, len, it);
                const uint32_t b = __ballot_sync(0xffffffffu, ok);
                const int slot = cur + __popc(b & ((1u << lane) - 1u));
                if (ok && slot < k) { oi[slot] = it; ov[slot] = __ldg(pop + it); }
                cur += __popc(b);
            }
        }
        for (int j = (cur < k ? cur : k) + lane; j < k; j += 32) { oi[j] = -1; ov[j] = 0; }
    }
}

// where the walk of the stream stands: the next word, the words available, and the user / slot it resumes at
struct RandWalk {
    int64_t pos, avail;
    int32_t user, filled;
};

// One warp.  For each user from st->user on: n_u = n_items - |train_u|, local_k = min(k, n_u); n_u <= 1 draws nothing
// (randint(1) = 0 consumes no word); otherwise values w & mask are accepted when <= n_u - 1, 32 words per step, and the
// first (local_k - filled) accepted ones are kept.  Slots past local_k get -1.  Returns early when the words run out.
__global__ void __launch_bounds__(32) random_walk_kernel(const uint32_t *__restrict__ words, RandWalk *st, int32_t n_users,
                                                        int32_t n_items, const int64_t *__restrict__ indptr, int k,
                                                        int32_t *__restrict__ r_out) {
    const int lane = threadIdx.x;
    int64_t pos = st->pos;
    const int64_t avail = st->avail;
    int filled = st->filled;
    int u = st->user;
    for (; u < n_users; u++, filled = 0) {
        const int n_u = n_items - (int)(__ldg(indptr + u + 1) - __ldg(indptr + u));
        const int lk = n_u < k ? (n_u > 0 ? n_u : 0) : k;
        int32_t *row = r_out + (int64_t)u * k;
        if (n_u <= 1) {
            if (lk == 1 && lane == 0) row[0] = 0;
        } else {
            const uint32_t rng = (uint32_t)(n_u - 1), mask = rand_mask(rng);
            while (filled < lk) {
                if (pos >= avail) break;
                const bool in = pos + lane < avail;
                const uint32_t v = in ? __ldg(words + pos + lane) & mask : 0xffffffffu;
                const bool ok = in && v <= rng;
                const uint32_t b = __ballot_sync(0xffffffffu, ok);
                const int rank = __popc(b & ((1u << lane) - 1u));
                const int need = lk - filled, got = __popc(b);
                if (ok && rank < need) row[filled + rank] = (int32_t)v;
                if (got >= need) {
                    // consumed through the need-th accepted word
                    const uint32_t last = __ballot_sync(0xffffffffu, ok && rank == need - 1);
                    pos += __ffs(last);
                    filled = lk;
                } else {
                    pos = pos + 32 < avail ? pos + 32 : avail;
                    filled += got;
                }
            }
            if (filled < lk) break;
        }
        for (int j = lk + lane; j < k; j += 32) row[j] = -1;
    }
    __syncwarp();
    if (lane == 0) { st->pos = pos; st->user = u; st->filled = u < n_users ? filled : 0; }
}

// out[q][j] = the r-th item outside user u's sorted train row t (r = r_in[u][j]): r + #{m : t_m - m <= r}
__global__ void complement_select_kernel(const int32_t *__restrict__ r_in, const int64_t *__restrict__ indptr,
                                         const int32_t *__restrict__ train, const int32_t *__restrict__ users,
                                         int32_t user_begin, int64_t n_sel, int k, int32_t *__restrict__ out) {
    const int64_t total = n_sel * k;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t q = t / k;
        const int j = (int)(t - q * k);
        const int64_t u = users ? (int64_t)__ldg(users + q) : (int64_t)user_begin + q;
        const int32_t r = __ldg(r_in + u * k + j);
        if (r < 0) { out[t] = -1; continue; }
        const int64_t a = __ldg(indptr + u);
        int lo = 0, hi = (int)(__ldg(indptr + u + 1) - a);
        while (lo < hi) {                                         // t_m - m is non-decreasing in m
            const int m = (lo + hi) >> 1;
            if (__ldg(train + a + m) - m <= r) lo = m + 1; else hi = m;
        }
        out[t] = r + lo;
    }
}

}  // namespace eb

using namespace eb;

extern "C" int eb_item_pop(const int32_t *indices, int64_t nnz, int32_t n_items, int32_t *pop, void *stream) {
    EB_ARG(pop && (indices || nnz == 0), "null pointer");
    EB_ARG(nnz >= 0 && n_items >= 1, "bad sizes nnz=%lld n_items=%d", (long long)nnz, n_items);
    cudaStream_t st = (cudaStream_t)stream;
    EB_CUDA(cudaMemsetAsync(pop, 0, sizeof(int32_t) * (size_t)n_items, st));
    if (nnz == 0) return EB_OK;
    item_pop_kernel<<<capped_grid(nnz), 256, 0, st>>>(indices, nnz, pop);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_mostpop_topk(const int32_t *order, const int32_t *pop, int32_t n_items, const int64_t *indptr,
                               const int32_t *train, const int32_t *users, int32_t user_begin, int64_t n_sel, int k,
                               int32_t *out_idx, int32_t *out_val, int32_t *skipped, void *stream) {
    EB_ARG(order && pop && indptr && train && out_idx && out_val && skipped, "null pointer");
    EB_ARG(n_items >= 1 && n_sel >= 0 && user_begin >= 0 && k >= 1, "bad sizes n_items=%d n_sel=%lld k=%d", n_items,
           (long long)n_sel, k);
    cudaStream_t st = (cudaStream_t)stream;
    EB_CUDA(cudaMemsetAsync(skipped, 0, sizeof(int32_t), st));
    if (n_sel == 0) return EB_OK;
    int64_t grid = (n_sel + MP_WARPS - 1) / MP_WARPS;
    const int64_t cap = (int64_t)sm_count() * 8;
    if (grid > cap) grid = cap;
    mostpop_lists_kernel<<<(unsigned)grid, MP_WARPS * 32, 0, st>>>(order, pop, n_items, indptr, train, users, user_begin,
                                                                   n_sel, k, out_idx, out_val, skipped);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" size_t eb_random_workspace_bytes(void) { return align_up(sizeof(RandWalk)); }

extern "C" int eb_random_draws(uint32_t *state, uint32_t *words, int64_t capacity, int64_t *pos_host, int32_t n_users,
                               int32_t n_items, const int64_t *indptr, int k, int32_t *r_out, int64_t *consumed_host,
                               void *workspace, size_t workspace_bytes, void *stream) {
    EB_ARG(state && words && pos_host && indptr && r_out && consumed_host, "null pointer");
    EB_ARG(capacity >= 1 && n_users >= 0 && n_items >= 1 && k >= 1, "bad sizes capacity=%lld n_users=%d n_items=%d k=%d",
           (long long)capacity, n_users, n_items, k);
    EB_ARG(pos_host[0] >= 0 && pos_host[0] <= pos_host[1] && pos_host[1] <= capacity, "bad stream position");
    if (!workspace || workspace_bytes < sizeof(RandWalk))
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace_bytes, sizeof(RandWalk));
    cudaStream_t st = (cudaStream_t)stream;
    RandWalk *w = (RandWalk *)workspace;
    RandWalk h{pos_host[0], pos_host[1], 0, 0};
    *consumed_host = 0;
    for (;;) {
        EB_CUDA(cudaMemcpyAsync(w, &h, sizeof(h), cudaMemcpyHostToDevice, st));
        random_walk_kernel<<<1, 32, 0, st>>>(words, w, n_users, n_items, indptr, k, r_out);
        EB_CUDA(cudaGetLastError());
        const int64_t pos0 = h.pos;
        EB_CUDA(cudaMemcpyAsync(&h, w, sizeof(h), cudaMemcpyDeviceToHost, st));
        EB_CUDA(cudaStreamSynchronize(st));
        *consumed_host += h.pos - pos0;
        if (h.user >= n_users) break;
        // the buffer is used up: refill it with the next `capacity` words of the stream and resume
        const int rc = eb_mt_raw(state, words, capacity, stream);
        if (rc != EB_OK) return rc;
        h.pos = 0;
        h.avail = capacity;
    }
    pos_host[0] = h.pos;
    pos_host[1] = h.avail;
    return EB_OK;
}

extern "C" int eb_complement_select(const int32_t *r_in, const int64_t *indptr, const int32_t *train, const int32_t *users,
                                    int32_t user_begin, int64_t n_sel, int k, int32_t *out, void *stream) {
    EB_ARG(r_in && indptr && train && out, "null pointer");
    EB_ARG(n_sel >= 0 && user_begin >= 0 && k >= 1, "bad sizes n_sel=%lld k=%d", (long long)n_sel, k);
    if (n_sel == 0) return EB_OK;
    complement_select_kernel<<<capped_grid(n_sel * k), 256, 0, (cudaStream_t)stream>>>(r_in, indptr, train, users,
                                                                                       user_begin, n_sel, k, out);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
