// bpr_sampler.cuh — the counter-based BPR sampler (custom_sampler.py:31-42 distribution, Philox stream): triple t of a call
// is drawn from Philox blocks keyed by seed with counter first + t, so any kernel can draw any triple in any order.
#pragma once
#include "common.cuh"

namespace eb {

struct SamplerParams {
    int32_t n_users, n_items;
    const int64_t *indptr;
    const int32_t *indices;
    uint64_t seed, first;
    // optional per-user membership signatures (eb_bloom_build): filter_log2bits bits per user
    const uint32_t *filter;
    int filter_log2bits;
};

// u of triple t: uniform over the users that own at least one and not every item.  r keeps the Philox block that drew the
// accepted u (its other words pick i and j), beg / len the user's CSR row.
__device__ __forceinline__ void sample_user(const SamplerParams &p, int64_t t, uint32_t (&r)[4], int &u, int64_t &beg, int &len) {
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
__device__ __forceinline__ void sample_triple(const SamplerParams &p, int64_t t, int &u, int &i, int &j) {
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

static inline int set_filter(SamplerParams &p, const uint32_t *filter, int filter_words) {
    if (!filter) return EB_OK;
    EB_ARG(filter_words >= 1 && filter_words <= 1024 && (filter_words & (filter_words - 1)) == 0,
           "filter_words must be a power of two in [1, 1024] (got %d)", filter_words);
    int lb = 5;
    while ((1 << (lb - 5)) < filter_words) lb++;
    p.filter = filter; p.filter_log2bits = lb;
    return EB_OK;
}

// the sampler arguments of an entry point, checked (n_users >= 1, n_items >= 2, non-null CSR)
static inline int sampler_params(SamplerParams &p, int32_t n_users, int32_t n_items, const int64_t *indptr, const int32_t *indices,
                                 const uint32_t *filter, int filter_words, uint64_t seed, uint64_t first) {
    EB_ARG(n_users > 0 && n_items > 1, "bad sizes (n_users=%d, n_items=%d)", n_users, n_items);
    EB_ARG(indptr && indices, "null CSR");
    p = SamplerParams{n_users, n_items, indptr, indices, seed, first, nullptr, 0};
    return set_filter(p, filter, filter_words);
}

}  // namespace eb
