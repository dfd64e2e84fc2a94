// eval_metrics.cu — the reference's ranking, novelty, popularity-bias, coverage and diversity metrics of top-k lists on
// the device (elliot/evaluation/metrics: accuracy/{ndcg_rendle2020,mrr,map,mar,f1,AUC/lauc}, coverage, novelty/{EPC,EFD},
// bias/{arp,aplt,aclt,pop_reo,pop_rsp}, diversity/{gini_index,shannon_entropy}).
//
// Like eval.cu, the top-k index tensor never leaves HBM.  A row's list is its entries before the first -1 within the
// cutoff (n_u of them).  Four launches after a memset of the item counts:
//   1. per-user pass: a group of G lanes per row; each lane looks its items up in the user's item-sorted relevant row
//      (binary search) and in small per-item tables (popularity, long-tail flag, EPC/EFD novelties) and per-position
//      tables (discount, MAP tail H(k)-H(r), inverse binary IDCG by min(|rel|, k)).  Hit count, sum of hit positions,
//      first hit and the weighted sums are combined by shuffle trees; every listed item of a user with test rows does an
//      integer atomicAdd into the per-item counts.  Block sums use a fixed tree, then an ordered finishing pass.
//   2. per-item pass: a histogram of the non-zero item counts (how many items were recommended c times), integer atomics.
//   3. one block: ItemCoverage = number of recommended items, and the Gini rank sum S = sum_j j * cs_j over the counts in
//      ascending order, from the histogram with a block scan.  All integers: exact and order-free.
//   4. per-user pass for SEntropy: sum_u (1/n_u) sum_{i in L_u} -log2(c_i / free_norm), fixed tree + ordered finish.
// Integer atomics and integer histograms give the same bits whatever the scheduling; every fp64 sum has a fixed order.
#include "common.cuh"

namespace eb {

constexpr int EM_THREADS = 256;
// out[] slots; the first EM_NUSER are summed over rows by the per-user pass
enum : int {
    EM_NREL = 0,          // users with test rows and >= 1 relevant item (the set the accuracy/novelty metrics average over)
    EM_RENDLE, EM_MRR, EM_MAP, EM_MAR, EM_F1, EM_LAUC, EM_NUMRET, EM_EPC, EM_EFD,
    EM_REO_NUM_H, EM_REO_NUM_T, EM_REO_DEN_H, EM_REO_DEN_T,
    EM_NROWS,             // users with any test row
    EM_ARP, EM_APLT, EM_ACLT, EM_RSP_NUM_H, EM_RSP_NUM_T, EM_RSP_DEN_H, EM_RSP_DEN_T,
    EM_UCOV, EM_UCOV_N, EM_FREE_NORM, EM_EMPTY,
    EM_NUSER,             // = 26
    EM_ITEMCOV = EM_NUSER, EM_GINI_S, EM_SENTROPY,
    EM_NOUT               // = 29
};
constexpr int EM_PER_USER = 12;   // nDCGRendle2020 MRR MAP MAR F1 LAUC NumRetrieved EPC EFD | ARP APLT ACLT

template <int G>
__device__ __forceinline__ int group_min(int v) {
#pragma unroll
    for (int o = G / 2; o; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o, G));
    return v;
}
template <int G, typename T>
__device__ __forceinline__ T group_sum(T v) {
#pragma unroll
    for (int o = G / 2; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, G);
    return v;
}

// length of the row's list: position of the first -1 within the cutoff (all lanes of the group get it)
template <int G>
__device__ __forceinline__ int list_len(const int32_t *__restrict__ row, int k, int lane) {
    int first = k;
    for (int r = lane; r < k; r += G)
        if (row[r] < 0) { first = r; break; }
    return group_min<G>(first);
}

template <int N, int UPB>
__device__ __forceinline__ void block_tree(double (*acc)[UPB], double *__restrict__ partial) {
    __syncthreads();
    for (int s = UPB / 2; s; s >>= 1) {                       // fixed tree -> deterministic
        if ((int)threadIdx.x < s) {
#pragma unroll
            for (int m = 0; m < N; ++m) acc[m][threadIdx.x] += acc[m][threadIdx.x + s];
        }
        __syncthreads();
    }
    if ((int)threadIdx.x < N) partial[(int64_t)blockIdx.x * N + threadIdx.x] = acc[threadIdx.x][0];
}

template <int G>
__global__ void __launch_bounds__(EM_THREADS) eval_metrics_user_kernel(
    const int32_t *__restrict__ topk, int64_t n_rows, int ld, int k, const int32_t *__restrict__ users,
    const int64_t *__restrict__ indptr, const int32_t *__restrict__ rel_items, const int32_t *__restrict__ uinfo,
    const int32_t *__restrict__ pop, const uint8_t *__restrict__ long_tail, const double *__restrict__ nov, int n_items,
    const double *__restrict__ disc, const double *__restrict__ map_tail, const double *__restrict__ inv_idcg,
    int32_t *__restrict__ item_count, int32_t *__restrict__ list_len_out, double *__restrict__ per_user,
    double *__restrict__ partial) {
    constexpr int UPB = EM_THREADS / G;
    __shared__ double acc[EM_NUSER][UPB];
    const int g = threadIdx.x / G, lane = threadIdx.x % G;
    const int64_t row = (int64_t)blockIdx.x * UPB + g;
    const bool live = row < n_rows;
    const int64_t u = live ? (users ? (int64_t)users[row] : row) : 0;
    const int32_t *info = uinfo + u * 6;                      // has_rows, |train_u|, REO den SH/LT, RSP den SH/LT
    const bool in_a = live && info[0] != 0;                   // user with any test row
    const int64_t lo = in_a ? indptr[u] : 0, hi = in_a ? indptr[u + 1] : 0;
    const int64_t n_rel = hi - lo;
    const int32_t *lst = topk + (live ? row : 0) * (int64_t)ld;
    const int n_list = list_len<G>(lst, k, lane);             // every lane of the warp takes part in the shuffles
    const int n = in_a ? n_list : 0;

    // ACLT, APLT, PopREO and PopRSP count each listed item once (the reference takes set() of the list): `first`
    int hits = 0, first_hit = k, hits_sh = 0, hits_lt = 0, n_lt = 0, n_distinct = 0;
    long long sum_r = 0, sum_pop = 0;
    double dcg = 0, map = 0, epc = 0, efd = 0, norm = 0;
    for (int r = lane; r < n; r += G) {
        const int32_t it = lst[r];
        const double d = disc[r];
        const bool lt = long_tail[it] != 0;
        bool first = true;
        for (int j = 0; j < r && first; ++j) first = lst[j] != it;
        norm += d;
        sum_pop += pop[it];
        n_lt += lt && first;
        n_distinct += first;
        atomicAdd(item_count + it, 1);
        if (n_rel > 0) {
            int64_t a = lo, b = hi;
            while (a < b) {
                const int64_t m = (a + b) >> 1;
                if (rel_items[m] < it) a = m + 1; else b = m;
            }
            if (a < hi && rel_items[a] == it) {
                ++hits;
                sum_r += r;
                first_hit = min(first_hit, r);
                hits_sh += !lt && first;
                hits_lt += lt && first;
                dcg += d;
                map += map_tail[r];
                epc += d * nov[2 * (int64_t)it];
                efd += d * nov[2 * (int64_t)it + 1];
            }
        }
    }
    // all 32 lanes shuffle (groups of one warp may belong to users in different sets)
    hits = group_sum<G>(hits); hits_sh = group_sum<G>(hits_sh); hits_lt = group_sum<G>(hits_lt); n_lt = group_sum<G>(n_lt);
    n_distinct = group_sum<G>(n_distinct);
    first_hit = group_min<G>(first_hit);
    sum_r = group_sum<G>(sum_r); sum_pop = group_sum<G>(sum_pop);
    dcg = group_sum<G>(dcg); map = group_sum<G>(map); epc = group_sum<G>(epc); efd = group_sum<G>(efd);
    norm = group_sum<G>(norm);

    double v[EM_NUSER];
#pragma unroll
    for (int m = 0; m < EM_NUSER; ++m) v[m] = 0;
    if (n_rel > 0) {
        const int m_rel = n_rel < k ? (int)n_rel : k;
        const double p = (double)hits / (double)k, rc = (double)hits / (double)n_rel;
        const double den = p + rc;
        const long long neg = (long long)n_items - info[1] - n_rel + 1;
        v[EM_NREL] = 1;
        v[EM_RENDLE] = inv_idcg[m_rel] * dcg;
        v[EM_MRR] = hits ? 1.0 / (double)(first_hit + 1) : 0.0;
        v[EM_MAP] = map / (double)k;
        v[EM_MAR] = (double)((long long)hits * k - sum_r) / (double)n_rel / (double)k;
        v[EM_F1] = den != 0 ? 2.0 * p * rc / den : 0.0;
        v[EM_LAUC] = (double)((long long)hits * neg - sum_r + (long long)hits * (hits - 1) / 2) / (double)neg / (double)m_rel;
        v[EM_NUMRET] = n;
        v[EM_EPC] = norm > 0 ? epc / norm : 0.0;
        v[EM_EFD] = norm > 0 ? efd / norm : 0.0;
        v[EM_REO_NUM_H] = hits_sh;
        v[EM_REO_NUM_T] = hits_lt;
        v[EM_REO_DEN_H] = info[2];
        v[EM_REO_DEN_T] = info[3];
    }
    if (in_a) {
        v[EM_NROWS] = 1;
        v[EM_ARP] = n ? (double)sum_pop / (double)n : 0.0;   // an empty list is counted in EM_EMPTY; the caller raises
        v[EM_APLT] = n ? (double)n_lt / (double)n : 0.0;
        v[EM_ACLT] = n_lt;
        v[EM_RSP_NUM_H] = n_distinct - n_lt;
        v[EM_RSP_NUM_T] = n_lt;
        v[EM_RSP_DEN_H] = info[4];
        v[EM_RSP_DEN_T] = info[5];
        v[EM_UCOV] = n > 0;
        v[EM_UCOV_N] = n >= k;
        v[EM_FREE_NORM] = n;
        v[EM_EMPTY] = n == 0;
    }
    if (live && lane == 0) {
        list_len_out[row] = in_a ? n : 0;
        if (per_user) {
            double *o = per_user + row * EM_PER_USER;
            const double nan = __longlong_as_double(0x7ff8000000000000LL);
            const int src[EM_PER_USER] = {EM_RENDLE, EM_MRR, EM_MAP, EM_MAR, EM_F1, EM_LAUC, EM_NUMRET, EM_EPC, EM_EFD,
                                          EM_ARP, EM_APLT, EM_ACLT};
#pragma unroll
            for (int j = 0; j < 9; ++j) o[j] = n_rel > 0 ? v[src[j]] : nan;
            o[9] = in_a && n ? v[EM_ARP] : nan;
            o[10] = in_a && n ? v[EM_APLT] : nan;
            o[11] = in_a ? v[EM_ACLT] : nan;
        }
    }
    if (lane == 0) {
#pragma unroll
        for (int m = 0; m < EM_NUSER; ++m) acc[m][g] = v[m];
    }
    block_tree<EM_NUSER, UPB>(acc, partial);
}

// ordered second pass: one warp per output, lanes stride the partials, fixed shuffle tree
__global__ void eval_metrics_finish_kernel(const double *__restrict__ partial, int64_t n_blocks, int n_out,
                                           double *__restrict__ out) {
    const int m = threadIdx.x / 32, lane = threadIdx.x % 32;
    double s = 0;
    for (int64_t b = lane; b < n_blocks; b += 32) s += partial[b * n_out + m];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[m] = s;
}

// hist[c] = number of items recommended exactly c times (c >= 1)
__global__ void eval_metrics_hist_kernel(const int32_t *__restrict__ item_count, int n_items, int64_t max_count,
                                         int32_t *__restrict__ hist) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t c = item_count[i];
        if (c > 0) atomicAdd(hist + (c < max_count ? c : max_count), 1);
    }
}

// One block.  With the counts in ascending order, the items recommended c times hold ranks [R_c, R_c + m_c), where
// R_c = sum_{c' < c} m_c', so they add c * (m_c R_c + m_c (m_c - 1) / 2) to S = sum_j j * cs_j.
constexpr int GINI_THREADS = 1024;
__global__ void __launch_bounds__(GINI_THREADS) eval_metrics_gini_kernel(const int32_t *__restrict__ hist, int64_t max_count,
                                                                         double *__restrict__ out) {
    __shared__ long long part[GINI_THREADS];
    __shared__ unsigned long long s_sum, s_items;
    const int t = threadIdx.x;
    const int64_t len = max_count + 1;
    const int64_t chunk = (len + GINI_THREADS - 1) / GINI_THREADS;
    const int64_t a = t * chunk < len ? t * chunk : len, b = a + chunk < len ? a + chunk : len;
    long long items = 0;
    for (int64_t c = a; c < b; ++c) items += hist[c];
    part[t] = items;
    if (t == 0) { s_sum = 0; s_items = 0; }
    __syncthreads();
    if (t == 0) {                                             // exclusive scan of the chunk totals (integers)
        long long run = 0;
        for (int j = 0; j < GINI_THREADS; ++j) { const long long x = part[j]; part[j] = run; run += x; }
        s_items = (unsigned long long)run;
    }
    __syncthreads();
    long long rank = part[t], s = 0;
    for (int64_t c = a; c < b; ++c) {
        const long long m = hist[c];
        s += c * (m * rank + m * (m - 1) / 2);
        rank += m;
    }
    atomicAdd(&s_sum, (unsigned long long)s);                 // integer: order-free
    __syncthreads();
    if (t == 0) {
        out[EM_ITEMCOV] = (double)s_items;
        out[EM_GINI_S] = (double)s_sum;
    }
}

template <int G>
__global__ void __launch_bounds__(EM_THREADS) eval_metrics_entropy_kernel(
    const int32_t *__restrict__ topk, int64_t n_rows, int ld, const int32_t *__restrict__ list_len,
    const int32_t *__restrict__ item_count, const double *__restrict__ out, double *__restrict__ partial) {
    constexpr int UPB = EM_THREADS / G;
    __shared__ double acc[1][UPB];
    const int g = threadIdx.x / G, lane = threadIdx.x % G;
    const int64_t row = (int64_t)blockIdx.x * UPB + g;
    const int n = row < n_rows ? list_len[row] : 0;
    const double free_norm = out[EM_FREE_NORM], ln2 = log(2.0);
    double s = 0;
    for (int r = lane; r < n; r += G) s += -log((double)item_count[topk[row * ld + r]] / free_norm) / ln2;
    s = group_sum<G>(s);
    if (lane == 0) acc[0][g] = n ? s / (double)n : 0.0;
    block_tree<1, UPB>(acc, partial);
}

static int em_group(int k) { return k <= 8 ? 8 : (k <= 16 ? 16 : 32); }

struct EmLayout {
    size_t partial, partial2, list_len, counts, hist, total;
};
static EmLayout em_layout(int64_t n_rows, int k, int n_items) {
    const int64_t blocks = (n_rows + EM_THREADS / em_group(k) - 1) / (EM_THREADS / em_group(k));
    auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
    EmLayout l;
    l.partial = 0;
    l.partial2 = up(l.partial + (size_t)blocks * EM_NUSER * sizeof(double));
    l.list_len = up(l.partial2 + (size_t)blocks * sizeof(double));
    l.counts = up(l.list_len + (size_t)n_rows * sizeof(int32_t));
    l.hist = l.counts + (size_t)n_items * sizeof(int32_t);          // counts and hist are zeroed by one memset
    l.total = up(l.hist + (size_t)(n_rows + 1) * sizeof(int32_t));
    return l;
}

}  // namespace eb

extern "C" size_t eb_eval_metrics_workspace_bytes(int64_t n_rows, int k, int n_items) {
    if (n_rows < 0 || k < 1 || n_items < 0) return 0;
    return eb::em_layout(n_rows, k, n_items).total;
}

extern "C" int eb_eval_metrics_f64(const int32_t *topk_idx, int64_t n_rows, int ld, int k, const int32_t *users,
                                   const int64_t *rel_indptr, const int32_t *rel_items, const int32_t *user_info,
                                   const int32_t *item_pop, const uint8_t *item_long_tail, const double *item_novelty,
                                   int n_items, const double *discount, const double *map_tail,
                                   const double *inv_binary_idcg, double *per_user, double *out, void *workspace,
                                   size_t workspace_bytes, void *stream) {
    using namespace eb;
    EB_ARG(out, "null output pointer");
    EB_ARG(n_rows >= 0 && k >= 1 && k <= 1024 && ld >= k && n_items >= 0, "bad shape (n_rows=%lld k=%d ld=%d n_items=%d)",
           (long long)n_rows, k, ld, n_items);
    cudaStream_t st = (cudaStream_t)stream;
    if (n_rows == 0) {                                          // empty list set: nothing evaluated
        EB_CUDA(cudaMemsetAsync(out, 0, EM_NOUT * sizeof(double), st));
        return EB_OK;
    }
    EB_ARG(topk_idx && rel_indptr && rel_items && user_info && item_pop && item_long_tail && item_novelty && discount &&
           map_tail && inv_binary_idcg, "null pointer");
    const EmLayout l = em_layout(n_rows, k, n_items);
    if (workspace_bytes < l.total || !workspace)
        return set_err(EB_ERR_WORKSPACE, "eval metrics workspace too small: need %zu bytes", l.total);
    const int G = em_group(k);
    const int upb = EM_THREADS / G;
    const int64_t blocks = (n_rows + upb - 1) / upb;
    EB_ARG(blocks <= 0x7fffffffLL, "too many rows for one launch");
    char *ws = (char *)workspace;
    double *partial = (double *)(ws + l.partial), *partial2 = (double *)(ws + l.partial2);
    int32_t *lens = (int32_t *)(ws + l.list_len), *counts = (int32_t *)(ws + l.counts), *hist = (int32_t *)(ws + l.hist);
    EB_CUDA(cudaMemsetAsync(counts, 0, l.total - l.counts, st));
#define EB_LAUNCH(GV)                                                                                                     \
    eval_metrics_user_kernel<GV><<<(unsigned)blocks, EM_THREADS, 0, st>>>(                                               \
        topk_idx, n_rows, ld, k, users, rel_indptr, rel_items, user_info, item_pop, item_long_tail, item_novelty, n_items, \
        discount, map_tail, inv_binary_idcg, counts, lens, per_user, partial)
    if (G == 8) EB_LAUNCH(8); else if (G == 16) EB_LAUNCH(16); else EB_LAUNCH(32);
#undef EB_LAUNCH
    EB_CUDA(cudaGetLastError());
    eval_metrics_finish_kernel<<<1, 32 * EM_NUSER, 0, st>>>(partial, blocks, EM_NUSER, out);
    EB_CUDA(cudaGetLastError());
    if (n_items > 0) {
        const int hb = n_items > 256 * 1024 ? 1024 : (n_items + 255) / 256;
        eval_metrics_hist_kernel<<<hb, 256, 0, st>>>(counts, n_items, n_rows, hist);
        EB_CUDA(cudaGetLastError());
    }
    eval_metrics_gini_kernel<<<1, GINI_THREADS, 0, st>>>(hist, n_rows, out);
    EB_CUDA(cudaGetLastError());
#define EB_LAUNCH(GV) \
    eval_metrics_entropy_kernel<GV><<<(unsigned)blocks, EM_THREADS, 0, st>>>(topk_idx, n_rows, ld, lens, counts, out, partial2)
    if (G == 8) EB_LAUNCH(8); else if (G == 16) EB_LAUNCH(16); else EB_LAUNCH(32);
#undef EB_LAUNCH
    EB_CUDA(cudaGetLastError());
    eval_metrics_finish_kernel<<<1, 32, 0, st>>>(partial2, blocks, 1, out + EM_SENTROPY);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
