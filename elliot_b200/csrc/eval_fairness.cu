// eval_fairness.cu — the reference's clustered fairness metrics of top-k lists on the device (elliot/evaluation/metrics/
// fairness: BiasDisparity/{BiasDisparityBR,BiasDisparityBD}, MAD/{User,Item}MAD{rating,ranking}, reo, rsp).  Users and
// items are grouped by a clustering file; the host turns the counts and sums below into the metrics (fairness.py).
//
// Like eval_metrics.cu, the top-k index tensor never leaves HBM.  A row's list is its entries before the first -1 within
// the cutoff.  A = the row's user has test rows, B = A and >= 1 relevant item.  Launches after one memset:
//   1. per-row pass, a group of G lanes per row (G as eb_eval_topk_f64 picks it):
//      - the row's nDCG, summed exactly as eb_eval_topk_f64 sums it (same lanes, same shuffle tree: the same bits), and
//        the mean of its scores (NaN for an empty list, as np.average([]));
//      - integer histograms: (user cluster, item cluster) entries of A rows (BiasDisparityBR), distinct listed items per
//        item cluster (RSP over A rows; REO over B rows, relevant items only), in shared memory when they fit;
//      - for B rows, one (item, entry) key per listed entry, its gain and its score when relevant, and the item's count.
//   2. a stable radix sort of the entries by item, so each item's entries stay in row order, then position order;
//   3. per item, the sequential sums of its entries' gains and relevant scores (the reference's dict walk order), / count;
//   4. stable sorts of the items by item cluster and of the rows by user cluster, and one warp per cluster summing its
//      values in that order with a fixed shuffle tree.
// Integer atomics give the same counts whatever the scheduling and every fp64 sum has a fixed order: reruns are
// bit-identical.  There is no cap on the number of clusters.
#include <cub/cub.cuh>

#include "common.cuh"

namespace eb {

constexpr int EF_THREADS = 256;
constexpr int EF_SHARED_BINS = 1024;   // BR + REO + RSP histograms of up to this many bins are kept in shared memory

static int ef_group(int k) { return k <= 8 ? 8 : (k <= 16 ? 16 : 32); }   // = eb_eval_topk_f64's grouping

template <int G>
__global__ void __launch_bounds__(EF_THREADS) fairness_row_kernel(
    const int32_t *__restrict__ topk, const double *__restrict__ scores, int64_t n_rows, int ld, int k,
    const int32_t *__restrict__ users, const int64_t *__restrict__ indptr, const int32_t *__restrict__ rel_items,
    const double *__restrict__ gains, const double *__restrict__ idcg, const double *__restrict__ disc,
    const uint8_t *__restrict__ has_rows, const int32_t *__restrict__ ucl, int nu, const int32_t *__restrict__ icl, int ni,
    int n_items, unsigned long long *__restrict__ hist_g,   // [nu*ni BR][ni REO][ni RSP] in the output counts
    int32_t *__restrict__ ukey, int32_t *__restrict__ urow, double *__restrict__ row_ndcg, double *__restrict__ row_mean,
    int32_t *__restrict__ ucount, int32_t *__restrict__ ekey, int32_t *__restrict__ eidx, double *__restrict__ egain,
    double *__restrict__ escore, int32_t *__restrict__ item_count) {
    constexpr int UPB = EF_THREADS / G;
    __shared__ unsigned int hist_s[EF_SHARED_BINS];
    const int n_bins = nu * ni + 2 * ni;
    const bool in_shared = n_bins <= EF_SHARED_BINS;
    if (in_shared)
        for (int b = threadIdx.x; b < n_bins; b += EF_THREADS) hist_s[b] = 0;
    __syncthreads();
    const int g = threadIdx.x / G, lane = threadIdx.x % G;
    const int64_t row = (int64_t)blockIdx.x * UPB + g;
    const bool live = row < n_rows;
    const int64_t u = live ? (users ? (int64_t)users[row] : row) : 0;
    const bool in_a = live && has_rows[u] != 0;
    const int64_t lo = in_a ? indptr[u] : 0, hi = in_a ? indptr[u + 1] : 0;
    const bool in_b = hi > lo;
    const int gu = in_a ? ucl[u] : -1;
    const int32_t *lst = topk + (live ? row : 0) * (int64_t)ld;
    int first = k;                                            // list length: the first -1 within the cutoff
    for (int r = lane; r < k; r += G)
        if (lst[r] < 0) { first = r; break; }
#pragma unroll
    for (int o = G / 2; o; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o, G));
    const int n = live ? first : 0;

    double dcg = 0, ssum = 0;
    for (int r = lane; r < k; r += G) {
        const int64_t e = row * k + r;
        const int32_t it = r < n ? lst[r] : -1;
        bool rel = false;
        double gain = 0;
        if (it >= 0 && in_b) {
            int64_t a = lo, b = hi;
            while (a < b) {
                const int64_t m = (a + b) >> 1;
                if (rel_items[m] < it) a = m + 1; else b = m;
            }
            if (a < hi && rel_items[a] == it) { rel = true; gain = gains[a]; }
        }
        if (it >= 0 && in_a) {
            const double s = scores ? scores[row * (int64_t)ld + r] : 0.0;
            if (in_b) {
                dcg += gain * disc[r];
                ssum += s;
            }
            const int ci = icl[it];
            bool distinct = true;                             // the reference takes set() of the list for REO / RSP
            for (int j = 0; j < r && distinct; ++j) distinct = lst[j] != it;
            int bins[3], nb = 0;
            if (gu >= 0 && ci >= 0) bins[nb++] = gu * ni + ci;
            if (distinct && ci >= 0) {
                bins[nb++] = nu * ni + ni + ci;
                if (in_b && rel) bins[nb++] = nu * ni + ci;
            }
            for (int q = 0; q < nb; ++q) {
                if (in_shared) atomicAdd(hist_s + bins[q], 1u);
                else atomicAdd(hist_g + bins[q], 1ull);
            }
            if (in_b) {
                atomicAdd(item_count + it, 1);
                egain[e] = gain;
                escore[e] = rel ? s : 0.0;
            }
        }
        if (live) {
            ekey[e] = it >= 0 && in_b ? it : n_items;         // the sentinel sorts after every item
            eidx[e] = (int32_t)e;
        }
    }
    // all 32 lanes shuffle; the same tree as eb_eval_topk_f64, so the nDCG has its bits
#pragma unroll
    for (int o = G / 2; o; o >>= 1) {
        dcg += __shfl_xor_sync(0xffffffffu, dcg, o, G);
        ssum += __shfl_xor_sync(0xffffffffu, ssum, o, G);
    }
    if (live && lane == 0) {
        const int key = in_b && gu >= 0 ? gu : nu;
        ukey[row] = key;
        urow[row] = (int32_t)row;
        row_ndcg[row] = in_b && dcg > 0 ? dcg / idcg[u] : 0.0;
        row_mean[row] = scores ? ssum / (double)n : 0.0;      // 0 / 0 = NaN for an empty list, as np.average([])
        atomicAdd(ucount + key, 1);
    }
    if (in_shared) {
        __syncthreads();
        for (int b = threadIdx.x; b < n_bins; b += EF_THREADS)
            if (hist_s[b]) atomicAdd(hist_g + b, (unsigned long long)hist_s[b]);
    }
}

// per item with entries: the sums of its entries' gains and relevant scores in sorted (row, position) order, / count;
// the item's key for the cluster sort (its item cluster, or ni when it has no entry or no cluster)
__global__ void fairness_item_kernel(const int32_t *__restrict__ item_count, const int32_t *__restrict__ item_off,
                                     const int32_t *__restrict__ sorted_e, const double *__restrict__ egain,
                                     const double *__restrict__ escore, const int32_t *__restrict__ icl, int ni,
                                     int n_items, double *__restrict__ v_rank, double *__restrict__ v_rate,
                                     int32_t *__restrict__ ikey, int32_t *__restrict__ iidx, int32_t *__restrict__ icount) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += gridDim.x * blockDim.x) {
        const int c = item_count[i];
        double gs = 0, rs = 0;
        for (int j = item_off[i], end = item_off[i] + c; j < end; ++j) {
            const int32_t e = sorted_e[j];
            gs += egain[e];
            rs += escore[e];
        }
        v_rank[i] = c ? gs / (double)c : 0.0;
        v_rate[i] = c ? rs / (double)c : 0.0;
        const int key = c > 0 && icl[i] >= 0 ? icl[i] : ni;
        ikey[i] = key;
        iidx[i] = i;
        atomicAdd(icount + key, 1);
    }
}

// one warp per cluster: user clusters 0..nu-1 sum (nDCG, mean score) over their rows, item clusters sum (ranking, rating)
// averages over their items, each in sorted order, lanes strided, fixed shuffle tree
__global__ void fairness_cluster_kernel(const int32_t *__restrict__ u_cnt, const int32_t *__restrict__ u_off,
                                        const int32_t *__restrict__ u_sorted, const double *__restrict__ row_ndcg,
                                        const double *__restrict__ row_mean, int nu, const int32_t *__restrict__ i_cnt,
                                        const int32_t *__restrict__ i_off, const int32_t *__restrict__ i_sorted,
                                        const double *__restrict__ v_rank, const double *__restrict__ v_rate, int ni,
                                        int64_t *__restrict__ counts, double *__restrict__ sums) {
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32;
    const int lane = threadIdx.x % 32;
    if (w >= (int64_t)nu + ni) return;                        // whole warps leave together
    const bool user = w < nu;
    const int c = user ? (int)w : (int)(w - nu);
    const int32_t cnt = user ? u_cnt[c] : i_cnt[c], off = user ? u_off[c] : i_off[c];
    const int32_t *idx = user ? u_sorted : i_sorted;
    const double *x = user ? row_ndcg : v_rank, *y = user ? row_mean : v_rate;
    double a = 0, b = 0;
    for (int j = lane; j < cnt; j += 32) {
        const int32_t t = idx[off + j];
        a += x[t];
        b += y[t];
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane == 0) {
        if (user) {
            counts[c] = cnt;
            sums[c] = a;
            sums[nu + c] = b;
        } else {
            counts[(int64_t)nu + (int64_t)nu * ni + 2 * ni + c] = cnt;
            sums[2 * nu + c] = a;
            sums[2 * nu + ni + c] = b;
        }
    }
}

struct EfLayout {
    size_t ukey[2], urow[2], row_ndcg, row_mean, ekey[2], eidx[2], egain, escore, ikey[2], iidx[2], v_rank, v_rate,
        zero, item_count, ucount, icount, zero_end, item_off, u_off, i_off, cub, cub_bytes, total;
};

static EfLayout ef_layout(int64_t n_rows, int k, int n_items, int nu, int ni) {
    const int64_t m = n_rows * k;
    EfLayout L;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t at = off; off += align_up(bytes); return at; };
    for (int b = 0; b < 2; ++b) {
        L.ukey[b] = take(sizeof(int32_t) * (size_t)n_rows);
        L.urow[b] = take(sizeof(int32_t) * (size_t)n_rows);
        L.ekey[b] = take(sizeof(int32_t) * (size_t)m);
        L.eidx[b] = take(sizeof(int32_t) * (size_t)m);
        L.ikey[b] = take(sizeof(int32_t) * (size_t)n_items);
        L.iidx[b] = take(sizeof(int32_t) * (size_t)n_items);
    }
    L.row_ndcg = take(sizeof(double) * (size_t)n_rows);
    L.row_mean = take(sizeof(double) * (size_t)n_rows);
    L.egain = take(sizeof(double) * (size_t)m);
    L.escore = take(sizeof(double) * (size_t)m);
    L.v_rank = take(sizeof(double) * (size_t)n_items);
    L.v_rate = take(sizeof(double) * (size_t)n_items);
    // the three histograms are contiguous: one memset zeroes them
    L.zero = off;
    L.item_count = off; off += sizeof(int32_t) * ((size_t)n_items + 1);
    L.ucount = off; off += sizeof(int32_t) * ((size_t)nu + 1);
    L.icount = off; off += sizeof(int32_t) * ((size_t)ni + 1);
    L.zero_end = off;
    off = align_up(off);
    L.item_off = take(sizeof(int32_t) * ((size_t)n_items + 1));
    L.u_off = take(sizeof(int32_t) * ((size_t)nu + 1));
    L.i_off = take(sizeof(int32_t) * ((size_t)ni + 1));
    size_t cb = 0, c1 = 0;
    cub::DoubleBuffer<int32_t> kb(nullptr, nullptr), vb(nullptr, nullptr);
    const int64_t most = m > n_items ? m : n_items;
    const int n_scan = (n_items > nu ? (n_items > ni ? n_items : ni) : (nu > ni ? nu : ni)) + 1;
    cub::DeviceRadixSort::SortPairs(nullptr, c1, kb, vb, (int)(most > n_rows ? most : n_rows), 0, 32);
    cb = c1;
    cub::DeviceScan::ExclusiveSum(nullptr, c1, (int32_t *)nullptr, (int32_t *)nullptr, n_scan);
    cb = cb > c1 ? cb : c1;
    L.cub_bytes = cb;
    L.cub = take(cb);
    L.total = off;
    return L;
}

static int64_t ef_counts_len(int nu, int ni) { return (int64_t)nu + (int64_t)nu * ni + 3 * (int64_t)ni; }

}  // namespace eb

extern "C" size_t eb_eval_fairness_workspace_bytes(int64_t n_rows, int k, int n_items, int n_user_clusters,
                                                   int n_item_clusters) {
    if (n_rows < 0 || k < 1 || n_items < 0 || n_user_clusters < 1 || n_item_clusters < 1) return 0;
    return eb::ef_layout(n_rows, k, n_items, n_user_clusters, n_item_clusters).total;
}

extern "C" int eb_eval_fairness_f64(const int32_t *topk_idx, const double *scores, int64_t n_rows, int ld, int k,
                                    const int32_t *users, const int64_t *rel_indptr, const int32_t *rel_items,
                                    const double *rel_gains, const double *idcg, const double *discount,
                                    const uint8_t *has_rows, const int32_t *user_cluster, int n_user_clusters,
                                    const int32_t *item_cluster, int n_item_clusters, int n_items, int64_t *counts,
                                    double *sums, void *workspace, size_t workspace_bytes, void *stream) {
    using namespace eb;
    const int nu = n_user_clusters, ni = n_item_clusters;
    EB_ARG(counts && sums, "null output pointer");
    EB_ARG(n_rows >= 0 && k >= 1 && k <= 1024 && ld >= k && n_items >= 0 && nu >= 1 && ni >= 1,
           "bad shape (n_rows=%lld k=%d ld=%d n_items=%d clusters=%d x %d)", (long long)n_rows, k, ld, n_items, nu, ni);
    EB_ARG((int64_t)nu * ni + 3 * (int64_t)ni < 0x7fffffffLL, "too many clusters (%d x %d)", nu, ni);
    EB_ARG(n_rows * k < 0x7fffffffLL, "too many list entries for one launch (%lld rows x %d)", (long long)n_rows, k);
    cudaStream_t st = (cudaStream_t)stream;
    EB_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * ef_counts_len(nu, ni), st));
    EB_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * (2 * (size_t)nu + 2 * (size_t)ni), st));
    if (n_rows == 0) return EB_OK;                             // empty list set: nothing evaluated
    EB_ARG(topk_idx && rel_indptr && rel_items && rel_gains && idcg && discount && has_rows && user_cluster && item_cluster,
           "null pointer");
    const EfLayout L = ef_layout(n_rows, k, n_items, nu, ni);
    if (workspace_bytes < L.total || !workspace)
        return set_err(EB_ERR_WORKSPACE, "eval fairness workspace too small: need %zu bytes", L.total);
    char *ws = (char *)workspace;
    auto I = [&](size_t o) { return (int32_t *)(ws + o); };
    auto D = [&](size_t o) { return (double *)(ws + o); };
    EB_CUDA(cudaMemsetAsync(ws + L.zero, 0, L.zero_end - L.zero, st));
    const int G = ef_group(k);
    const int64_t blocks = (n_rows + EF_THREADS / G - 1) / (EF_THREADS / G);
    EB_ARG(blocks <= 0x7fffffffLL, "too many rows for one launch");
    unsigned long long *hist = (unsigned long long *)(counts + nu);
#define EB_LAUNCH(GV)                                                                                                  \
    fairness_row_kernel<GV><<<(unsigned)blocks, EF_THREADS, 0, st>>>(                                                  \
        topk_idx, scores, n_rows, ld, k, users, rel_indptr, rel_items, rel_gains, idcg, discount, has_rows, user_cluster, \
        nu, item_cluster, ni, n_items, hist, I(L.ukey[0]), I(L.urow[0]), D(L.row_ndcg), D(L.row_mean), I(L.ucount),     \
        I(L.ekey[0]), I(L.eidx[0]), D(L.egain), D(L.escore), I(L.item_count))
    if (G == 8) EB_LAUNCH(8); else if (G == 16) EB_LAUNCH(16); else EB_LAUNCH(32);
#undef EB_LAUNCH
    EB_CUDA(cudaGetLastError());

    size_t cb = L.cub_bytes;
    const int m = (int)(n_rows * k);
    cub::DoubleBuffer<int32_t> ek(I(L.ekey[0]), I(L.ekey[1])), ev(I(L.eidx[0]), I(L.eidx[1]));
    EB_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.cub, cb, ek, ev, m, 0, bits_for((uint64_t)n_items), st));
    cb = L.cub_bytes;
    EB_CUDA(cub::DeviceScan::ExclusiveSum(ws + L.cub, cb, I(L.item_count), I(L.item_off), n_items + 1, st));
    if (n_items > 0) {
        const int ib = n_items > 256 * 1024 ? 1024 : (n_items + 255) / 256;
        fairness_item_kernel<<<ib, 256, 0, st>>>(I(L.item_count), I(L.item_off), ev.Current(), D(L.egain), D(L.escore),
                                                 item_cluster, ni, n_items, D(L.v_rank), D(L.v_rate), I(L.ikey[0]),
                                                 I(L.iidx[0]), I(L.icount));
        EB_CUDA(cudaGetLastError());
    }
    cb = L.cub_bytes;
    cub::DoubleBuffer<int32_t> ik(I(L.ikey[0]), I(L.ikey[1])), iv(I(L.iidx[0]), I(L.iidx[1]));
    EB_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.cub, cb, ik, iv, n_items, 0, bits_for((uint64_t)ni), st));
    cb = L.cub_bytes;
    cub::DoubleBuffer<int32_t> uk(I(L.ukey[0]), I(L.ukey[1])), uv(I(L.urow[0]), I(L.urow[1]));
    EB_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.cub, cb, uk, uv, (int)n_rows, 0, bits_for((uint64_t)nu), st));
    cb = L.cub_bytes;
    EB_CUDA(cub::DeviceScan::ExclusiveSum(ws + L.cub, cb, I(L.ucount), I(L.u_off), nu + 1, st));
    cb = L.cub_bytes;
    EB_CUDA(cub::DeviceScan::ExclusiveSum(ws + L.cub, cb, I(L.icount), I(L.i_off), ni + 1, st));
    const int64_t warps = (int64_t)nu + ni;
    fairness_cluster_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(
        I(L.ucount), I(L.u_off), uv.Current(), D(L.row_ndcg), D(L.row_mean), nu, I(L.icount), I(L.i_off), iv.Current(),
        D(L.v_rank), D(L.v_rate), ni, counts, sums);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
