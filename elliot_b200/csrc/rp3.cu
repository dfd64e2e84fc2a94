// rp3.cu — RP3beta (graph_based/RP3beta/rp3beta.py:73-176) on the GPU, with the reference's float32 sparse products
// reproduced bit for bit.  SciPy's float32 `csr * csr` computes each output row as acc[j] = fp32(acc[j] + fp32(a_e * b_ej))
// over the left row's entries e in stored order; every kernel here that sums keeps exactly that order per column, with
// __fmul_rn / __fadd_rn (no FMA contraction, no atomics).
//   rp3_rows_kernel<true>   : similarity row i = Piu[i] . Pui, times degree in fp64, diagonal zeroed, the k largest nonzero
//                             values (value desc, column asc) written as fp32 in column order;
//   rp3_rows_kernel<false>  : score row u = R[u] . W, train items masked, the k best (score desc, column asc);
//   rp3_l1_rows_kernel      : W rows <- fp32(v / sum |v|), the sum in fp64 in stored (column) order;
//   prune kernels           : per column of W the k largest nonzero values (value desc, row asc), W rebuilt as a CSR.
// The three selects run block_select.cuh on 64-bit keys with 8-bit digits: fp64 bit patterns (similarity) or
// (value, index) pair keys (scores, prune).
#include <math_constants.h>

#include "block_select.cuh"
#include "common.cuh"

namespace eb {

constexpr int RP3_NT = 512;                  // threads per CTA
constexpr int RP3_NW = RP3_NT / 32;
constexpr int RP3_TILE = 49152;              // fp32 accumulators per column tile (192 KB of shared memory)
constexpr int RP3_BITS = 8;                  // radix digit: 8 x 8 bits of the 64-bit keys

using Rp3Sel = SelectShared<RP3_NT, RP3_BITS>;

// first index in [lo, hi) of the sorted a[] with a[idx] >= key; every lane of the warp gets it (<= 2 probe rounds for
// rows of up to 1 024 entries)
__device__ __forceinline__ int64_t warp_lower_bound(const int32_t *__restrict__ a, int64_t lo, int64_t hi, int32_t key,
                                                    int lane) {
    while (hi - lo > 32) {
        const int64_t step = (hi - lo + 31) >> 5;
        const int64_t q = lo + (int64_t)lane * step;
        const int cnt = __popc(__ballot_sync(0xffffffffu, q < hi && __ldg(a + q) < key));
        if (cnt == 0) return lo;
        const int64_t nhi = lo + (int64_t)cnt * step;
        lo += (int64_t)(cnt - 1) * step + 1;
        hi = nhi < hi ? nhi : hi;
    }
    const int64_t q = lo + lane;
    return lo + __popc(__ballot_sync(0xffffffffu, q < hi && __ldg(a + q) < key));
}

struct Rp3Params {
    const int64_t *a_indptr; const int32_t *a_indices; const float *a_values;     // left rows, summed in stored order
    const int64_t *b_indptr; const int32_t *b_indices; const float *b_values;     // right rows, sorted by column
    int32_t n_cols;
    const int32_t *users;       // output row q reads left row users[q] (or user_begin + q)
    int32_t user_begin;
    int64_t n_sel;
    const int32_t *order;       // visiting order of the output rows (NULL: 0, 1, ...)
    int k, tile;
    float *row_ws;              // [gridDim.x][n_cols] when n_cols > tile
    int64_t stride;             // output row stride
    int32_t *out_idx;
    float *out_val;
    // similarity
    const double *degree;
    int32_t *out_cnt;
    // scoring
    const int64_t *mask_indptr; const int32_t *mask_indices;
};

// acc[c - c0] (c in [c0, c0 + tn)) += the left row a0..a1 times the right rows, in left-entry order per column.  Warp w owns
// a slice of the tile's columns and walks every left entry; the entries of one right row hit distinct columns, so the
// lanes add them in parallel, and __syncwarp orders consecutive left entries.  No CTA barrier inside.
__device__ __forceinline__ void rp3_accumulate(const Rp3Params &p, float *acc, int64_t a0, int64_t a1, int c0, int tn) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int per = (tn + RP3_NW - 1) / RP3_NW;
    const int lo = c0 + warp * per, hi = min(lo + per, c0 + tn);
    if (lo >= hi) return;
    for (int64_t e = a0; e < a1; e++) {
        const int32_t r = __ldg(p.a_indices + e);
        const float a = __ldg(p.a_values + e);
        const int64_t b0 = __ldg(p.b_indptr + r), b1 = __ldg(p.b_indptr + r + 1);
        for (int64_t j = warp_lower_bound(p.b_indices, b0, b1, lo, lane) + lane; j < b1; j += 32) {
            const int32_t c = __ldg(p.b_indices + j);
            if (c >= hi) break;
            float *s = acc + (c - c0);
            *s = __fadd_rn(*s, __fmul_rn(a, __ldg(p.b_values + j)));
        }
        __syncwarp();
    }
}

// Three CTAs per SM (40 registers) whenever the accumulator row leaves room for them.
template <bool SIM>
__global__ void __launch_bounds__(RP3_NT, 3) rp3_rows_kernel(const Rp3Params p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *acc = reinterpret_cast<float *>(smem_raw);                                  // [tile]
    uint64_t *keys = reinterpret_cast<uint64_t *>(acc + p.tile);                       // [SELECT_KMAX], scoring only
    __shared__ Rp3Sel sh;
    const bool tiled = p.n_cols > p.tile;
    float *grow = tiled ? p.row_ws + (int64_t)blockIdx.x * p.n_cols : nullptr;
    for (int64_t t = blockIdx.x; t < p.n_sel; t += gridDim.x) {
        const int64_t q = p.order ? (int64_t)p.order[t] : t;
        const int r = p.users ? p.users[q] : p.user_begin + (int)q;
        const int64_t a0 = p.a_indptr[r], a1 = p.a_indptr[r + 1];
        for (int c0 = 0; c0 < p.n_cols; c0 += p.tile) {
            const int tn = min(p.tile, p.n_cols - c0);
            for (int i = threadIdx.x; i < tn; i += RP3_NT) acc[i] = 0.f;
            __syncthreads();
            rp3_accumulate(p, acc, a0, a1, c0, tn);
            __syncthreads();
            if (!SIM && p.mask_indptr) {
                const int64_t m0 = p.mask_indptr[r], m1 = p.mask_indptr[r + 1];
                for (int64_t m = m0 + threadIdx.x; m < m1; m += RP3_NT) {
                    const int32_t c = __ldg(p.mask_indices + m);
                    if (c >= c0 && c < c0 + tn) acc[c - c0] = -CUDART_INF_F;
                }
                __syncthreads();
            }
            if (tiled) {
                for (int i = threadIdx.x; i < tn; i += RP3_NT) grow[c0 + i] = acc[i];
                __syncthreads();
            }
        }
        const float *row = tiled ? grow : acc;
        if (SIM) {
            const double *deg = p.degree;
            auto get = [row, deg, r](int i, uint64_t &key) {
                const double v = i == r ? 0.0 : (double)row[i] * __ldg(deg + i);       // rp3beta.py:120-121
                key = (uint64_t)__double_as_longlong(v);
                return v > 0.0 && v < CUDART_INF;
            };
            uint64_t T;
            int need_eq;
            radix_threshold(get, p.n_cols, p.k, sh, T, need_eq);
            int32_t *oi = p.out_idx + q * p.stride;
            float *ov = p.out_val + q * p.stride;
            const int m = collect(get, p.n_cols, T, need_eq, sh, [oi, ov](int slot, int i, uint64_t key) {
                oi[slot] = i;
                ov[slot] = (float)__longlong_as_double((long long)key);
            });
            if (threadIdx.x == 0) p.out_cnt[q] = m;
        } else {
            auto get = [row](int i, uint64_t &key) {
                const float v = row[i];
                key = pair_key(v, (uint32_t)i);
                return v != -CUDART_INF_F;
            };
            uint64_t T;
            int need_eq;
            radix_threshold(get, p.n_cols, p.k, sh, T, need_eq);
            auto put = [keys](int slot, int, uint64_t key) { keys[slot] = key; };
            const int m = collect(get, p.n_cols, T, need_eq, sh, put);
            sort_desc<RP3_NT>(keys, m);
            write_topk<RP3_NT>(keys, m, p.k, p.out_idx + q * p.stride, p.out_val + q * p.stride, -CUDART_INF_F);
        }
        __syncthreads();
    }
}

__global__ void rp3_l1_rows_kernel(int32_t n_rows, int64_t stride, const int32_t *__restrict__ cnt, float *val) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        float *v = val + r * stride;
        const int m = cnt[r];
        double s = 0.0;
        for (int j = 0; j < m; j++) s += fabs((double)v[j]);
        if (s == 0.0) continue;                                   // sklearn leaves such rows alone
        for (int j = 0; j < m; j++) v[j] = (float)((double)v[j] / s);
    }
}

// ---------------------------------------------------------------- column prune
// W's rows as fixed-stride lists (row r: columns idx[r * stride + j] ascending, j < cnt[r]).
__global__ void rp3_count_cols_kernel(int32_t n, int64_t stride, const int32_t *__restrict__ cnt,
                                      const int32_t *__restrict__ idx, const float *__restrict__ val, int32_t *col_cnt) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((int64_t)gridDim.x * blockDim.x) >> 5)
        for (int j = lane; j < cnt[r]; j += 32)
            if (val[r * stride + j] != 0.f) atomicAdd(col_cnt + idx[r * stride + j], 1);
}

// out[0] = 0, out[i + 1] = out[i] + in[i] (one CTA)
__global__ void __launch_bounds__(1024) rp3_scan_kernel(const int32_t *__restrict__ in, int32_t n, int64_t *out) {
    __shared__ long long wsum[32];
    __shared__ long long carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { carry = 0; out[0] = 0; }
    __syncthreads();
    for (int i0 = 0; i0 < n; i0 += 1024) {
        const int i = i0 + (int)threadIdx.x;
        long long v = i < n ? in[i] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += y;
        }
        if (lane == 31) wsum[warp] = v;
        __syncthreads();
        long long before = carry;
        for (int w = 0; w < warp; w++) before += wsum[w];
        if (i < n) out[i + 1] = before + v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = before + v;
        __syncthreads();
    }
}

__global__ void rp3_scatter_cols_kernel(int32_t n, int64_t stride, const int32_t *__restrict__ cnt,
                                        const int32_t *__restrict__ idx, const float *__restrict__ val,
                                        const int64_t *__restrict__ col_ptr, int32_t *col_fill, uint64_t *ckeys) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((int64_t)gridDim.x * blockDim.x) >> 5)
        for (int j = lane; j < cnt[r]; j += 32) {
            const float v = val[r * stride + j];
            if (v == 0.f) continue;                                // rp3beta.py:163
            const int32_t c = idx[r * stride + j];
            ckeys[col_ptr[c] + atomicAdd(col_fill + c, 1)] = pair_key(v, (uint32_t)r);   // slot order is irrelevant
        }
}

// per column: the k largest (value, row) keys; each kept entry is flagged at its place in its row's list
__global__ void __launch_bounds__(RP3_NT) rp3_select_cols_kernel(int32_t n, int64_t stride, const int32_t *__restrict__ cnt,
                                                                 const int32_t *__restrict__ idx,
                                                                 const int64_t *__restrict__ col_ptr,
                                                                 const uint64_t *__restrict__ ckeys, int k, uint8_t *keep) {
    __shared__ Rp3Sel sh;
    for (int c = blockIdx.x; c < n; c += gridDim.x) {
        const uint64_t *ck = ckeys + col_ptr[c];
        const int len = (int)(col_ptr[c + 1] - col_ptr[c]);
        auto mark = [=](int, int, uint64_t key) {
            const int64_t r = pair_index(key);
            const int32_t *row = idx + r * stride;
            int lo = 0, hi = cnt[r];
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (row[mid] < c) lo = mid + 1; else hi = mid;
            }
            keep[r * stride + lo] = 1;
        };
        if (len <= k) {                                            // keep all (uniform)
            for (int i = threadIdx.x; i < len; i += RP3_NT) mark(0, i, ck[i]);
            continue;
        }
        auto get = [ck](int i, uint64_t &key) { key = ck[i]; return true; };
        uint64_t T;
        int need_eq;
        radix_threshold(get, len, k, sh, T, need_eq);
        collect(get, len, T, need_eq, sh, mark);
        __syncthreads();
    }
}

__global__ void rp3_count_kept_kernel(int32_t n, int64_t stride, const int32_t *__restrict__ cnt,
                                      const uint8_t *__restrict__ keep, int32_t *row_cnt) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        int s = 0;
        for (int j = lane; j < cnt[r]; j += 32) s += keep[r * stride + j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) row_cnt[r] = s;
    }
}

__global__ void rp3_compact_kernel(int32_t n, int64_t stride, const int32_t *__restrict__ cnt,
                                   const int32_t *__restrict__ idx, const float *__restrict__ val,
                                   const uint8_t *__restrict__ keep, const int64_t *__restrict__ indptr, int32_t *out_indices,
                                   float *out_values) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n; r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
        int64_t o = indptr[r];
        for (int j0 = 0; j0 < cnt[r]; j0 += 32) {
            const int j = j0 + lane;
            const bool kp = j < cnt[r] && keep[r * stride + j];
            const unsigned b = __ballot_sync(0xffffffffu, kp);
            if (kp) {
                const int64_t at = o + __popc(b & ((1u << lane) - 1u));
                out_indices[at] = idx[r * stride + j];
                out_values[at] = val[r * stride + j];
            }
            o += __popc(b);
        }
    }
}

struct PruneWs {
    int32_t *col_cnt, *col_fill;
    int64_t *col_ptr;
    uint64_t *ckeys;
    uint8_t *keep;
    size_t bytes;
};

static size_t align256(size_t b) { return (b + 255) / 256 * 256; }

static PruneWs prune_ws(void *base, int32_t n, int64_t stride, int64_t nnz) {
    PruneWs w{};
    size_t o = 0;
    unsigned char *b = (unsigned char *)base;
    w.col_cnt = (int32_t *)(b + o); o += align256((size_t)n * 4);
    w.col_fill = (int32_t *)(b + o); o += align256((size_t)n * 4);
    w.col_ptr = (int64_t *)(b + o); o += align256((size_t)(n + 1) * 8);
    w.ckeys = (uint64_t *)(b + o); o += align256((size_t)nnz * 8);
    w.keep = (uint8_t *)(b + o); o += align256((size_t)n * (size_t)stride);
    w.bytes = o;
    return w;
}

static size_t rows_smem(const Rp3Params &p, bool sim) {
    return (size_t)p.tile * 4 + (sim ? 0 : (size_t)SELECT_KMAX * 8);
}

template <bool SIM>
static int launch_rows(Rp3Params p, void *workspace, size_t workspace_bytes, void *stream) {
    p.tile = p.n_cols < RP3_TILE ? (p.n_cols + 3) / 4 * 4 : RP3_TILE;
    const size_t smem = rows_smem(p, SIM);
    EB_CUDA(cudaFuncSetAttribute(rp3_rows_kernel<SIM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    EB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rp3_rows_kernel<SIM>, RP3_NT, smem));
    if (per_sm < 1) per_sm = 1;
    int64_t grid = (int64_t)sm_count() * per_sm;
    if (p.n_cols > p.tile) {
        const int64_t fit = (int64_t)(workspace_bytes / ((size_t)p.n_cols * 4));
        EB_ARG(workspace && fit >= 1, "workspace: %zu bytes, a column-tiled row needs %zu", workspace_bytes,
               (size_t)p.n_cols * 4);
        if (grid > fit) grid = fit;
        p.row_ws = (float *)workspace;
    }
    if (grid > p.n_sel) grid = p.n_sel;
    rp3_rows_kernel<SIM><<<(unsigned)grid, RP3_NT, smem, (cudaStream_t)stream>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

static unsigned warp_grid(int64_t rows) {          // one warp per row, 8 warps per CTA, at most 16 CTAs per SM
    int64_t g = (rows + 7) / 8;
    const int64_t cap = (int64_t)sm_count() * 16;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace eb

using namespace eb;

extern "C" int eb_rp3_tile_cols(void) { return RP3_TILE; }

extern "C" size_t eb_rp3_row_workspace_bytes(int32_t n_cols) {
    return n_cols > RP3_TILE ? (size_t)sm_count() * (size_t)n_cols * 4 : 0;
}

extern "C" int eb_rp3_similarity_f32(const int64_t *a_indptr, const int32_t *a_indices, const float *a_values,
                                     const int64_t *b_indptr, const int32_t *b_indices, const float *b_values,
                                     const double *degree, int32_t n_items, const int32_t *order, int k, int64_t stride,
                                     int32_t *out_idx, float *out_val, int32_t *out_cnt, void *workspace,
                                     size_t workspace_bytes, void *stream) {
    EB_ARG(a_indptr && a_indices && a_values && b_indptr && b_indices && b_values && degree && out_idx && out_val && out_cnt,
           "null pointer");
    EB_ARG(n_items >= 1, "bad shape n_items=%d", n_items);
    EB_ARG(k >= 1 && stride >= (k < n_items ? k : n_items), "k=%d stride=%lld: need k >= 1 and stride >= min(k, n_items)", k,
           (long long)stride);
    Rp3Params p{};
    p.a_indptr = a_indptr; p.a_indices = a_indices; p.a_values = a_values;
    p.b_indptr = b_indptr; p.b_indices = b_indices; p.b_values = b_values;
    p.n_cols = n_items; p.n_sel = n_items; p.order = order; p.k = k < n_items ? k : n_items; p.stride = stride;
    p.out_idx = out_idx; p.out_val = out_val; p.degree = degree; p.out_cnt = out_cnt;
    return launch_rows<true>(p, workspace, workspace_bytes, stream);
}

extern "C" int eb_rp3_l1_rows_f32(int32_t n_rows, int64_t stride, const int32_t *cnt, float *val, void *stream) {
    EB_ARG(cnt && val, "null pointer");
    EB_ARG(n_rows >= 0 && stride >= 1, "bad shape n_rows=%d stride=%lld", n_rows, (long long)stride);
    if (n_rows == 0) return EB_OK;
    int64_t grid = ((int64_t)n_rows + 255) / 256;
    rp3_l1_rows_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(n_rows, stride, cnt, val);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" size_t eb_rp3_prune_workspace_bytes(int32_t n, int64_t stride, int64_t nnz) {
    return prune_ws(nullptr, n, stride, nnz).bytes;
}

extern "C" int eb_rp3_prune_cols_f32(int32_t n, int64_t stride, const int32_t *cnt, const int32_t *idx, const float *val,
                                     int64_t nnz, int k, int64_t *out_indptr, int32_t *out_indices, float *out_values,
                                     void *workspace, size_t workspace_bytes, void *stream) {
    EB_ARG(cnt && idx && val && out_indptr && out_indices && out_values && workspace, "null pointer");
    EB_ARG(n >= 1 && stride >= 1 && nnz >= 0 && k >= 1, "bad shape n=%d stride=%lld nnz=%lld k=%d", n, (long long)stride,
           (long long)nnz, k);
    PruneWs w = prune_ws(workspace, n, stride, nnz);
    EB_ARG(workspace_bytes >= w.bytes, "workspace: %zu bytes, need %zu", workspace_bytes, w.bytes);
    cudaStream_t st = (cudaStream_t)stream;
    EB_CUDA(cudaMemsetAsync(w.col_cnt, 0, (size_t)n * 4, st));
    EB_CUDA(cudaMemsetAsync(w.col_fill, 0, (size_t)n * 4, st));
    EB_CUDA(cudaMemsetAsync(w.keep, 0, (size_t)n * (size_t)stride, st));
    const unsigned g = warp_grid(n);
    rp3_count_cols_kernel<<<g, 256, 0, st>>>(n, stride, cnt, idx, val, w.col_cnt);
    rp3_scan_kernel<<<1, 1024, 0, st>>>(w.col_cnt, n, w.col_ptr);
    rp3_scatter_cols_kernel<<<g, 256, 0, st>>>(n, stride, cnt, idx, val, w.col_ptr, w.col_fill, w.ckeys);
    int64_t cg = (int64_t)sm_count() * 4;
    if (cg > n) cg = n;
    rp3_select_cols_kernel<<<(unsigned)cg, RP3_NT, 0, st>>>(n, stride, cnt, idx, w.col_ptr, w.ckeys, k, w.keep);
    rp3_count_kept_kernel<<<g, 256, 0, st>>>(n, stride, cnt, w.keep, w.col_cnt);
    rp3_scan_kernel<<<1, 1024, 0, st>>>(w.col_cnt, n, out_indptr);
    rp3_compact_kernel<<<g, 256, 0, st>>>(n, stride, cnt, idx, val, w.keep, out_indptr, out_indices, out_values);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_rp3_score_topk_f32(const int64_t *a_indptr, const int32_t *a_indices, const float *a_values,
                                     const int64_t *b_indptr, const int32_t *b_indices, const float *b_values, int32_t n_cols,
                                     const int64_t *mask_indptr, const int32_t *mask_indices, const int32_t *users,
                                     int32_t user_begin, int64_t n_sel, const int32_t *order, int k, int32_t *out_idx,
                                     float *out_val, void *workspace, size_t workspace_bytes, void *stream) {
    EB_ARG(a_indptr && a_indices && a_values && b_indptr && b_indices && b_values && out_idx && out_val, "null pointer");
    EB_ARG(n_cols >= 1 && n_sel >= 0 && user_begin >= 0, "bad shape n_cols=%d n_sel=%lld", n_cols, (long long)n_sel);
    EB_ARG(k >= 1 && k <= SELECT_KMAX, "k=%d outside [1, %d]", k, SELECT_KMAX);
    EB_ARG((mask_indptr == nullptr) == (mask_indices == nullptr), "mask CSR: both or neither");
    if (n_sel == 0) return EB_OK;
    Rp3Params p{};
    p.a_indptr = a_indptr; p.a_indices = a_indices; p.a_values = a_values;
    p.b_indptr = b_indptr; p.b_indices = b_indices; p.b_values = b_values;
    p.n_cols = n_cols; p.users = users; p.user_begin = user_begin; p.n_sel = n_sel; p.order = order; p.k = k; p.stride = k;
    p.out_idx = out_idx; p.out_val = out_val; p.mask_indptr = mask_indptr; p.mask_indices = mask_indices;
    return launch_rows<false>(p, workspace, workspace_bytes, stream);
}
