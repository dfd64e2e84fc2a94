// peer.cu — embedding tables spread over the GPUs of ONE NVSwitch box and addressed directly by the kernels
// (SURVEY.md §8e; no reference counterpart: the reference is single-device, SURVEY.md §2.1).
//
// One process per GPU.  A rank allocates its part of a table with eb_peer_alloc (plain cudaMalloc, so that the
// allocation can be exported), publishes the 64-byte CUDA IPC handle (eb_peer_export; the host exchanges the handles
// with torch.distributed), and maps every other rank's part into its own address space (eb_peer_open:
// cudaIpcOpenMemHandle with lazy peer access).  From then on kernels take an array of base pointers — one per rank —
// and load / atomically add rows wherever they live: NVLink 5 carries 128-bit loads and `red.add.v4.f32` natively, so
// the "all-to-all of ids -> owners gather -> all-to-all of rows -> update -> all-to-all of deltas -> owners scatter"
// pipeline of an NCCL formulation collapses into the training kernel itself (bpr_train.cu PEER mode, the NeuMF kernels
// below), with no bucketing, no staging buffers and no host synchronisation.
//
//   eb_table_reconcile_peer_f32   REPLICATED tables (small catalogues, C2): every rank trains on its own copy; rank r
//       owns slice r of the table and, in ONE kernel, reads that slice of every rank's copy over NVLink, forms each
//       rank's delta against the slice's last agreed value `prev`, averages (or sums) the deltas and pushes
//       `agreed - delta_p` back into every copy with vector atomics, then advances `prev`.  Because the correction is
//       ADDED atomically, a training kernel running on the target GPU at the same time loses nothing: whatever it adds
//       after the snapshot simply stays in that copy as not-yet-shared progress.  No barrier, no collective call, and
//       `prev` exists only on the slice's owner.
//   eb_neumf_gather_peer / eb_neumf_scatter_peer   NeuMF with the two item tables side by side in one row-sharded
//       [items, 2f] table (neural_matrix_factorization_model.py:74-106): item rows are read from, and item-row
//       gradients are added into, the owner's memory.
#include "common.cuh"

namespace eb {

struct PeerTab {
    float *base[EB_MAX_PEERS];
};

struct ShardMap {
    uint32_t rows, magic;
    __device__ __forceinline__ void locate(int i, int &owner, int &local) const {
        uint32_t o = __umulhi((uint32_t)i, magic);
        uint32_t r = (uint32_t)i - o * rows;
        if (r >= rows) { o++; r -= rows; }
        owner = (int)o; local = (int)r;
    }
};

static ShardMap shard_map(int32_t shard_rows) {
    const uint64_t m = (1ull << 32) / (uint64_t)shard_rows;
    return ShardMap{(uint32_t)shard_rows, (uint32_t)(m > 0xffffffffull ? 0xffffffffull : m)};
}

static int fill_tab(PeerTab &t, float *const *ptrs, int n) {
    EB_ARG(ptrs && n >= 1 && n <= EB_MAX_PEERS, "1 <= n_peers <= %d", EB_MAX_PEERS);
    for (int s = 0; s < n; s++) {
        EB_ARG(ptrs[s] && ((uintptr_t)ptrs[s] % 16) == 0, "null / misaligned peer pointer %d", s);
        t.base[s] = ptrs[s];
    }
    for (int s = n; s < EB_MAX_PEERS; s++) t.base[s] = ptrs[0];
    return EB_OK;
}

// ---------------------------------------------------------------- replicated-table reconciliation
// e indexes float4 elements of this rank's slice; T.base[p] points at element 0 of the slice inside rank p's copy.
template <int NP>
__global__ void __launch_bounds__(256) table_reconcile_peer_kernel(PeerTab T, float4 *__restrict__ prev, int64_t n4, float scale) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += stride) {
        const float4 pv = prev[e];
        float4 snap[NP];
#pragma unroll
        for (int p = 0; p < NP; p++) snap[p] = ld_sys_v4(reinterpret_cast<const float4 *>(T.base[p]) + e);
        float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
        bool touched = false;
#pragma unroll
        for (int p = 0; p < NP; p++) {
            const float4 dl = make_float4(snap[p].x - pv.x, snap[p].y - pv.y, snap[p].z - pv.z, snap[p].w - pv.w);
            touched |= dl.x != 0.f || dl.y != 0.f || dl.z != 0.f || dl.w != 0.f;
            sum.x += dl.x; sum.y += dl.y; sum.z += dl.z; sum.w += dl.w;
        }
        if (!touched) continue;                                                                         // no copy moved since `prev`
        const float4 ag = make_float4(sum.x * scale, sum.y * scale, sum.z * scale, sum.w * scale);     // agreed step of this element
#pragma unroll
        for (int p = 0; p < NP; p++) {
            const float4 c = make_float4(ag.x - (snap[p].x - pv.x), ag.y - (snap[p].y - pv.y), ag.z - (snap[p].z - pv.z),
                                         ag.w - (snap[p].w - pv.w));
            if (c.x != 0.f || c.y != 0.f || c.z != 0.f || c.w != 0.f) red_add_v4_sys(T.base[p] + 4 * e, c);
        }
        prev[e] = make_float4(pv.x + ag.x, pv.y + ag.y, pv.z + ag.z, pv.w + ag.w);
    }
}

// ---------------------------------------------------------------- NeuMF over a row-sharded [items, 2f] table
// one warp per sample, lanes over f/4 float4 (f % 4 == 0, f <= 128); item row = [I_mf (f) | I_mlp (f)]
__global__ void __launch_bounds__(256) neumf_gather_peer_kernel(const float *Umf, const float *Umlp, int64_t ldu, PeerTab I, ShardMap sm,
                                                                int64_t ldi, int f, const int32_t *u, const int32_t *it, int64_t n,
                                                                float *x0, int64_t ldx, float *pm, int64_t ldp) {
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (; w < n; w += nw) {
        const int uu = u[w];
        int o, l;
        sm.locate(it[w], o, l);
        const float *row = I.base[o] + (int64_t)l * ldi;
        for (int c = lane * 4; c < f; c += 128) {
            const float4 a = *reinterpret_cast<const float4 *>(Umlp + (int64_t)uu * ldu + c);
            const float4 m1 = *reinterpret_cast<const float4 *>(Umf + (int64_t)uu * ldu + c);
            const float4 m2 = ld_sys_v4(reinterpret_cast<const float4 *>(row + c));
            const float4 b = ld_sys_v4(reinterpret_cast<const float4 *>(row + f + c));
            *reinterpret_cast<float4 *>(x0 + w * ldx + c) = a;
            *reinterpret_cast<float4 *>(x0 + w * ldx + f + c) = b;
            *reinterpret_cast<float4 *>(pm + w * ldp + c) = make_float4(m1.x * m2.x, m1.y * m2.y, m1.z * m2.z, m1.w * m2.w);
        }
    }
}

// dU_mf[u] += dpm * I_mf[i];  dI_mf[i] += dpm * U_mf[u];  dU_mlp[u] += dx0[:f];  dI_mlp[i] += dx0[f:]
// (item-row gradients go into the OWNER's dense gradient shard GI, same [rows, 2f] layout as the item table)
__global__ void __launch_bounds__(256) neumf_scatter_peer_kernel(const float *Umf, int64_t ldu, PeerTab I, PeerTab GI, ShardMap sm,
                                                                 int64_t ldi, int f, const int32_t *u, const int32_t *it, int64_t n,
                                                                 const float *dpm, int64_t ldp, const float *dx0, int64_t ldx,
                                                                 float *dUmf, float *dUmlp) {
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (; w < n; w += nw) {
        const int uu = u[w];
        int o, l;
        sm.locate(it[w], o, l);
        const float *row = I.base[o] + (int64_t)l * ldi;
        float *grow = GI.base[o] + (int64_t)l * ldi;
        for (int c = lane * 4; c < f; c += 128) {
            const float4 g = *reinterpret_cast<const float4 *>(dpm + w * ldp + c);
            const float4 a = *reinterpret_cast<const float4 *>(Umf + (int64_t)uu * ldu + c);
            const float4 b = ld_sys_v4(reinterpret_cast<const float4 *>(row + c));
            red_add_v4(dUmf + (int64_t)uu * ldu + c, make_float4(g.x * b.x, g.y * b.y, g.z * b.z, g.w * b.w));
            red_add_v4_sys(grow + c, make_float4(g.x * a.x, g.y * a.y, g.z * a.z, g.w * a.w));
            red_add_v4(dUmlp + (int64_t)uu * ldu + c, *reinterpret_cast<const float4 *>(dx0 + w * ldx + c));
            red_add_v4_sys(grow + f + c, *reinterpret_cast<const float4 *>(dx0 + w * ldx + f + c));
        }
    }
}

// out[t][0..w) = shard(ids[t])[local(ids[t])][0..w)  — rows of a sharded table into a local buffer (scoring, tests)
__global__ void __launch_bounds__(256) gather_rows_peer_kernel(PeerTab T, ShardMap sm, int64_t ld, const int32_t *ids, int64_t n, int w,
                                                               float *out, int64_t ldo) {
    const int64_t total = n * (w / 4);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = e / (w / 4); const int c = (int)(e - t * (w / 4)) * 4;
        int o, l;
        sm.locate(ids[t], o, l);
        *reinterpret_cast<float4 *>(out + t * ldo + c) = ld_sys_v4(reinterpret_cast<const float4 *>(T.base[o] + (int64_t)l * ld + c));
    }
}

static inline unsigned pgrid(int64_t threads, int per_sm = 8) {
    int64_t g = (threads + 255) / 256; const int64_t cap = (int64_t)sm_count() * per_sm;
    return (unsigned)(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace eb

using namespace eb;

// ---------------------------------------------------------------- memory that peers can map
extern "C" int eb_peer_alloc(size_t bytes, void **dev_ptr) {
    EB_ARG(dev_ptr && bytes > 0, "bad argument");
    void *p = nullptr;
    EB_CUDA(cudaMalloc(&p, bytes));
    cudaError_t e = cudaMemset(p, 0, bytes);
    if (e != cudaSuccess) { cudaFree(p); return set_err(EB_ERR_CUDA, "cudaMemset -> %s", cudaGetErrorString(e)); }
    EB_CUDA(cudaDeviceSynchronize());
    *dev_ptr = p;
    return EB_OK;
}

extern "C" int eb_peer_free(void *dev_ptr) {
    if (dev_ptr) EB_CUDA(cudaFree(dev_ptr));
    return EB_OK;
}

extern "C" int eb_peer_export(const void *dev_ptr, void *handle64_host) {
    EB_ARG(dev_ptr && handle64_host, "null pointer");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    cudaIpcMemHandle_t h;
    EB_CUDA(cudaIpcGetMemHandle(&h, const_cast<void *>(dev_ptr)));
    memcpy(handle64_host, &h, sizeof(h));
    return EB_OK;
}

extern "C" int eb_peer_open(const void *handle64_host, void **dev_ptr) {
    EB_ARG(dev_ptr && handle64_host, "null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64_host, sizeof(h));
    void *p = nullptr;
    EB_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    *dev_ptr = p;
    return EB_OK;
}

extern "C" int eb_peer_close(void *dev_ptr) {
    if (dev_ptr) EB_CUDA(cudaIpcCloseMemHandle(dev_ptr));
    return EB_OK;
}

// ---------------------------------------------------------------- kernels' entry points
extern "C" int eb_table_reconcile_peer_f32(float *const *slice_ptrs, int n_peers, float *prev_slice, int64_t n, float scale,
                                           int max_ctas, void *stream) {
    PeerTab T;
    if (int rc = fill_tab(T, slice_ptrs, n_peers)) return rc;
    EB_ARG(prev_slice && ((uintptr_t)prev_slice % 16) == 0 && n >= 0 && n % 4 == 0, "prev_slice must be 16-byte aligned, n a multiple of 4");
    if (n == 0) return EB_OK;
    const int64_t n4 = n / 4;
    unsigned grid = pgrid(n4, 4);
    if (max_ctas > 0 && grid > (unsigned)max_ctas) grid = (unsigned)max_ctas;
    cudaStream_t st = (cudaStream_t)stream;
    float4 *pv = reinterpret_cast<float4 *>(prev_slice);
    switch (n_peers) {
        case 1: table_reconcile_peer_kernel<1><<<grid, 256, 0, st>>>(T, pv, n4, scale); break;
        case 2: table_reconcile_peer_kernel<2><<<grid, 256, 0, st>>>(T, pv, n4, scale); break;
        case 3: table_reconcile_peer_kernel<3><<<grid, 256, 0, st>>>(T, pv, n4, scale); break;
        case 4: table_reconcile_peer_kernel<4><<<grid, 256, 0, st>>>(T, pv, n4, scale); break;
        case 5: table_reconcile_peer_kernel<5><<<grid, 256, 0, st>>>(T, pv, n4, scale); break;
        case 6: table_reconcile_peer_kernel<6><<<grid, 256, 0, st>>>(T, pv, n4, scale); break;
        case 7: table_reconcile_peer_kernel<7><<<grid, 256, 0, st>>>(T, pv, n4, scale); break;
        default: table_reconcile_peer_kernel<8><<<grid, 256, 0, st>>>(T, pv, n4, scale); break;
    }
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_neumf_gather_peer(const float *Umf, const float *Umlp, int64_t ldu, float *const *I_shards, int n_shards,
                                    int32_t shard_rows, int64_t ldi, int f, const int32_t *u, const int32_t *it, int64_t n, float *x0,
                                    int64_t ldx, float *pm, int64_t ldp, void *stream) {
    PeerTab I;
    if (int rc = fill_tab(I, I_shards, n_shards)) return rc;
    EB_ARG(Umf && Umlp && u && it && x0 && pm && f >= 4 && f % 4 == 0 && f <= 128 && ldu % 4 == 0 && ldi >= 2 * f && ldi % 4 == 0 &&
               ldx % 4 == 0 && ldp % 4 == 0 && shard_rows >= 1,
           "bad argument (f must be a multiple of 4, <= 128; item rows are [mf | mlp], ldi >= 2f)");
    if (n <= 0) return EB_OK;
    neumf_gather_peer_kernel<<<pgrid(n * 32), 256, 0, (cudaStream_t)stream>>>(Umf, Umlp, ldu, I, shard_map(shard_rows), ldi, f, u, it, n, x0,
                                                                               ldx, pm, ldp);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_neumf_scatter_peer(const float *Umf, int64_t ldu, float *const *I_shards, float *const *GI_shards, int n_shards,
                                     int32_t shard_rows, int64_t ldi, int f, const int32_t *u, const int32_t *it, int64_t n,
                                     const float *dpm, int64_t ldp, const float *dx0, int64_t ldx, float *dUmf, float *dUmlp,
                                     void *stream) {
    PeerTab I, GI;
    if (int rc = fill_tab(I, I_shards, n_shards)) return rc;
    if (int rc = fill_tab(GI, GI_shards, n_shards)) return rc;
    EB_ARG(Umf && u && it && dpm && dx0 && dUmf && dUmlp && f >= 4 && f % 4 == 0 && f <= 128 && ldi >= 2 * f && shard_rows >= 1,
           "bad argument");
    if (n <= 0) return EB_OK;
    neumf_scatter_peer_kernel<<<pgrid(n * 32), 256, 0, (cudaStream_t)stream>>>(Umf, ldu, I, GI, shard_map(shard_rows), ldi, f, u, it, n,
                                                                                dpm, ldp, dx0, ldx, dUmf, dUmlp);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

// ---------------------------------------------------------------- batches ordered by owner
// 256-byte rows gathered at random from many peers interleaved arrive far more slowly than the same rows drawn owner by owner
// (a requester-side limit, tools/peer_fanout_probe.py measures it); the same ids GROUPED by owner — every rank starting at
// its right-hand neighbour — keep the links busy.  A batch whose rows live on more than four peers is therefore bucketed by
// owner before the peer kernels see it: a counting sort over <= 64 keys
//     key = ((owner(id1) - rank) mod W) [* W + ((owner(id2) - rank) mod W)]
// (order inside a bucket is arbitrary: the samples of a step are exchangeable).
struct GroupParams {
    const int32_t *a, *b, *c;      // three 32-bit payload arrays that travel together (b, c may be null)
    const int32_t *id1, *id2;      // the arrays holding the row ids (id2 null: one id per element)
    int64_t n;
    int32_t shard_rows;
    int rank, world;
    int32_t *out_a, *out_b, *out_c;
    int32_t *counts, *cursor;      // [64] each
};

__device__ __forceinline__ int group_key(const GroupParams &p, int64_t e) {
    const int w = p.world;
    int o1 = p.id1[e] / p.shard_rows; o1 = o1 >= w ? w - 1 : o1;
    int k = (o1 - p.rank + w) % w;
    if (p.id2) {
        int o2 = p.id2[e] / p.shard_rows; o2 = o2 >= w ? w - 1 : o2;
        k = k * w + (o2 - p.rank + w) % w;
    }
    return k;
}

__global__ void __launch_bounds__(256) group_count_kernel(const GroupParams p) {
    __shared__ int hist[64];
    if (threadIdx.x < 64) hist[threadIdx.x] = 0;
    __syncthreads();
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < p.n; e += (int64_t)gridDim.x * blockDim.x)
        atomicAdd(&hist[group_key(p, e)], 1);
    __syncthreads();
    if (threadIdx.x < 64 && hist[threadIdx.x]) atomicAdd(p.counts + threadIdx.x, hist[threadIdx.x]);
}

__global__ void group_scan_kernel(const GroupParams p) {
    if (threadIdx.x == 0) {
        int run = 0;
        for (int k = 0; k < 64; k++) { p.cursor[k] = run; run += p.counts[k]; }
    }
}

constexpr int GROUP_CHUNK = 2048;      // elements per block pass: one global reservation per key and chunk

__global__ void __launch_bounds__(256) group_scatter_kernel(const GroupParams p) {
    __shared__ int hist[64], base[64];
    const int64_t n_chunks = (p.n + GROUP_CHUNK - 1) / GROUP_CHUNK;
    for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
        __syncthreads();
        if (threadIdx.x < 64) hist[threadIdx.x] = 0;
        __syncthreads();
        int key[GROUP_CHUNK / 256], slot[GROUP_CHUNK / 256];
#pragma unroll
        for (int j = 0; j < GROUP_CHUNK / 256; j++) {
            const int64_t e = ch * GROUP_CHUNK + j * 256 + threadIdx.x;
            key[j] = e < p.n ? group_key(p, e) : -1;
            slot[j] = key[j] >= 0 ? atomicAdd(&hist[key[j]], 1) : 0;
        }
        __syncthreads();
        if (threadIdx.x < 64) base[threadIdx.x] = hist[threadIdx.x] ? atomicAdd(p.cursor + threadIdx.x, hist[threadIdx.x]) : 0;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < GROUP_CHUNK / 256; j++) {
            const int64_t e = ch * GROUP_CHUNK + j * 256 + threadIdx.x;
            if (key[j] < 0) continue;
            const int64_t o = (int64_t)base[key[j]] + slot[j];
            p.out_a[o] = p.a[e];
            if (p.b) p.out_b[o] = p.b[e];
            if (p.c) p.out_c[o] = p.c[e];
        }
    }
}

extern "C" int eb_group_by_owner_i32(const int32_t *a, const int32_t *b, const int32_t *c, int key1, int key2, int64_t n,
                                     int32_t shard_rows, int rank, int world, int32_t *out_a, int32_t *out_b, int32_t *out_c,
                                     int32_t *work, void *stream) {
    EB_ARG(a && out_a && work && n >= 0 && n < (1ll << 31), "null pointer or bad size");
    EB_ARG((b == nullptr) == (out_b == nullptr) && (c == nullptr) == (out_c == nullptr), "payload arrays and outputs must match");
    EB_ARG(shard_rows >= 1 && world >= 1 && world <= 8 && rank >= 0 && rank < world, "bad shard geometry (world <= 8)");
    const int32_t *arr[3] = {a, b, c};
    EB_ARG(key1 >= 0 && key1 <= 2 && arr[key1] && key2 >= -1 && key2 <= 2 && (key2 < 0 || arr[key2]), "key1 / key2 name the id arrays (0..2)");
    if (n == 0) return EB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    EB_CUDA(cudaMemsetAsync(work, 0, 128 * sizeof(int32_t), st));
    GroupParams p{a, b, c, arr[key1], key2 >= 0 ? arr[key2] : nullptr, n, shard_rows, rank, world, out_a, out_b, out_c, work, work + 64};
    group_count_kernel<<<pgrid(n), 256, 0, st>>>(p);
    group_scan_kernel<<<1, 32, 0, st>>>(p);
    const int64_t n_chunks = (n + GROUP_CHUNK - 1) / GROUP_CHUNK;
    const int64_t cap = (int64_t)sm_count() * 8;
    group_scatter_kernel<<<(unsigned)(n_chunks < cap ? n_chunks : cap), 256, 0, st>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

extern "C" int eb_gather_rows_peer_f32(float *const *shards, int n_shards, int32_t shard_rows, int64_t ld, const int32_t *ids, int64_t n,
                                       int width, float *out, int64_t ldo, void *stream) {
    PeerTab T;
    if (int rc = fill_tab(T, shards, n_shards)) return rc;
    EB_ARG(ids && out && n >= 0 && width >= 4 && width % 4 == 0 && ld >= width && ldo >= width && ld % 4 == 0 && ldo % 4 == 0 &&
               shard_rows >= 1,
           "bad argument (width, ld, ldo must be multiples of 4)");
    if (n == 0) return EB_OK;
    gather_rows_peer_kernel<<<pgrid(n * (width / 4)), 256, 0, (cudaStream_t)stream>>>(T, shard_map(shard_rows), ld, ids, n, width, out, ldo);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
