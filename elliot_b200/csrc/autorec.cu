// autorec.cu — the decoder of UserAutoRec / ItemAutoRec (neural/UserAutoRec/userautorec_model.py:92-107,
// neural/ItemAutoRec/itemautorec_model.py:89-104) over the observed entries of a batch.
//
//   eb_autorec_decoder_f32   one training step's decoder and its backward.  The reference's loss reads
//                            act(o) * sign(x), so only a row's train entries carry a gradient: for each entry p of row
//                            rows[b] (item or user i = indices[p], x = values[p])
//                              o = h_b . W2[i] + b2[i];  r = act(o);  e = x - r;  loss += scale e^2 (fp64)
//                              g = -2 scale e act'(o);  dW2[i] += g h_b;  db2[i] += g;  dh_b += g W2[i]
//                            then dpre1_b = dh_b * h_b * (1 - h_b) (the encoder's sigmoid).
//
// Each entry's W2 row is loaded once into registers: the dot and the dh accumulation read the same load.  A lane group
// of LPE lanes (KC float4 chunks per lane) takes one entry at a time; a CTA takes a SEGMENT of at most SEG entries of
// one row, so a long row (an ItemAutoRec row is an item's column: up to ~67 000 entries at the ML-20M shape) is spread
// over many CTAs of a persistent grid instead of holding one SM.  dh and the loss are combined in a fixed order —
// the entries of a group in index order, the groups of a CTA in group order, the segments of a row in segment order —
// so they do not depend on scheduling; only the dW2 / db2 reductions (red.global.add) may differ in the last bits.
#include "common.cuh"

namespace eb {

constexpr int AR_THREADS = 256;
constexpr int AR_EPG = 32;                      // entries per lane group per segment: SEG = (AR_THREADS / LPE) * AR_EPG

struct ArShape {
    int G, LPE, KC, seg;                        // float4 chunks per row, lanes per entry, chunks per lane, entries per segment
};

static ArShape ar_shape(int H) {
    ArShape s;
    s.G = H / 4;
    if (s.G <= 32) {
        s.KC = 1;
        s.LPE = 1;
        while (s.LPE < s.G) s.LPE <<= 1;
    } else {
        s.LPE = 32;
        s.KC = s.G <= 64 ? 2 : (s.G <= 128 ? 4 : 8);
    }
    s.seg = (AR_THREADS / s.LPE) * AR_EPG;
    return s;
}

struct ArParams {
    const int64_t *indptr;
    const int32_t *indices;
    const float *values;
    const int32_t *rows;
    int64_t B;
    const float *h;
    int64_t ldh;
    const float *W2, *b2;
    int H, act, LPE, seg;
    float scale;
    float *dW2, *db2, *dpre1;
    int64_t ldd;
    double *loss;
    // workspace
    int64_t *seg_off;          // [B + 1] first segment of each row (exclusive prefix of ceil(len / seg))
    int64_t *part_off;         // [B + 1] first dh partial slot of each row split over more than one segment
    double *loss_part;         // [seg_cap] one loss partial per segment
    float *part;               // [part_cap][H] dh partials of split rows
    int64_t seg_cap, part_cap;
};

// one CTA: both prefixes over the batch's rows, chunks of consecutive rows per thread, then a scan over the threads
__global__ void __launch_bounds__(1024) autorec_scan_kernel(const ArParams p) {
    __shared__ int64_t s_seg[1024], s_part[1024];
    const int64_t per = (p.B + blockDim.x - 1) / blockDim.x;
    const int64_t b0 = min((int64_t)threadIdx.x * per, p.B), b1 = min(b0 + per, p.B);
    int64_t ns = 0, np = 0;
    for (int64_t b = b0; b < b1; b++) {
        const int r = p.rows[b];
        const int64_t n = (p.indptr[r + 1] - p.indptr[r] + p.seg - 1) / p.seg;
        ns += n;
        np += n > 1 ? n : 0;
    }
    s_seg[threadIdx.x] = ns; s_part[threadIdx.x] = np;
    __syncthreads();
    for (int o = 1; o < (int)blockDim.x; o <<= 1) {            // inclusive Hillis-Steele scan
        const int64_t a = threadIdx.x >= (unsigned)o ? s_seg[threadIdx.x - o] : 0;
        const int64_t c = threadIdx.x >= (unsigned)o ? s_part[threadIdx.x - o] : 0;
        __syncthreads();
        s_seg[threadIdx.x] += a; s_part[threadIdx.x] += c;
        __syncthreads();
    }
    ns = s_seg[threadIdx.x] - ns; np = s_part[threadIdx.x] - np;
    for (int64_t b = b0; b < b1; b++) {
        const int r = p.rows[b];
        const int64_t n = (p.indptr[r + 1] - p.indptr[r] + p.seg - 1) / p.seg;
        p.seg_off[b] = ns; p.part_off[b] = np;
        ns += n;
        np += n > 1 ? n : 0;
    }
    if (threadIdx.x == blockDim.x - 1) { p.seg_off[p.B] = ns; p.part_off[p.B] = np; }
}

__device__ __forceinline__ float ar_dot4(float4 a, float4 b, float s) {
    s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s); return fmaf(a.w, b.w, s);
}

// persistent grid over the batch's segments; KC float4 chunks per lane (chunk c = lane + LPE k of the row)
template <int KC>
__global__ void __launch_bounds__(AR_THREADS, 2) autorec_decoder_kernel(const ArParams p) {
    __shared__ float4 s_dh[AR_THREADS * KC];                  // [group][G] dh partials (n_groups * G <= AR_THREADS * KC)
    __shared__ double s_loss[AR_THREADS];
    const int LPE = p.LPE, G = p.H / 4, n_groups = AR_THREADS / LPE;
    const int grp = threadIdx.x / LPE, lane = threadIdx.x % LPE;
    const int64_t n_seg = min(p.seg_off[p.B], p.seg_cap);
    for (int64_t seg = blockIdx.x; seg < n_seg; seg += gridDim.x) {
        int64_t lo = 0, hi = p.B;                               // the row b with seg_off[b] <= seg < seg_off[b + 1]
        while (hi - lo > 1) {
            const int64_t mid = (lo + hi) >> 1;
            if (p.seg_off[mid] <= seg) lo = mid; else hi = mid;
        }
        const int64_t b = lo, k = seg - p.seg_off[b], nseg = p.seg_off[b + 1] - p.seg_off[b];
        const int r = p.rows[b];
        const int64_t end = p.indptr[r + 1];
        const int64_t p0 = p.indptr[r] + k * p.seg, p1 = min(p0 + p.seg, end);
        const float *hb = p.h + b * p.ldh;
        float4 h[KC], dh[KC];
#pragma unroll
        for (int q = 0; q < KC; q++) {
            const int c = lane + LPE * q;
            h[q] = c < G ? *reinterpret_cast<const float4 *>(hb + 4 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
            dh[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        double lsum = 0.0;
        // every lane runs the same number of passes (the shuffles need the whole warp); a group past the end idles
        for (int64_t base = p0; base < p1; base += n_groups) {
            const int64_t e = base + grp;
            const bool valid = e < p1;
            const int64_t i = valid ? __ldg(p.indices + e) : 0;
            const float x = valid ? __ldg(p.values + e) : 0.f;
            const float *wr = p.W2 + i * p.H;
            float4 w[KC];
            float s = 0.f;
#pragma unroll
            for (int q = 0; q < KC; q++) {
                const int c = lane + LPE * q;
                w[q] = valid && c < G ? __ldg(reinterpret_cast<const float4 *>(wr + 4 * c)) : make_float4(0.f, 0.f, 0.f, 0.f);
                s = ar_dot4(w[q], h[q], s);
            }
            for (int o = LPE >> 1; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (!valid) continue;
            const float out = s + __ldg(p.b2 + i);
            const float rec = p.act ? 1.f / (1.f + expf(-out)) : out;
            const float err = x - rec;
            const float g = -2.f * p.scale * err * (p.act ? rec * (1.f - rec) : 1.f);
#pragma unroll
            for (int q = 0; q < KC; q++) {
                const int c = lane + LPE * q;
                if (c < G) {
                    red_add_v4(p.dW2 + i * p.H + 4 * c, make_float4(g * h[q].x, g * h[q].y, g * h[q].z, g * h[q].w));
                    dh[q].x = fmaf(g, w[q].x, dh[q].x); dh[q].y = fmaf(g, w[q].y, dh[q].y);
                    dh[q].z = fmaf(g, w[q].z, dh[q].z); dh[q].w = fmaf(g, w[q].w, dh[q].w);
                }
            }
            if (lane == 0) {
                red_add_f32(p.db2 + i, g);
                lsum += (double)err * (double)err;
            }
        }
#pragma unroll
        for (int q = 0; q < KC; q++) {
            const int c = lane + LPE * q;
            if (c < G) s_dh[grp * G + c] = dh[q];
        }
        if (lane == 0) s_loss[grp] = lsum;
        __syncthreads();
        const int t = threadIdx.x;
        if (t < G) {
            float4 a = s_dh[t];
            for (int j = 1; j < n_groups; j++) {
                const float4 v = s_dh[j * G + t];
                a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
            }
            if (nseg == 1) {
                const float4 hv = *reinterpret_cast<const float4 *>(hb + 4 * t);
                *reinterpret_cast<float4 *>(p.dpre1 + b * p.ldd + 4 * t) =
                    make_float4(a.x * hv.x * (1.f - hv.x), a.y * hv.y * (1.f - hv.y), a.z * hv.z * (1.f - hv.z),
                                a.w * hv.w * (1.f - hv.w));
            } else if (p.part_off[b] + k < p.part_cap) {
                *reinterpret_cast<float4 *>(p.part + (p.part_off[b] + k) * p.H + 4 * t) = a;
            }
        }
        if (t == 0) {
            double l = 0.0;
            for (int j = 0; j < n_groups; j++) l += s_loss[j];
            p.loss_part[seg] = l;
        }
        __syncthreads();
    }
}

// rows over the grid: an empty row gets dpre1 = 0, a split row the sum of its segments' partials in segment order; CTA 0
// first adds scale times the sum of the segments' loss partials (fixed order) to *loss
__global__ void __launch_bounds__(256) autorec_finish_kernel(const ArParams p) {
    const int G = p.H / 4;
    if (blockIdx.x == 0) {
        __shared__ double sl[256];
        const int64_t n_seg = min(p.seg_off[p.B], p.seg_cap);
        double s = 0.0;
        for (int64_t j = threadIdx.x; j < n_seg; j += blockDim.x) s += p.loss_part[j];
        sl[threadIdx.x] = s;
        __syncthreads();
        for (int w = 128; w >= 1; w >>= 1) {
            if ((int)threadIdx.x < w) sl[threadIdx.x] += sl[threadIdx.x + w];
            __syncthreads();
        }
        if (threadIdx.x == 0) *p.loss += (double)p.scale * sl[0];
    }
    for (int64_t b = blockIdx.x; b < p.B; b += gridDim.x) {
        const int64_t nseg = p.seg_off[b + 1] - p.seg_off[b];
        if (nseg == 1) continue;
        for (int t = threadIdx.x; t < G; t += blockDim.x) {
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int64_t k = 0; k < nseg && p.part_off[b] + k < p.part_cap; k++) {
                const float4 v = *reinterpret_cast<const float4 *>(p.part + (p.part_off[b] + k) * p.H + 4 * t);
                a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
            }
            const float4 hv = *reinterpret_cast<const float4 *>(p.h + b * p.ldh + 4 * t);
            *reinterpret_cast<float4 *>(p.dpre1 + b * p.ldd + 4 * t) =
                make_float4(a.x * hv.x * (1.f - hv.x), a.y * hv.y * (1.f - hv.y), a.z * hv.z * (1.f - hv.z),
                            a.w * hv.w * (1.f - hv.w));
        }
    }
}

struct ArLayout {
    size_t seg_off, part_off, loss_part, part, total;
    int64_t seg_cap, part_cap;
};

// a batch of B rows holding at most max_entries entries: segments <= B + max_entries / seg, and a row split over n > 1
// segments holds more than (n - 1) seg >= n seg / 2 entries, so split rows' segments <= 2 max_entries / seg
static ArLayout ar_layout(int64_t B, int H, int64_t max_entries) {
    const ArShape s = ar_shape(H);
    ArLayout L;
    L.seg_cap = B + max_entries / s.seg + 1;
    L.part_cap = 2 * max_entries / s.seg + 1;
    size_t off = 0;
    L.seg_off = off; off += align_up(sizeof(int64_t) * (size_t)(B + 1));
    L.part_off = off; off += align_up(sizeof(int64_t) * (size_t)(B + 1));
    L.loss_part = off; off += align_up(sizeof(double) * (size_t)L.seg_cap);
    L.part = off; off += align_up(sizeof(float) * (size_t)L.part_cap * H);
    L.total = off;
    return L;
}

template <int KC>
static int ar_launch(const ArParams &p, cudaStream_t st) {
    static int per_sm = 0;
    if (per_sm == 0) {
        EB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, autorec_decoder_kernel<KC>, AR_THREADS, 0));
        if (per_sm < 1) per_sm = 1;
    }
    autorec_decoder_kernel<KC><<<(unsigned)(sm_count() * per_sm), AR_THREADS, 0, st>>>(p);
    return EB_OK;
}

}  // namespace eb

using namespace eb;

extern "C" size_t eb_autorec_decoder_workspace_bytes(int64_t B, int H, int64_t max_entries) {
    if (H < 4 || H > 1024 || H % 4 || B < 0 || max_entries < 0) return 0;
    return ar_layout(B < 1 ? 1 : B, H, max_entries).total;
}

extern "C" int eb_autorec_decoder_f32(const int64_t *indptr, const int32_t *indices, const float *values, const int32_t *rows,
                                      int64_t B, int64_t max_entries, const float *h, int64_t ldh, const float *W2,
                                      const float *b2, int H, int act, float scale, float *dW2, float *db2, float *dpre1,
                                      int64_t ldd, double *loss, void *workspace, size_t workspace_bytes, void *stream) {
    EB_ARG(indptr && indices && values && rows && h && W2 && b2 && dW2 && db2 && dpre1 && loss, "null pointer");
    EB_ARG(H >= 4 && H <= 1024 && H % 4 == 0 && ldh >= H && ldh % 4 == 0 && ldd >= H && ldd % 4 == 0,
           "H=%d must be a multiple of 4 in [4, 1024], ldh and ldd multiples of 4 >= H", H);
    EB_ARG(((uintptr_t)h % 16) == 0 && ((uintptr_t)W2 % 16) == 0 && ((uintptr_t)dW2 % 16) == 0 && ((uintptr_t)dpre1 % 16) == 0,
           "16-byte alignment");
    EB_ARG(act == 0 || act == 1, "act=%d must be 0 (linear) or 1 (sigmoid)", act);
    EB_ARG(max_entries >= 0, "max_entries=%lld", (long long)max_entries);
    if (B <= 0) return EB_OK;
    const ArLayout L = ar_layout(B, H, max_entries);
    if (!workspace || workspace_bytes < L.total)
        return set_err(EB_ERR_WORKSPACE, "workspace %zu < required %zu", workspace_bytes, L.total);
    const ArShape s = ar_shape(H);
    char *ws = (char *)workspace;
    ArParams p;
    p.indptr = indptr; p.indices = indices; p.values = values; p.rows = rows; p.B = B;
    p.h = h; p.ldh = ldh; p.W2 = W2; p.b2 = b2; p.H = H; p.act = act; p.LPE = s.LPE; p.seg = s.seg; p.scale = scale;
    p.dW2 = dW2; p.db2 = db2; p.dpre1 = dpre1; p.ldd = ldd; p.loss = loss;
    p.seg_off = (int64_t *)(ws + L.seg_off); p.part_off = (int64_t *)(ws + L.part_off);
    p.loss_part = (double *)(ws + L.loss_part); p.part = (float *)(ws + L.part);
    p.seg_cap = L.seg_cap; p.part_cap = L.part_cap;
    cudaStream_t st = (cudaStream_t)stream;
    autorec_scan_kernel<<<1, 1024, 0, st>>>(p);
    int rc;
    switch (s.KC) {
        case 1: rc = ar_launch<1>(p, st); break;
        case 2: rc = ar_launch<2>(p, st); break;
        case 4: rc = ar_launch<4>(p, st); break;
        default: rc = ar_launch<8>(p, st); break;
    }
    if (rc != EB_OK) return rc;
    autorec_finish_kernel<<<capped_grid(B * 256), 256, 0, st>>>(p);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
