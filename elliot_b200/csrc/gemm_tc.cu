// gemm_tc.cu — general bf16 tensor-core GEMM for the dense layers of MultiVAE / NeuMF.
//
//   C[M][N] (fp32, row stride ldc) = A[M][K] * B[N][K]^T  (+ bias[N]) (optional tanh / relu)
//
// Both operands are bf16, K-major (row-major with K contiguous), which is what the Keras Dense
// layers of the reference need once weights are kept as [out][in]
// (multi_vae_model.py:44-53,72-78; neural_matrix_factorization_model.py:57-70).  Backward GEMMs
// read MN-major operands directly (A_MN / B_MN below) or use transposed copies (tc_transpose_kernel).
// Structure (PTX wrappers shared with score_topk_tc.cu through tc_ptx.cuh): persistent CTAs, warp 8 TMA producer
// (4-stage ring of {A 128x64, B 128x64} bf16 tiles, 128B swizzle), warpgroups 0 and 1 the consumers: each issues
// wgmma.m64n128k16 for its 64 rows of the 128 x 128 tile (fp32 accumulators in registers, one k-block in flight while the
// previous stage is released) and writes its rows (bias / activation / split-K reduction) straight from the registers.
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace eb {

constexpr int G_BM = 128, G_BN = 128, G_BK = 64, G_STAGES = 4, G_THREADS = 288;
constexpr int G_STAGE_BYTES = (G_BM + G_BN) * G_BK * 2;      // 32 KB
constexpr int G_SMEM = G_STAGES * G_STAGE_BYTES + 256;

struct GemmParams {
    float *C;
    int64_t ldc;
    const float *bias;   // [N] or null
    int M, N, K;
    int act;             // 0 none, 1 tanh, 2 relu
    float alpha;         // C = alpha * (A B^T) + bias, then activation
    int splits;          // split-K factor: > 1 -> each work item covers a K range and STORES its partial tile into ws
    float *ws;           // split-K partials [splits][M][N], summed into C in split order by splitk_reduce_kernel
    __nv_bfloat16 *Cb;   // optional second output: the same values as bf16 rows (row stride ldcb) — the next layer's operand copy
    int64_t ldcb;
};

__device__ __forceinline__ float g_act(float x, int act) { return act == 1 ? tanhf(x) : (act == 2 ? fmaxf(x, 0.f) : x); }

// A_MN / B_MN: the operand is given with its M (resp. N) index contiguous — a [K][M] row-major matrix — instead of K-major.
// TMA then fetches {64 m, 64 k} boxes (two per 128-wide tile) whose 128-byte rows are 64 consecutive M elements, and the
// shared-memory descriptor says "MN-major" (gmma_desc_sw128_mn; wgmma transposes the operand on the fly).  The weight-gradient
// GEMMs dW = dY^T . X (K = the batch) and dX = dY . W with W kept [K][N] read their operands this way, so no transposed
// bf16 copies of activations or weights are ever written.
template <bool A_MN, bool B_MN>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
    extern __shared__ __align__(1024) uint8_t sm[];
    uint64_t *bars = reinterpret_cast<uint64_t *>(sm + G_STAGES * G_STAGE_BYTES);
    const uint32_t bar0 = smem_u32(bars);
    auto FULL = [&](int s) { return bar0 + 8u * (uint32_t)s; };
    auto EMPTY = [&](int s) { return bar0 + 8u * (uint32_t)(G_STAGES + s); };
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // provably warp-uniform (see elect_one_sync)
    const int lane = threadIdx.x & 31;
    const int tiles_m = (p.M + G_BM - 1) / G_BM, tiles_n = (p.N + G_BN - 1) / G_BN;
    const int k_blocks_all = (p.K + G_BK - 1) / G_BK;
    const int kb_per = (k_blocks_all + p.splits - 1) / p.splits;     // k-blocks per split (the last may be shorter)
    const int n_tiles = tiles_m * tiles_n * p.splits;               // work items: (tile, split)

    if (threadIdx.x == 0) {
        if (smem_u32(sm) & 1023u) __trap();
        for (int s = 0; s < G_STAGES; s++) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), 2); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (elect_one_sync()) {
            tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
            int s = 0; uint32_t ph = 0;
            for (int work = blockIdx.x; work < n_tiles; work += gridDim.x) {
                const int tile = work / p.splits, split = work % p.splits;
                const int tm = tile / tiles_n, tn = tile % tiles_n;
                const int kb0 = split * kb_per, kb1 = min(kb0 + kb_per, k_blocks_all);
                for (int kb = kb0; kb < kb1; kb++) {
                    mbar_wait(EMPTY(s), ph ^ 1);
                    mbar_expect_tx(FULL(s), G_STAGE_BYTES);
                    const uint32_t a_dst = smem_u32(sm + s * G_STAGE_BYTES), b_dst = a_dst + G_BM * G_BK * 2;
                    if (A_MN) {
                        tma_load_2d(a_dst, &tmA, FULL(s), tm * G_BM, kb * G_BK);
                        tma_load_2d(a_dst + 64 * G_BK * 2, &tmA, FULL(s), tm * G_BM + 64, kb * G_BK);
                    } else {
                        tma_load_2d(a_dst, &tmA, FULL(s), kb * G_BK, tm * G_BM);
                    }
                    if (B_MN) {
                        tma_load_2d(b_dst, &tmB, FULL(s), tn * G_BN, kb * G_BK);
                        tma_load_2d(b_dst + 64 * G_BK * 2, &tmB, FULL(s), tn * G_BN + 64, kb * G_BK);
                    } else {
                        tma_load_2d(b_dst, &tmB, FULL(s), kb * G_BK, tn * G_BN);
                    }
                    if (++s == G_STAGES) { s = 0; ph ^= 1; }
                }
            }
        }
    } else if (warp < 8) {
        // consumer warpgroup h computes rows [64 h, 64 h + 64) of every 128 x 128 tile
        const int h = warp >> 2, wq = warp & 3;
        int s = 0; uint32_t ph = 0;
        float acc[64];
        for (int work = blockIdx.x; work < n_tiles; work += gridDim.x) {
            const int tile = work / p.splits, split = work % p.splits;
            const int tm = tile / tiles_n, tn = tile % tiles_n;
            const int kb0 = split * kb_per, kb1 = min(kb0 + kb_per, k_blocks_all);
            if (kb0 >= kb1) continue;                                   // trailing split without k-blocks: nothing to add
            int prev = -1;
            for (int kb = kb0; kb < kb1; kb++) {
                mbar_wait(FULL(s), ph);
                const uint32_t a_addr = smem_u32(sm + s * G_STAGE_BYTES) + (uint32_t)h * (64 * G_BK * 2), b_addr = smem_u32(sm + s * G_STAGE_BYTES) + G_BM * G_BK * 2;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; k++)
                    wgmma_m64n128k16<A_MN ? 1 : 0, B_MN ? 1 : 0>(
                        acc, A_MN ? gmma_desc_sw128_mn(a_addr + k * 2048) : gmma_desc_sw128(a_addr + k * 32),
                        B_MN ? gmma_desc_sw128_mn(b_addr + k * 2048) : gmma_desc_sw128(b_addr + k * 32), ((kb - kb0) | k) != 0);
                wgmma_commit();
                wgmma_wait<1>();                                        // the previous k-block's MMAs have retired
                if (prev >= 0 && threadIdx.x % 128 == 0) mbar_arrive(EMPTY(prev));
                prev = s;
                if (++s == G_STAGES) { s = 0; ph ^= 1; }
            }
            wgmma_wait<0>();
            wgmma_acc_fence<64>(acc);
            if (threadIdx.x % 128 == 0) mbar_arrive(EMPTY(prev));
            const int r0 = tm * G_BM + h * 64 + wq * 16 + (lane >> 2);
            const bool pair_ok = (p.ldc & 1) == 0 && ((reinterpret_cast<uintptr_t>(p.C) & 7) == 0);
            const bool pair_okb = p.Cb && (p.ldcb & 1) == 0;
#pragma unroll
            for (int half = 0; half < 2; half++) {
                const int row = r0 + 8 * half;
                if (row >= p.M) continue;
                float *crow = p.C + (int64_t)row * p.ldc;
#pragma unroll
                for (int j = 0; j < 16; j++) {
                    const int col = tn * G_BN + 8 * j + 2 * (lane & 3);
                    if (col >= p.N) continue;
                    float x0 = p.alpha * acc[4 * j + 2 * half], x1 = p.alpha * acc[4 * j + 2 * half + 1];
                    const bool two = col + 1 < p.N;
                    if (p.splits > 1) {
                        float *wrow = p.ws + ((int64_t)split * p.M + row) * p.N;
                        wrow[col] = x0;
                        if (two) wrow[col + 1] = x1;
                        continue;
                    }
                    if (p.bias) { x0 += __ldg(p.bias + col); if (two) x1 += __ldg(p.bias + col + 1); }
                    x0 = g_act(x0, p.act); x1 = g_act(x1, p.act);
                    if (two && pair_ok) *reinterpret_cast<float2 *>(crow + col) = make_float2(x0, x1);
                    else { crow[col] = x0; if (two) crow[col + 1] = x1; }
                    if (p.Cb) {                                         // bf16 copy of the same values, straight from the registers
                        __nv_bfloat16 *cb = p.Cb + (int64_t)row * p.ldcb + col;
                        if (two && pair_okb) *reinterpret_cast<__nv_bfloat162 *>(cb) = __floats2bfloat162_rn(x0, x1);
                        else { cb[0] = __float2bfloat16_rn(x0); if (two) cb[1] = __float2bfloat16_rn(x1); }
                    }
                }
            }
        }
    }
}

// C[r][c] = sum_s ws[s][r][c], s = 0, 1, ... in order: the split-K sum is the same bits on every run
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float *__restrict__ ws, int splits, int M, int N, float *__restrict__ C,
                                                            int64_t ldc) {
    const int64_t total = (int64_t)M * N;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        float t = ws[e];
        for (int s = 1; s < splits; s++) t += ws[(int64_t)s * total + e];
        const int64_t r = e / N;
        C[r * ldc + (e - r * N)] = t;
    }
}

// fp32 [R][C] (row stride ld) -> bf16 [R][dst_ld] (same layout, zero padded columns)
__global__ void __launch_bounds__(256) tc_convert_kernel2(const float *__restrict__ src, int R, int C, int64_t ld,
                                                          __nv_bfloat16 *__restrict__ dst, int64_t dst_ld) {
    const int64_t total = (int64_t)R * dst_ld;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / dst_ld; const int c = (int)(e - r * dst_ld);
        dst[e] = __float2bfloat16_rn(c < C ? src[r * ld + c] : 0.f);
    }
}
// fp32 [R][C] -> bf16 [C][dst_ld] (transposed; columns r >= R zero padded); 32x32 tiles through shared memory
__global__ void __launch_bounds__(256) tc_transpose_kernel(const float *__restrict__ src, int R, int C, int64_t ld,
                                                           __nv_bfloat16 *__restrict__ dst, int64_t dst_ld) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8 threads
    for (int j = ty; j < 32; j += 8) {
        const int r = r0 + j, c = c0 + tx;
        tile[j][tx] = (r < R && c < C) ? src[(int64_t)r * ld + c] : 0.f;
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        const int c = c0 + j, r = r0 + tx;
        if (c < C && r < dst_ld) dst[(int64_t)c * dst_ld + r] = __float2bfloat16_rn(tile[tx][j]);
    }
}

typedef CUresult (*GEncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                              const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// mn = false: operand [rows][K] (K contiguous), boxes {64 k, box_rows}; mn = true: operand [K][rows] (rows contiguous), boxes {64 rows, 64 k}
static int g_make_map(CUtensorMap *m, const void *base, uint64_t rows, uint64_t K, uint64_t ld_elems, uint32_t box_rows, bool mn = false) {
    static GEncodeFn enc = nullptr;
    if (!enc) {
        void *fp = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return set_err(EB_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
        enc = (GEncodeFn)fp;
    }
    cuuint64_t dims[2] = {(cuuint64_t)(mn ? rows : K), (cuuint64_t)(mn ? K : rows)};
    cuuint64_t strides[1] = {(cuuint64_t)ld_elems * 2};
    cuuint32_t box[2] = {64, mn ? (cuuint32_t)G_BK : box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_err(EB_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return EB_OK;
}

}  // namespace eb

using namespace eb;

extern "C" int eb_convert_bf16(const float *src, int rows, int cols, int64_t ld, void *dst_bf16, int64_t dst_ld, int transpose,
                               void *stream) {
    EB_ARG(src && dst_bf16 && rows >= 1 && cols >= 1 && ld >= cols, "bad argument");
    EB_ARG(dst_ld % 8 == 0 && dst_ld >= (transpose ? rows : cols), "dst_ld must be a multiple of 8 and cover the row");
    cudaStream_t st = (cudaStream_t)stream;
    if (!transpose) {
        int64_t grid = ((int64_t)rows * dst_ld + 255) / 256; const int64_t cap = (int64_t)sm_count() * 8; if (grid > cap) grid = cap;
        tc_convert_kernel2<<<(unsigned)grid, 256, 0, st>>>(src, rows, cols, ld, (__nv_bfloat16 *)dst_bf16, dst_ld);
    } else {
        dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((dst_ld + 31) / 32));
        tc_transpose_kernel<<<grid, 256, 0, st>>>(src, rows, cols, ld, (__nv_bfloat16 *)dst_bf16, dst_ld);
    }
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}

static int gemm_bf16(const void *A_bf16, int64_t lda, bool a_mn, const void *B_bf16, int64_t ldb, bool b_mn, float *C, int64_t ldc,
                     int M, int N, int K, const float *bias, float alpha, int act, void *ws, size_t ws_bytes, void *stream,
                     void *C_bf16 = nullptr, int64_t ldcb = 0) {
    EB_ARG(A_bf16 && B_bf16 && C, "null pointer");
    EB_ARG(M >= 1 && N >= 1 && K >= 1 && lda >= (a_mn ? M : K) && ldb >= (b_mn ? N : K) && ldc >= N, "bad shape M=%d N=%d K=%d", M, N, K);
    EB_ARG(lda % 8 == 0 && ldb % 8 == 0, "lda/ldb must be multiples of 8 bf16 (16-byte TMA strides)");
    EB_ARG(((uintptr_t)A_bf16 % 16) == 0 && ((uintptr_t)B_bf16 % 16) == 0, "operands must be 16-byte aligned");
    EB_ARG(act >= 0 && act <= 2, "act must be 0 (none), 1 (tanh) or 2 (relu)");
    EB_ARG(!C_bf16 || (ldcb >= N && ldcb % 8 == 0 && ((uintptr_t)C_bf16 % 8) == 0), "bf16 second output: ldcb must be a multiple of 8 covering N");
    CUtensorMap ma, mb;
    if (int rc = g_make_map(&ma, A_bf16, (uint64_t)M, (uint64_t)K, (uint64_t)lda, G_BM, a_mn)) return rc;
    if (int rc = g_make_map(&mb, B_bf16, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, G_BN, b_mn)) return rc;
    const int n_out_tiles = ((M + G_BM - 1) / G_BM) * ((N + G_BN - 1) / G_BN);
    const int k_blocks = (K + G_BK - 1) / G_BK;
    // split-K: few output tiles with a long K (dh2 = dlogits . W4: 20 tiles, K = 26 744) leave most SMs idle and each
    // busy CTA load-latency bound; split the K range over the idle SMs, store the partial tiles into the caller's workspace
    // and sum them in split order (bit-reproducible: a run-to-run change in the last bits would move bf16 operand copies
    // of the result by a whole bf16 ulp).  No workspace, or EB_GEMM_SPLITK=0: every GEMM single-pass.
    static const bool splitk_off = [] { const char *e = getenv("EB_GEMM_SPLITK"); return e && e[0] == '0'; }();
    int splits = 1;
    if (!splitk_off && ws && !bias && act == 0 && !C_bf16 && n_out_tiles * 2 <= sm_count() && k_blocks >= 16) {
        splits = sm_count() / n_out_tiles;
        if (splits > k_blocks / 8) splits = k_blocks / 8;           // at least 8 k-blocks per work item
        if (splits < 1) splits = 1;
        const int per = (k_blocks + splits - 1) / splits;
        splits = (k_blocks + per - 1) / per;                         // no empty trailing splits
    }
    if (splits > 1 && ws_bytes < (size_t)splits * M * N * sizeof(float))   // splits * M * N <= sm_count * G_BM * G_BN always
        return set_err(EB_ERR_WORKSPACE, "split-K workspace too small: need %zu bytes", (size_t)splits * M * N * sizeof(float));
    GemmParams p{C, ldc, bias, M, N, K, act, alpha, splits, (float *)ws, (__nv_bfloat16 *)C_bf16, ldcb};
    const int n_tiles = n_out_tiles * splits;
    int grid = sm_count();
    if (grid > n_tiles) grid = n_tiles;
#define EB_GEMM_LAUNCH(AM, BM)                                                                                        \
    do {                                                                                                              \
        EB_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<AM, BM>, cudaFuncAttributeMaxDynamicSharedMemorySize, G_SMEM));   \
        gemm_tc_kernel<AM, BM><<<grid, G_THREADS, G_SMEM, (cudaStream_t)stream>>>(ma, mb, p);                     \
    } while (0)
    if (a_mn && b_mn) EB_GEMM_LAUNCH(true, true);
    else if (a_mn) EB_GEMM_LAUNCH(true, false);
    else if (b_mn) EB_GEMM_LAUNCH(false, true);
    else EB_GEMM_LAUNCH(false, false);
#undef EB_GEMM_LAUNCH
    EB_CUDA(cudaGetLastError());
    if (splits > 1) {
        int64_t g = ((int64_t)M * N + 255) / 256; const int64_t cap = (int64_t)sm_count() * 8; if (g > cap) g = cap;
        splitk_reduce_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>((const float *)ws, splits, M, N, C, ldc);
        EB_CUDA(cudaGetLastError());
    }
    return EB_OK;
}

extern "C" size_t eb_gemm_workspace_bytes(void) { return (size_t)sm_count() * G_BM * G_BN * sizeof(float); }

extern "C" int eb_gemm_bf16_tn(const void *A_bf16, int64_t lda, const void *B_bf16, int64_t ldb, float *C, int64_t ldc,
                               int M, int N, int K, const float *bias, float alpha, int act, void *workspace, size_t workspace_bytes,
                               void *stream) {
    return gemm_bf16(A_bf16, lda, false, B_bf16, ldb, false, C, ldc, M, N, K, bias, alpha, act, workspace, workspace_bytes, stream);
}

extern "C" int eb_gemm_bf16(const void *A_bf16, int64_t lda, int a_rows_are_k, const void *B_bf16, int64_t ldb, int b_rows_are_k,
                            float *C, int64_t ldc, int M, int N, int K, const float *bias, float alpha, int act, void *workspace,
                            size_t workspace_bytes, void *stream) {
    return gemm_bf16(A_bf16, lda, a_rows_are_k != 0, B_bf16, ldb, b_rows_are_k != 0, C, ldc, M, N, K, bias, alpha, act, workspace,
                     workspace_bytes, stream);
}

extern "C" int eb_gemm_bf16_out(const void *A_bf16, int64_t lda, int a_rows_are_k, const void *B_bf16, int64_t ldb, int b_rows_are_k,
                                float *C, int64_t ldc, void *C_bf16, int64_t ldcb, int M, int N, int K, const float *bias, float alpha,
                                int act, void *stream) {
    return gemm_bf16(A_bf16, lda, a_rows_are_k != 0, B_bf16, ldb, b_rows_are_k != 0, C, ldc, M, N, K, bias, alpha, act, nullptr, 0, stream,
                     C_bf16, ldcb);
}
