// gemm_ref.cu — fp32 CUDA-core GEMM with the calling convention of eb_gemm_bf16 (gemm_tc.cu): a CHECKING path, not a fast one.
//
// The tensor-core GEMM rounds its operands to bf16, so tests of the dense-layer models against the fp64 restatements
// (oracle/tf_models.py) can only agree to ~1e-2.  With `ops.exact_gemm(True)` the host wrappers keep the fp32 tensors and
// route every dense layer through this kernel instead: same operand-major flags, same bias / activation epilogue, fp32
// FMA accumulation in a fixed order — the model WIRING (which operand, which transpose, which bias, which activation, which
// gradient goes where) is then checked to 1e-5 and the top-k lists exactly, independently of bf16 rounding
// (VERDICT r1, "what's weak").  Never used by the product path.
#include "common.cuh"

namespace eb {

// C[m][n] = act(alpha * sum_k A(m,k) * B(n,k) + bias[n]);  A(m,k) = a_mn ? A[k*lda+m] : A[m*lda+k], B likewise
__global__ void __launch_bounds__(256) gemm_f32_ref_kernel(const float *__restrict__ A, int64_t lda, int a_mn, const float *__restrict__ B,
                                                           int64_t ldb, int b_mn, float *__restrict__ C, int64_t ldc, int M, int N, int K,
                                                           const float *__restrict__ bias, float alpha, int act) {
    __shared__ float sa[16][17], sb[16][17];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int n = blockIdx.x * 16 + tx;
    for (int mt = blockIdx.y; mt * 16 < M; mt += gridDim.y) {          // row tiles beyond the 65535 of grid.y: loop
        const int m = mt * 16 + ty;
        float acc = 0.f;
        for (int k0 = 0; k0 < K; k0 += 16) {
            const int ka = k0 + tx;                                     // A tile element (m, ka)
            sa[ty][tx] = (m < M && ka < K) ? (a_mn ? A[(int64_t)ka * lda + m] : A[(int64_t)m * lda + ka]) : 0.f;
            const int kb = k0 + ty, nb = blockIdx.x * 16 + tx;         // B tile element (nb, kb)
            sb[ty][tx] = (nb < N && kb < K) ? (b_mn ? B[(int64_t)kb * ldb + nb] : B[(int64_t)nb * ldb + kb]) : 0.f;
            __syncthreads();
#pragma unroll
            for (int k = 0; k < 16; k++) acc = fmaf(sa[ty][k], sb[k][tx], acc);
            __syncthreads();
        }
        if (m < M && n < N) {
            float x = alpha * acc + (bias ? bias[n] : 0.f);
            if (act == 1) x = tanhf(x);
            else if (act == 2) x = fmaxf(x, 0.f);
            C[(int64_t)m * ldc + n] = x;
        }
    }
}

}  // namespace eb

extern "C" int eb_gemm_f32_ref(const float *A, int64_t lda, int a_rows_are_k, const float *B, int64_t ldb, int b_rows_are_k, float *C,
                               int64_t ldc, int M, int N, int K, const float *bias, float alpha, int act, void *stream) {
    using namespace eb;
    EB_ARG(A && B && C && M >= 1 && N >= 1 && K >= 1 && ldc >= N && act >= 0 && act <= 2, "bad argument");
    EB_ARG(lda >= (a_rows_are_k ? M : K) && ldb >= (b_rows_are_k ? N : K), "leading dimensions too small");
    const int m_tiles = (M + 15) / 16;
    dim3 grid((unsigned)((N + 15) / 16), (unsigned)(m_tiles < 65535 ? m_tiles : 65535));
    gemm_f32_ref_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A, lda, a_rows_are_k, B, ldb, b_rows_are_k, C, ldc, M, N, K, bias, alpha, act);
    EB_CUDA(cudaGetLastError());
    return EB_OK;
}
