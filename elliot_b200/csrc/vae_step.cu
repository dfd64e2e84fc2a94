// vae_step.cu — one MultiVAE training step as ONE native call (SURVEY.md §8a V2).
//
// The step is ~35 kernel launches (8 tensor-core GEMMs, the row-major bf16 operand copies they read, the sparse first
// layer, reparameterisation, softmax/NLL, bias column sums, Adam on 8 parameters, operand refresh).  Driven launch
// by launch from Python it is bound by interpreter + ctypes overhead, not by the GPU; this entry point issues the
// same kernels, in the same order, back to back from C++ on the caller's stream, with every intermediate carved
// out of one caller-provided workspace.  Formulas: multi_vae_model.py:32-83 (encoder/decoder), :114-142
// (loss, train_step); the per-kernel restatements live in vae.cu / gemm_tc.cu / bpr_batch.cu.
// phase bit 0: forward + backward (gradients into m->g*, loss terms into acc); bit 1: Adam + refresh of the bf16
// operand copies (the W*t fields of eb_vae_model are no longer read: no transposed copies exist).  Data-parallel callers run bit 0, all-reduce the flat gradient buffer, then bit 1.
#include "common.cuh"

namespace eb {
namespace {

inline size_t up256(size_t x) { return (x + 255) / 256 * 256; }
inline int64_t pad8(int64_t x) { return (x + 7) / 8 * 8; }
inline int64_t pad4(int64_t x) { return (x + 3) / 4 * 4; }

struct VaeWs {
    float *h1, *ml, *z, *h2, *logits, *dh2, *dpre2, *dz, *dml, *dh1, *dpre1;
    void *h1b, *zb, *h2b, *dlb, *dpre2b, *dmlb;
    void *gws;                                 // split-K workspace of the GEMMs (one at a time)
    size_t gws_bytes, total;
};

VaeWs carve(char *base, int64_t I, int64_t H, int64_t L, int64_t B) {
    VaeWs w{};
    size_t off = 0;
    auto f32 = [&](int64_t n) { float *p = (float *)(base + off); off += up256((size_t)n * 4); return p; };
    auto b16 = [&](int64_t n) { void *p = (void *)(base + off); off += up256((size_t)n * 2); return p; };
    w.h1 = f32(B * H); w.ml = f32(B * 2 * L); w.z = f32(B * L); w.h2 = f32(B * H); w.logits = f32(B * I);
    w.dh2 = f32(B * H); w.dpre2 = f32(B * H); w.dz = f32(B * L); w.dml = f32(B * 2 * L); w.dh1 = f32(B * H); w.dpre1 = f32(B * H);
    w.h1b = b16(B * pad8(H)); w.zb = b16(B * pad8(L)); w.h2b = b16(B * pad8(H));
    w.dlb = b16(B * pad8(I)); w.dpre2b = b16(B * pad8(H)); w.dmlb = b16(B * pad8(2 * L));
    w.gws_bytes = eb_gemm_workspace_bytes();
    w.gws = (void *)(base + off); off += up256(w.gws_bytes);
    w.total = off;
    return w;
}

}  // namespace
}  // namespace eb

extern "C" size_t eb_vae_step_workspace_bytes(int n_items, int H, int L, int B) {
    return eb::carve(nullptr, n_items, H, L, B).total + 256;
}

#define EB_TRY(call)                      \
    do {                                  \
        const int rc_ = (call);           \
        if (rc_ != EB_OK) return rc_;     \
    } while (0)

extern "C" int eb_vae_train_step(const eb_vae_model *m, const int32_t *rows, int B, float drop_rate, uint64_t noise_seed,
                                 uint64_t drop_seed, uint64_t step, float anneal, float lr, double *acc, void *workspace,
                                 size_t workspace_bytes, int phase, void *stream) {
    using namespace eb;
    EB_ARG(m && m->W1 && m->W2 && m->W3 && m->W4 && m->gW1 && m->W2b && m->W3b && m->W4b && m->indptr && m->indices, "incomplete model");
    const int64_t I = m->n_items, H = m->H, L = m->L;
    EB_ARG(I >= 1 && H >= 8 && L >= 8 && H % 8 == 0 && L % 8 == 0, "need H, L multiples of 8 (H=%d L=%d)", (int)H, (int)L);
    if (phase & 1) {
        EB_ARG(rows && B >= 1 && acc, "rows / B / acc");
        EB_ARG(workspace && ((uintptr_t)workspace % 256) == 0, "workspace must be 256-byte aligned");
        const VaeWs w = carve((char *)workspace, I, H, L, B);
        if (workspace_bytes < w.total) return set_err(EB_ERR_WORKSPACE, "vae step workspace too small: need %zu bytes", w.total);
        const int64_t H8 = pad8(H), L8 = pad8(L), I8 = pad8(I), LL = 2 * L, LL8 = pad8(2 * L);
        // ---- forward (multi_vae_model.py:56-64, 80-83)
        EB_TRY(eb_vae_embed_fwd(m->W1, m->b1, (int)H, m->indptr, m->indices, rows, B, w.h1, H, drop_rate, drop_seed, stream));
        EB_TRY(eb_convert_bf16(w.h1, B, (int)H, H, w.h1b, H8, 0, stream));
        EB_TRY(eb_gemm_bf16_tn(w.h1b, H8, m->W2b, H8, w.ml, LL, B, (int)LL, (int)H, m->b2, 1.f, 0, w.gws, w.gws_bytes, stream));
        EB_TRY(eb_vae_reparam_fwd(w.ml, LL, B, (int)L, w.z, L, noise_seed, step, acc + 0, stream));
        EB_TRY(eb_convert_bf16(w.z, B, (int)L, L, w.zb, L8, 0, stream));
        EB_TRY(eb_gemm_bf16_tn(w.zb, L8, m->W3b, L8, w.h2, H, B, (int)H, (int)L, m->b3, 1.f, 1, w.gws, w.gws_bytes, stream));
        EB_TRY(eb_convert_bf16(w.h2, B, (int)H, H, w.h2b, H8, 0, stream));
        EB_TRY(eb_gemm_bf16_tn(w.h2b, H8, m->W4b, H8, w.logits, I, B, (int)I, (int)H, m->b4, 1.f, 0, w.gws, w.gws_bytes, stream));
        // ---- loss + backward (multi_vae_model.py:114-142); dlogits overwrite the logits.  Every backward GEMM reads the row-major
        // bf16 copies as they lie: "rows are K" operands (eb_gemm_bf16) instead of transposed copies — dW = dY^T . X contracts over
        // the batch rows of both operands, dX = dY . W takes the [out][in] weight as a [K][N] matrix.
        EB_TRY(eb_vae_softmax_bf16(w.logits, I, (int)I, m->indptr, m->indices, rows, B, acc + 1, nullptr, 1, w.dlb, I8, stream));
        EB_TRY(eb_gemm_bf16(w.dlb, I8, 1, w.h2b, H8, 1, m->gW4, H, (int)I, (int)H, B, nullptr, 1.f, 0, w.gws, w.gws_bytes, stream));
        EB_TRY(eb_colsum(w.logits, B, (int)I, I, m->gb4, stream));
        EB_TRY(eb_gemm_bf16(w.dlb, I8, 0, m->W4b, H8, 1, w.dh2, H, B, (int)H, (int)I, nullptr, 1.f, 0, w.gws, w.gws_bytes, stream));
        EB_TRY(eb_tanh_bwd(w.dh2, w.h2, w.dpre2, B * H, stream));
        EB_TRY(eb_convert_bf16(w.dpre2, B, (int)H, H, w.dpre2b, H8, 0, stream));
        EB_TRY(eb_gemm_bf16(w.dpre2b, H8, 1, w.zb, L8, 1, m->gW3, L, (int)H, (int)L, B, nullptr, 1.f, 0, w.gws, w.gws_bytes, stream));
        EB_TRY(eb_colsum(w.dpre2, B, (int)H, H, m->gb3, stream));
        EB_TRY(eb_gemm_bf16(w.dpre2b, H8, 0, m->W3b, L8, 1, w.dz, L, B, (int)L, (int)H, nullptr, 1.f, 0, w.gws, w.gws_bytes, stream));
        EB_TRY(eb_vae_reparam_bwd(w.ml, LL, B, (int)L, w.dz, L, w.dml, LL, noise_seed, step, anneal, stream));
        EB_TRY(eb_convert_bf16(w.dml, B, (int)LL, LL, w.dmlb, LL8, 0, stream));
        EB_TRY(eb_gemm_bf16(w.dmlb, LL8, 1, w.h1b, H8, 1, m->gW2, H, (int)LL, (int)H, B, nullptr, 1.f, 0, w.gws, w.gws_bytes, stream));
        EB_TRY(eb_colsum(w.dml, B, (int)LL, LL, m->gb2, stream));
        EB_TRY(eb_gemm_bf16(w.dmlb, LL8, 0, m->W2b, H8, 1, w.dh1, H, B, (int)H, (int)LL, nullptr, 1.f, 0, w.gws, w.gws_bytes, stream));
        EB_TRY(eb_tanh_bwd(w.dh1, w.h1, w.dpre1, B * H, stream));
        EB_TRY(eb_colsum(w.dpre1, B, (int)H, H, m->gb1, stream));
        EB_TRY(eb_vae_embed_bwd(m->gW1, (int)H, m->indptr, m->indices, rows, B, w.dpre1, H, drop_rate, drop_seed, stream));
    }
    if (phase & 2) {
        // ---- Keras Adam on every parameter (clears the gradients), then the bf16 operand copies in both orientations
        const float b1 = 0.9f, b2 = 0.999f, eps = 1e-7f;
        EB_TRY(eb_adam_dense_f32(m->W1, m->mW1, m->vW1, m->gW1, I * H, lr, b1, b2, eps, (int64_t)step, stream));
        EB_TRY(eb_adam_dense_f32(m->b1, m->mb1, m->vb1, m->gb1, pad4(H), lr, b1, b2, eps, (int64_t)step, stream));
        // kernels whose row length is a multiple of 8 get their bf16 operand copy straight from the optimiser pass
        const bool c2 = H % 8 == 0, c3 = L % 8 == 0;
        EB_TRY(eb_adam_dense_copy_f32(m->W2, m->mW2, m->vW2, m->gW2, 2 * L * H, lr, b1, b2, eps, (int64_t)step, c2 ? m->W2b : nullptr, stream));
        EB_TRY(eb_adam_dense_f32(m->b2, m->mb2, m->vb2, m->gb2, pad4(2 * L), lr, b1, b2, eps, (int64_t)step, stream));
        EB_TRY(eb_adam_dense_copy_f32(m->W3, m->mW3, m->vW3, m->gW3, H * L, lr, b1, b2, eps, (int64_t)step, c3 ? m->W3b : nullptr, stream));
        EB_TRY(eb_adam_dense_f32(m->b3, m->mb3, m->vb3, m->gb3, pad4(H), lr, b1, b2, eps, (int64_t)step, stream));
        EB_TRY(eb_adam_dense_copy_f32(m->W4, m->mW4, m->vW4, m->gW4, I * H, lr, b1, b2, eps, (int64_t)step, c2 ? m->W4b : nullptr, stream));
        EB_TRY(eb_adam_dense_f32(m->b4, m->mb4, m->vb4, m->gb4, pad4(I), lr, b1, b2, eps, (int64_t)step, stream));
        const int64_t H8 = pad8(H), L8 = pad8(L), LL = 2 * L;
        if (!c2) EB_TRY(eb_convert_bf16(m->W2, (int)LL, (int)H, H, m->W2b, H8, 0, stream));
        if (!c3) EB_TRY(eb_convert_bf16(m->W3, (int)H, (int)L, L, m->W3b, L8, 0, stream));
        if (!c2) EB_TRY(eb_convert_bf16(m->W4, (int)I, (int)H, H, m->W4b, H8, 0, stream));
    }
    return EB_OK;
}
