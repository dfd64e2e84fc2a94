/*
 * elliot_b200.h — C ABI of the H100 (sm_90a) embedding-training core.
 *
 * The reference (sisinflab/elliot v0.3.1) is pure Python and has no FFI of its
 * own; its hot path lives in per-model Python classes.  Every entry point below
 * replaces the arithmetic of one reference function (cited per function,
 * paths relative to the upstream tree) and is what the host-side plugin classes
 * in elliot_b200/recommender/ bind through ctypes (see INTEGRATION.md for the
 * stub a maintainer of the reference would add).
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host / says host;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *   - tables are row-major, row stride `ld` elements (ld >= d, ld % 4 == 0 for
 *     the f32 kernels, padding columns must be zero and stay zero);
 *   - ids are PRIVATE indices (dataset.py:211-217), int32;
 *   - the library never allocates or frees caller-visible memory: scratch is
 *     passed in, sized by the matching *_workspace_bytes() call;
 *   - every function returns 0 on success, a negative EB_* code otherwise;
 *     eb_last_error() gives the message for the calling thread.
 *   - no CPU fallback exists: without a CUDA device every compute call fails.
 */
#ifndef ELLIOT_B200_H
#define ELLIOT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EB_OK 0
#define EB_ERR_ARG (-1)      /* bad argument (shape, alignment, null) */
#define EB_ERR_CUDA (-2)     /* CUDA runtime error */
#define EB_ERR_WORKSPACE (-3)/* workspace too small */
#define EB_ERR_DATA (-4)     /* data the reference itself cannot handle (e.g. a user owning every item) */

const char *eb_last_error(void);
int eb_version(void);
/* number of SMs / compute capability major*10+minor of the current device */
int eb_device_info(int *sm_count, int *cc);

/* ------------------------------------------------------------------------
 * BPR-MF training step.
 * Replaces MFModel.train_step/update_factors
 *   (elliot/recommender/latent_factor_models/BPRMF/BPRMF_model.py:87-117):
 *   x_uk = b_k + U[u].V[k];  z = 1/(1+exp(x_ui-x_uj));
 *   b_i += lr(z - reg_b b_i); b_j += lr(-z - reg_b b_j);
 *   U[u] += lr((V_i-V_j) z - reg_u U[u]);
 *   V_i += lr(U'[u] z - reg_pos V_i); V_j += lr(-U'[u] z - reg_neg V_j)
 *   with U' the ALREADY UPDATED user row (the reference's view-aliasing).
 * ------------------------------------------------------------------------ */

/* Throughput mode: fp32, one launch over n materialised triples, rows updated
 * with 128-bit vector atomics (Hogwild: reads within a launch may be stale).
 * loss (optional, device double[1]) += sum softplus(-(x_ui-x_uj)).
 * flags: bit0 = plain stores instead of atomics (racy Hogwild); bit6 = deterministic rounds (cooperative launch: every
 * triple reads the values left by the previous rounds of reads-then-atomic-adds, so reruns give the same tables up to
 * fp32 summation order; slower); bits 8..15 = number of SMs the persistent grid leaves free (so a collective kernel on
 * another stream can run beside it).  The same flags apply to the sampled and host-triple variants below; bit 2 is
 * refused with EB_ERR_ARG. */
int eb_bpr_step_f32(float *U, float *V, float *item_bias, int d, int ld,
                    const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n,
                    float lr, float reg_u, float reg_b, float reg_pos, float reg_neg,
                    double *loss, int flags, void *stream);

/* Throughput mode with the sampler fused in: replaces Sampler.step/sample()
 * (elliot/dataset/samplers/custom_sampler.py:24-46) by a counter-based device
 * sampler with the same distribution (u uniform over users, i uniform over
 * u's train items, j uniform over items not in u's train set, by rejection)
 * but a different stream (Philox4x32-10 keyed by seed, counter = triple index
 * `first_triple`+t), then applies the update above.  csr_indices rows must be
 * sorted ascending.  out_u/out_i/out_j (optional) receive the sampled triples, triple t at index t.
 * Free-running (flags bit 6 clear), the call is a key pass that writes the user each triple draws, a stable cub radix
 * sort of the triple indices by user (a histogram kernel, a scan kernel and one pass per 8 key bits: 3 at 1 M users), and
 * the update, which applies the triples grouped by user in
 * ascending user order, keeping a user's row in registers across its triples and adding the run's summed update to it
 * once (a Hogwild launch applies its triples in no fixed order; which triples are drawn does not change).
 * workspace: device scratch of at least eb_bpr_step_sampled_workspace_bytes(n, n_users) bytes, else EB_ERR_WORKSPACE;
 * deterministic rounds (flags bit 6) apply the triples in sampler order and may pass NULL.  Flags bits 8..15: the key
 * pass and the update leave that many SMs free; the sort's kernels size their own grids and do not. */
size_t eb_bpr_step_sampled_workspace_bytes(int64_t n, int32_t n_users);
int eb_bpr_step_sampled_f32(float *U, float *V, float *item_bias, int d, int ld,
                            int32_t n_users, int32_t n_items,
                            const int64_t *csr_indptr, const int32_t *csr_indices,
                            int64_t n, uint64_t seed, uint64_t first_triple,
                            float lr, float reg_u, float reg_b, float reg_pos, float reg_neg,
                            double *loss, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                            void *workspace, size_t workspace_bytes, int flags, void *stream);

/* Per-user membership signatures for the sampler's rejection test (`j in ui`, custom_sampler.py:40-41): a Bloom
 * filter of 32*filter_words bits (filter_words a power of two, 32 = 1024 bits suits ~100 items/user) with 2 hash
 * functions per user, out[u*filter_words ...].  A candidate the signature rules out is accepted without touching the
 * CSR row; only "maybe" answers run the binary search, so the samples are EXACTLY those of the unfiltered sampler
 * (same stream, same triples) — only the dependent-load chain gets shorter. */
int eb_bloom_build(const int64_t *csr_indptr, const int32_t *csr_indices, int32_t n_users, int filter_words,
                   uint32_t *out, void *stream);
/* eb_bpr_step_sampled_f32 with the signatures (filter may be NULL) */
int eb_bpr_step_sampled_filter_f32(float *U, float *V, float *item_bias, int d, int ld,
                                   int32_t n_users, int32_t n_items,
                                   const int64_t *csr_indptr, const int32_t *csr_indices,
                                   const uint32_t *filter, int filter_words,
                                   int64_t n, uint64_t seed, uint64_t first_triple,
                                   float lr, float reg_u, float reg_b, float reg_pos, float reg_neg,
                                   double *loss, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                                   void *workspace, size_t workspace_bytes, int flags, void *stream);
/* The two halves of the free-running sampled step above, for one call of at most INT32_MAX triples; the step is the
 * schedule followed by the apply.  The schedule is the key pass and the stable sort: it reads only csr_indptr (never the
 * tables), so the schedule of the next call can run on another stream while this call's apply runs.  workspace: at least
 * eb_bpr_step_sampled_workspace_bytes(n, n_users) bytes; the ordered triple indices (n int32) are left at byte
 * *order_offset of it.  Flags bits 8..15: the key pass leaves that many SMs free.
 * The apply samples triple order[k] for k = 0..n-1 (triple t draws the same as in the step, whatever the order, and is
 * emitted at index t) and applies it grouped as in the step.  Any permutation of [0, n) gives the step's triples; one
 * sorted by user (the schedule's) gives long user runs.  Flags as for the step, without deterministic rounds (bit 6). */
int eb_bpr_schedule_sampled(int32_t n_users, int32_t n_items, const int64_t *csr_indptr, int64_t n, uint64_t seed,
                            uint64_t first_triple, void *workspace, size_t workspace_bytes, size_t *order_offset, int flags,
                            void *stream);
int eb_bpr_apply_sampled_filter_f32(float *U, float *V, float *item_bias, int d, int ld,
                                    int32_t n_users, int32_t n_items,
                                    const int64_t *csr_indptr, const int32_t *csr_indices,
                                    const uint32_t *filter, int filter_words,
                                    int64_t n, uint64_t seed, uint64_t first_triple,
                                    float lr, float reg_u, float reg_b, float reg_pos, float reg_neg,
                                    double *loss, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                                    const int32_t *order, int flags, void *stream);
/* Sample only (no update): same sampler as above (filter may be NULL), for tests and for host
 * pipelines that want materialised triples. */
int eb_bpr_sample_philox_filter(int32_t n_users, int32_t n_items, const int64_t *csr_indptr,
                                const int32_t *csr_indices, const uint32_t *filter, int filter_words, int64_t n,
                                uint64_t seed, uint64_t first_triple, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                                void *stream);

/* End-to-end variant of eb_bpr_step_f32 for HOST triples, PACKED one uint64 per triple, u | i << bits_u | j << (bits_u + bits_i)
 * (bits_u + 2*bits_i <= 64; 20 + 17 + 17 bits cover the C2 shape): ONE host-to-device copy of 8 bytes per triple into
 * `staging` (device, n uint64), the step (the kernel unpacks), the loss copied back into *loss_host, and the stream
 * synchronised (flags bit1 = do NOT synchronise: lets the caller pipeline steps on two streams so the next batch's H2D
 * overlaps this kernel). */
int eb_bpr_step_host_packed_f32(float *U, float *V, float *item_bias, int d, int ld, const uint64_t *packed_host, int64_t n,
                                int bits_u, int bits_i, float lr, float reg_u, float reg_b, float reg_pos, float reg_neg,
                                uint64_t *staging, double *loss_dev, double *loss_host, int flags, void *stream);

/* Exact mode: fp64, result identical to applying the n triples strictly one
 * after the other in array order (what the reference does with batch_size
 * forced to 1, BPRMF.py:80,119-127).  Row-level turn counters serialise only
 * the triples that really conflict.  n_users/n_items size the counters. */
size_t eb_bpr_exact_workspace_bytes(int64_t n, int32_t n_users, int32_t n_items);
int eb_bpr_exact_f64(double *U, double *V, double *item_bias, int d, int ld,
                     int32_t n_users, int32_t n_items,
                     const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n,
                     double lr, double reg_u, double reg_b, double reg_pos, double reg_neg,
                     double *loss, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------
 * Exact replay of the reference sampler's random stream on the device.
 * Replaces Sampler.__init__/step (custom_sampler.py:14-46): legacy
 * np.random.seed(42) MT19937, randint() = 32-bit masked rejection, no draw
 * when the range is 1.  `state` is 625 uint32 (624 words + position) on the
 * device; it advances by exactly the draws the reference would consume, so
 * consecutive calls continue one stream across epochs as the reference does.
 * set_indices rows are in the reference's list(set(...)) order
 * (custom_sampler.py:21); sorted_indices is the same CSR with rows sorted
 * (membership tests).  Returns EB_ERR_DATA if a sampled user owns every item
 * (the reference never terminates there).
 * ------------------------------------------------------------------------ */
int eb_mt_seed(uint32_t *state, uint32_t seed, void *stream);
size_t eb_mt_sampler_workspace_bytes(int64_t events);
int eb_mt_sampler_step(uint32_t *state, int32_t n_users, int32_t n_items,
                       const int64_t *indptr, const int32_t *set_indices, const int32_t *sorted_indices,
                       int64_t events, int32_t *out_u, int32_t *out_i, int32_t *out_j,
                       void *workspace, size_t workspace_bytes, void *stream);
/* Pointwise ratio sampler (dataset/samplers/pointwise_pos_neg_ratio_ratings_sampler.py, DMF): the same MT19937
 * stream.  Each sample: u = randint(n_users); np.random.shuffle of the list [0]*neg_ratio + [1]; if the list's
 * first slot holds the 1, a positive set_indices[randint(lui)] of u's row with its set_ratings value, else a
 * negative randint(n_items) redrawn while it is a train item, rating 0.  *list_pos (device int32) is the position
 * of the 1 in the list: the caller sets it to neg_ratio at each epoch's start (the reference rebuilds the list per
 * step() call) and the call leaves it where the last sample left it, as it advances the MT state by the draws
 * consumed.  0 <= neg_ratio <= 15.  Returns EB_ERR_DATA if a sampled user owns every item or none.
 * workspace: eb_mt_pointwise_ratio_workspace_bytes(events, n_users, neg_ratio) bytes, about 2.3 KB per event at
 * neg_ratio 5: call in windows (the stream does not depend on how it is windowed). */
size_t eb_mt_pointwise_ratio_workspace_bytes(int64_t events, int32_t n_users, int32_t neg_ratio);
int eb_mt_pointwise_ratio_step(uint32_t *state, int32_t *list_pos, int32_t n_users, int32_t n_items,
                               const int64_t *indptr, const int32_t *set_indices, const float *set_ratings,
                               const int32_t *sorted_indices, int32_t neg_ratio, int64_t events, int32_t *out_u,
                               int32_t *out_i, float *out_r, void *workspace, size_t workspace_bytes, void *stream);
/* raw tempered 32-bit outputs (testing the generator against numpy) */
int eb_mt_raw(uint32_t *state, uint32_t *out, int64_t n, void *stream);

/* ------------------------------------------------------------------------
 * Full-catalogue scoring + train-item mask + per-user top-k.
 * Replaces MFModel.get_user_predictions (BPRMF_model.py:70-85) and
 * BPRMF_batch_model.predict/get_top_k (BPRMF_batch_model.py:82-88):
 *   s = bias + U[u] @ V.T;  s[train items of u] = -inf;  top-k, descending,
 *   ties -> lower item index first (tf.nn.top_k rule).
 * users: optional list of n_sel private user ids (NULL = user_begin..+n_sel).
 * mask CSR rows = train items per user (NULL = no mask).  Slots with no
 * finite candidate get idx -1 / val -inf.
 * ------------------------------------------------------------------------ */
size_t eb_score_topk_workspace_bytes(int64_t n_sel, int32_t n_items, int elem_size);
int eb_score_topk_f32(const float *U, const float *V, const float *item_bias, int32_t n_items, int d, int ld,
                      const int64_t *mask_indptr, const int32_t *mask_indices,
                      const int32_t *users, int32_t user_begin, int64_t n_sel, int k,
                      int32_t *out_idx, float *out_val, void *workspace, size_t workspace_bytes, void *stream);
int eb_score_topk_f64(const double *U, const double *V, const double *item_bias, int32_t n_items, int d, int ld,
                      const int64_t *mask_indptr, const int32_t *mask_indices,
                      const int32_t *users, int32_t user_begin, int64_t n_sel, int k,
                      int32_t *out_idx, double *out_val, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------
 * Rank of every relevant item in the user's full list (the AUC / GAUC
 * counts of elliot/evaluation/metrics/accuracy/AUC/auc.py, gauc.py).
 * The full list is what eb_score_topk_* lists with k = n_items: every item
 * outside the train mask whose score (the same bits) is neither -inf nor
 * NaN, by (score desc, item asc).  Same scoring arguments and row choice as
 * eb_score_topk_*; rel CSR (indexed by user id): the user's relevant items,
 * sorted by item, -1 for items outside the catalogue.  Per row q:
 *   out_n_pos[q] = number of relevant items in the list (positives),
 *   out_sum_c[q] = sum over them of the non-relevant entries ahead of each.
 * out_c (optional, one per rel CSR entry of the selected users): that count
 * for a positive, -1 for an entry that is not in the list.  Integer counts:
 * the results do not depend on launch order.  No workspace.
 * ------------------------------------------------------------------------ */
int eb_score_rank_f32(const float *U, const float *V, const float *item_bias, int32_t n_items, int d, int ld,
                      const int64_t *mask_indptr, const int32_t *mask_indices,
                      const int64_t *rel_indptr, const int32_t *rel_items,
                      const int32_t *users, int32_t user_begin, int64_t n_sel,
                      int64_t *out_n_pos, int64_t *out_sum_c, int64_t *out_c, void *stream);
int eb_score_rank_f64(const double *U, const double *V, const double *item_bias, int32_t n_items, int d, int ld,
                      const int64_t *mask_indptr, const int32_t *mask_indices,
                      const int64_t *rel_indptr, const int32_t *rel_items,
                      const int32_t *users, int32_t user_begin, int64_t n_sel,
                      int64_t *out_n_pos, int64_t *out_sum_c, int64_t *out_c, void *stream);

/* ------------------------------------------------------------------------
 * Mini-batch BPR-MF with Adam (the reference's TensorFlow variant).
 * Replaces BPRMF_batch_model.call/train_step (BPRMF_batch_model.py:46-80):
 * eb_bpr_batch_grad_f32 accumulates the batch gradient of
 *   sum softplus(-clip(x_pos-x_neg,-80,1e8)) + l_w(|gu|^2+|gpos|^2+|gneg|^2)/2 + l_b bpos^2/2 + l_b bneg^2/20
 * into dense gradient tables (duplicates summed, like IndexedSlices);
 * eb_adam_dense_f32 is Keras Adam applied to every element (TF 2.3 moves all rows even for
 * sparse gradients) and clears the gradient.  lr_t = lr sqrt(1-b2^step)/(1-b1^step).
 * ------------------------------------------------------------------------ */
int eb_bpr_batch_grad_f32(const float *Gu, const float *Gi, const float *Bi, float *dGu, float *dGi, float *dBi,
                          int d, int ld, const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n,
                          float l_w, float l_b, double *loss, void *stream);
int eb_adam_dense_f32(float *var, float *m, float *v, float *grad, int64_t n, float lr, float beta1, float beta2,
                      float eps, int64_t step, void *stream);
/* the same, also writing the updated values as a bf16 array of the same length and layout (the tensor-core operand copy of a
 * dense kernel whose row length is a multiple of 8: no separate conversion pass after the optimiser) */
int eb_adam_dense_copy_f32(float *var, float *m, float *v, float *grad, int64_t n, float lr, float beta1, float beta2,
                           float eps, int64_t step, void *copy_bf16, void *stream);

/* ------------------------------------------------------------------------
 * MultiVAE pieces around the dense layers (multi_vae_model.py:20-159, sparse_sampler.py:13-25).
 * rows[b] = private user id of batch row b; indptr/indices = train CSR (the dense B x I input of
 * the reference is never materialised).  See elliot_b200/csrc/vae.cu for the per-call formulas.
 * ------------------------------------------------------------------------ */
int eb_vae_embed_fwd(const float *W1, const float *b1, int H, const int64_t *indptr, const int32_t *indices,
                     const int32_t *rows, int B, float *h1, int64_t ldh, float drop_rate, uint64_t seed, void *stream);
int eb_vae_embed_bwd(float *dW1, int H, const int64_t *indptr, const int32_t *indices, const int32_t *rows, int B,
                     const float *dpre1, int64_t ldd, float drop_rate, uint64_t seed, void *stream);
/* eps of element e = b L + l at step `step` is the Philox draw (key seed, counter (step, e)): no two steps share a draw
 * whatever their batch sizes; B L < 2^32 */
int eb_vae_reparam_fwd(const float *ml, int64_t ldml, int B, int L, float *z, int64_t ldz, uint64_t seed, uint64_t step,
                       double *kl_sum, void *stream);
int eb_vae_reparam_bwd(const float *ml, int64_t ldml, int B, int L, const float *dz, int64_t lddz, float *dml,
                       int64_t lddml, uint64_t seed, uint64_t step, float anneal, void *stream);
int eb_vae_softmax(float *logits, int64_t ld, int n_items, const int64_t *indptr, const int32_t *indices,
                   const int32_t *rows, int B, double *nll_sum, float *lse_out, int write_grad, void *stream);
/* the same, additionally writing the gradient as bf16 rows (row stride ld_bf16 >= n_items and a multiple of 8, grad_bf16
 * 16-byte aligned, padding columns zeroed): the operand copy the backward GEMMs read.  Rows up to 200 KB are staged in shared
 * memory (one pass over the B x I block). */
int eb_vae_softmax_bf16(float *logits, int64_t ld, int n_items, const int64_t *indptr, const int32_t *indices,
                        const int32_t *rows, int B, double *nll_sum, float *lse_out, int write_grad, void *grad_bf16,
                        int64_t ld_bf16, void *stream);
int eb_tanh_bwd(const float *dout, const float *out, float *dpre, int64_t n, void *stream);
int eb_colsum(const float *src, int rows, int cols, int64_t ld, float *out, void *stream);
/* One whole MultiVAE training step as ONE native call: the same kernels as the entry points above, issued back to back
 * from C++ (the step is ~35 launches).  Replaces
 * VariationalAutoEncoder.train_step (multi_vae_model.py:125-142).  Layouts: W1 [I][H] fp32; W2 [2L][H], W3 [H][L],
 * W4 [I][H] fp32 ([out][in]); biases padded to multiples of 4; g* gradients, m* / v* Adam moments, same shapes;
 * W?b: bf16 operand copies [out][pad8(in)], refreshed by phase bit 1 (the backward GEMMs read the same copies as
 * [K][N] matrices through eb_gemm_bf16, so the W?t fields are no longer read and may be NULL).
 * phase: bit 0 = forward + backward (gradients into g*, acc[0] += KL sum term, acc[1] += NLL sum);
 *        bit 1 = Adam (lr_t = lr sqrt(1-b2^step)/(1-b1^step), clears g*) + operand refresh.
 * A data-parallel caller runs phase 1, all-reduces the gradients, then phase 2. */
typedef struct eb_vae_model {
    int n_items, H, L, reserved;
    float *W1, *b1, *W2, *b2, *W3, *b3, *W4, *b4;
    float *gW1, *gb1, *gW2, *gb2, *gW3, *gb3, *gW4, *gb4;
    float *mW1, *mb1, *mW2, *mb2, *mW3, *mb3, *mW4, *mb4;
    float *vW1, *vb1, *vW2, *vb2, *vW3, *vb3, *vW4, *vb4;
    void *W2b, *W3b, *W4b, *W2t, *W3t, *W4t;
    const int64_t *indptr;
    const int32_t *indices;
} eb_vae_model;
size_t eb_vae_step_workspace_bytes(int n_items, int H, int L, int B);
int eb_vae_train_step(const eb_vae_model *m, const int32_t *rows, int B, float drop_rate, uint64_t noise_seed,
                      uint64_t drop_seed, uint64_t step, float anneal, float lr, double *acc, void *workspace,
                      size_t workspace_bytes, int phase, void *stream);
/* masked top-k over an existing dense score block (scores are overwritten); out_val = score + shift[row] */
int eb_dense_topk_f32(float *scores, int64_t ld, int n_rows, int n_items, const int64_t *mask_indptr,
                      const int32_t *mask_indices, const int32_t *rows, const float *shift, int k, int32_t *out_idx,
                      float *out_val, void *stream);

/* ------------------------------------------------------------------------
 * NeuMF pieces around the dense layers (neural_matrix_factorization_model.py:38-148,
 * NeuMF/custom_sampler.py:27-48).  See elliot_b200/csrc/neumf.cu for the per-call formulas.
 * ------------------------------------------------------------------------ */
int eb_neumf_gather(const float *Umf, const float *Imf, const float *Umlp, const float *Imlp, int f, int64_t ldt,
                    const int32_t *u, const int32_t *it, int64_t n, float *x0, int64_t ldx, float *pm, int64_t ldp, void *stream);
int eb_neumf_head(const float *pm, int64_t ldp, const float *h3, int64_t ldh, int f, const float *wp, const float *bp,
                  const float *label, int64_t n, float *dpm, float *dh3, float *dwp, float *dbp, double *loss,
                  float *prob_out, void *stream);
/* the same with the BinaryCrossentropy mean taken over `mean_over` samples instead of the n passed in (a rank's slice of
 * a global batch: the loss and every gradient root are scaled by 1/mean_over) */
int eb_neumf_head_norm(const float *pm, int64_t ldp, const float *h3, int64_t ldh, int f, const float *wp, const float *bp,
                       const float *label, int64_t n, int64_t mean_over, float *dpm, float *dh3, float *dwp, float *dbp,
                       double *loss, float *prob_out, void *stream);
int eb_relu_bwd(const float *dout, const float *out, float *dpre, int64_t n, void *stream);
/* the same, also writing dpre as a bf16 array of the same length (operand copy; row length a multiple of 8) */
int eb_relu_bwd_copy(const float *dout, const float *out, float *dpre, int64_t n, void *copy_bf16, void *stream);
int eb_neumf_scatter(const float *Umf, const float *Imf, int f, int64_t ldt, const int32_t *u, const int32_t *it, int64_t n,
                     const float *dpm, int64_t ldp, const float *dx0, int64_t ldx, float *dUmf, float *dImf, float *dUmlp,
                     float *dImlp, void *stream);
int eb_neumf_sample(int32_t n_users, int32_t n_items, const int64_t *indptr, const int32_t *indices, int m, uint64_t seed,
                    int64_t total, int32_t *out_u, int32_t *out_i, float *out_label, void *stream);
int eb_neumf_pair_h1(const float *Au, int64_t ldau, const float *Ai, int64_t ldai, const float *b1, int n_ub, int n_items,
                     int h1, void *out_bf16, int64_t ldo, void *stream);
/* checking mode (ops.exact_gemm): the same first layer kept in fp32 */
int eb_neumf_pair_h1_f32(const float *Au, int64_t ldau, const float *Ai, int64_t ldai, const float *b1, int n_ub, int n_items,
                         int h1, float *out, int64_t ldo, void *stream);
int eb_neumf_pair_head(const float *Umf, const float *Imf, int64_t ldt, int f, int u0, int n_ub, int n_items, const float *h3,
                       int64_t ldh, const float *wp, const float *bp, float *prob, int64_t ldpr, void *stream);

/* Multi-GPU reconciliation of a REPLICATED table (item factors / biases; SURVEY.md §8e): every
 * rank computes delta = cur - prev, the host all-reduces `delta` (NCCL), then
 * cur = prev = prev + scale * sum(delta)  (scale 1 = every rank's updates applied in full, 1/world = averaged,
 * the stable default when many ranks hit the same rows).  No reference counterpart (single-device reference). */
int eb_table_delta_f32(const float *cur, const float *prev, float *delta, int64_t n, void *stream);
int eb_table_apply_delta_f32(float *cur, float *prev, const float *delta_sum, int64_t n, float scale, void *stream);
/* overlapped variant (the all-reduce of step k runs while step k+1 computes):
 *   cur += scale*delta_sum - delta_local;  prev += scale*delta_sum */
int eb_table_apply_delta_late_f32(float *cur, float *prev, const float *delta_sum, const float *delta_local, int64_t n,
                                  float scale, void *stream);

/* ------------------------------------------------------------------------
 * MF2020: pointwise logistic matrix factorisation (sibling model on the same gather/dot/scatter shape).
 * Replaces MFModel.train_step (elliot/recommender/latent_factor_models/MF2020/MF_model.py:80-112):
 *   pred = gb + ub[u] + ib[i] + U[u].V[i]; grad = rating - sigmoid(pred);
 *   U[u] += lr(grad V[i] - reg U[u]); V[i] += lr(grad U'[u] - reg V[i]) (U' already updated: view aliasing);
 *   ub[u], ib[i], gb += lr(grad - reg .)
 * eb_mf_pointwise_exact_f64: the reference's order, fp64 — the global bias makes every sample depend on the
 *   previous one, so one warp walks the list (software-pipelined).  su/si/sr: the epoch's (user, item, label)
 *   list as produced by custom_sampler_rendle.Sampler.step; batch_loss[t / batch] (optional) = sum of this_loss
 *   over each `batch` consecutive samples (MF.py:120-124 divides by len(batch) itself); global_bias: device double[1].
 * eb_mf_pointwise_step_f32: throughput mode.  The epoch is the list of every positive (pos_u[p], pos_i[p], 1) plus m
 *   uniform items (pos_u[p], j, 0) — not rejected against the train set, like custom_sampler_rendle.py:66-69 — in a
 *   pseudo-random visiting order (affine permutation re-drawn per epoch instead of random.sample), Philox negatives
 *   keyed by (seed, epoch); one launch applies positions [first, first+count) of it with fp32 vector atomics
 *   (Hogwild: keep count small enough that a row is not hit by many stale updates).  The global bias, hit by every
 *   sample, is advanced once per launch by the closed-form integral of the c sequential steps (see mf2020.cu);
 *   gb_work: device double[4] scratch, zero before the first call, left zero.
 *   out_u/out_i/out_r (optional, n_pos*(1+m) each, indexed by epoch position).  loss (optional): += sum this_loss.
 * ------------------------------------------------------------------------ */
int eb_mf_pointwise_exact_f64(double *U, double *V, double *user_bias, double *item_bias, double *global_bias,
                              int d, int ld, const int32_t *su, const int32_t *si, const int32_t *sr, int64_t n,
                              double lr, double reg, int64_t batch, double *batch_loss, void *stream);
int eb_mf_pointwise_step_f32(float *U, float *V, float *user_bias, float *item_bias, float *global_bias, int d, int ld,
                             const int32_t *pos_u, const int32_t *pos_i, int64_t n_pos, int m, int32_t n_items,
                             uint64_t seed, uint64_t epoch, int64_t first, int64_t count, float lr, float reg, double *loss,
                             double *gb_work, int32_t *out_u, int32_t *out_i, int32_t *out_r, void *stream);

/* ------------------------------------------------------------------------
 * Accuracy metrics of top-k lists, on the device.
 * Replaces the per-user loops of Evaluator.eval (elliot/evaluation/evaluator.py:117-147) for nDCG
 * (ndcg.py:68-125; discount relevance.py:55, gains relevance.py:80-82), HR, Precision, Recall.
 * topk_idx[n_rows][ld]: private item ids, -1 = empty slot (as written by eb_score_topk_*); users (optional):
 * private user id of each row (NULL = row r is user r).  rel_indptr/rel_items/rel_gains: CSR over private
 * users of the relevant test items, rows sorted by item id (items absent from training carry id -1: they
 * count for Recall/IDCG but can never be hit).  idcg[u]: ideal DCG@k of user u; discount[k]: ln2/ln(r+2).
 * Users without relevant items are skipped (evaluator.py:121).
 * out[5] (device) = {evaluated users, sum nDCG, sum HR, sum Precision, sum Recall}: fp64, deterministic.
 * per_user (optional, device double[n_rows][4]): the per-user values (NaN for skipped users).
 * ------------------------------------------------------------------------ */
size_t eb_eval_topk_workspace_bytes(int64_t n_rows, int k);
int eb_eval_topk_f64(const int32_t *topk_idx, int64_t n_rows, int ld, int k, const int32_t *users,
                     const int64_t *rel_indptr, const int32_t *rel_items, const double *rel_gains,
                     const double *idcg, const double *discount, double *per_user, double *out,
                     void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------
 * The reference's other list metrics, on the device (elliot/evaluation/metrics): nDCGRendle2020, MRR, MAP, MAR, F1,
 * LAUC, NumRetrieved, EPC, EFD, ARP, APLT, ACLT, PopREO, PopRSP, ItemCoverage, UserCoverage, UserCoverageAtN, Gini,
 * SEntropy.  topk_idx / ld / k / users as for eb_eval_topk_f64; a row's list is its entries before the first -1.
 * rel_indptr/rel_items: the item-sorted relevant CSR of eb_eval_topk_f64 (gains are not needed: relevance is binary).
 * user_info[n_users][6] int32: has any test row, |train_u|, PopREO denominators (short head, long tail: relevant items
 * not in train_u), PopRSP denominators (|short head - train_u|, |long tail - train_u|).  Per private item: item_pop
 * (train users), item_long_tail (1 = long tail, 0 = short head), item_novelty[n_items][2] (EPC, EFD novelty).
 * Per position r < k: discount[r] = ln2/ln(r+2), map_tail[r] = H(k) - H(r); inv_binary_idcg[m] (m = 1..k) = 1 / sum_{i<m}
 * discount[i].  Rows whose user has no test row are skipped; the accuracy and novelty sums also skip users without a
 * relevant item.  Lists must hold distinct items.
 * out[29] (device, fp64, deterministic): {users with a relevant item, sums of nDCGRendle2020 MRR MAP MAR F1 LAUC
 * NumRetrieved EPC EFD, PopREO hits in short head / long tail, PopREO denominators (2), users with test rows, sums of
 * ARP APLT ACLT, PopRSP numerators (2), PopRSP denominators (2), UserCoverage, UserCoverageAtN, sum of list lengths,
 * users with test rows and an empty list, ItemCoverage, Gini rank sum sum_j j*cs_j over the ascending item counts,
 * SEntropy sum_u (1/n_u) sum_i -log2(c_i / sum n_u)}.
 * per_user (optional, device double[n_rows][12]): nDCGRendle2020 MRR MAP MAR F1 LAUC NumRetrieved EPC EFD ARP APLT
 * ACLT per row, NaN where the reference has no value for the user.
 * ------------------------------------------------------------------------ */
size_t eb_eval_metrics_workspace_bytes(int64_t n_rows, int k, int n_items);
int eb_eval_metrics_f64(const int32_t *topk_idx, int64_t n_rows, int ld, int k, const int32_t *users,
                        const int64_t *rel_indptr, const int32_t *rel_items, const int32_t *user_info,
                        const int32_t *item_pop, const uint8_t *item_long_tail, const double *item_novelty,
                        int n_items, const double *discount, const double *map_tail,
                        const double *inv_binary_idcg, double *per_user, double *out, void *workspace,
                        size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------
 * The reference's clustered fairness metrics, on the device (elliot/evaluation/metrics/fairness: BiasDisparityBR / BD,
 * User/ItemMADrating, User/ItemMADranking, REO, RSP).  topk_idx / ld / k / users and the relevant CSR with its gains,
 * per-user IDCG@k and discounts as for eb_eval_topk_f64; a row's list is its entries before the first -1.  scores
 * (optional, fp64, same ld as topk_idx): the lists' scores, read only for the rating sums.  has_rows[n_users]: the user
 * has any test row.  user_cluster[n_users] / item_cluster[n_items]: the cluster of each private id in 0..n-1, -1 = not
 * clustered.  A row counts when its user has test rows (A); the per-user and per-item sums also need >= 1 relevant
 * item (B).
 * counts (int64, n_user_clusters + n_user_clusters * n_item_clusters + 3 * n_item_clusters):
 *   [nu] B users per user cluster | [nu][ni] list entries of A users per (user cluster, item cluster), repeated items
 *   every time | [ni] distinct listed relevant items of B users (REO numerators) | [ni] distinct listed items of A users
 *   (RSP numerators) | [ni] listed items of B users per item cluster.
 * sums (fp64, 2 * nu + 2 * ni, deterministic): [nu] sum of nDCG over B users (each the bits eb_eval_topk_f64 gives) |
 *   [nu] sum of the mean list score (NaN for an empty list) | [ni] sum over listed items of their summed gains / count |
 *   [ni] sum over listed items of their summed relevant scores / count; an item's sums run in row, then list order.
 * ------------------------------------------------------------------------ */
size_t eb_eval_fairness_workspace_bytes(int64_t n_rows, int k, int n_items, int n_user_clusters, int n_item_clusters);
int eb_eval_fairness_f64(const int32_t *topk_idx, const double *scores, int64_t n_rows, int ld, int k,
                         const int32_t *users, const int64_t *rel_indptr, const int32_t *rel_items,
                         const double *rel_gains, const double *idcg, const double *discount, const uint8_t *has_rows,
                         const int32_t *user_cluster, int n_user_clusters, const int32_t *item_cluster,
                         int n_item_clusters, int n_items, int64_t *counts, double *sums, void *workspace,
                         size_t workspace_bytes, void *stream);

/* SM partition for compute/collective overlap (no reference counterpart): creates a green context holding
 * all but >= reserve_sms SMs of the current device (rounded to the driver's 8-SM granularity) and n_streams
 * CUDA streams bound to it.  Kernels launched on those streams run only inside the partition, so a collective
 * (NCCL) kernel on an ordinary stream always finds the SMs left out.  *granted_sms = SMs in the partition; pass
 * (device SMs - granted) as the reserve bits of eb_bpr_step_*'s flags so the persistent grid is sized to it.
 * The context lives until process exit. */
int eb_partition_streams_create(int reserve_sms, int n_streams, void **streams, int *granted_sms);

/* ------------------------------------------------------------------------
 * Dense layers (MultiVAE encoder/decoder, NeuMF MLP): bf16 tensor-core GEMM
 *   C[M][N] (fp32) = act(alpha * A[M][K] . B[N][K]^T + bias[N])      act: 0 none, 1 tanh, 2 relu
 * A and B are bf16 with K contiguous (Keras Dense kernels kept as [out][in]); replaces the
 * tf.keras.layers.Dense calls of multi_vae_model.py:44-53,72-78 and
 * neural_matrix_factorization_model.py:57-70.  eb_convert_bf16 produces the bf16 operand from an
 * fp32 matrix, optionally transposed ([rows][cols] -> [cols][dst_ld]); dst_ld % 8 == 0.
 * ------------------------------------------------------------------------ */
int eb_convert_bf16(const float *src, int rows, int cols, int64_t ld, void *dst_bf16, int64_t dst_ld, int transpose,
                    void *stream);
/* workspace (may be NULL): eb_gemm_workspace_bytes() bytes that let a GEMM with few output tiles and a long K (no bias, no
 * activation) split K over the idle SMs; the partial tiles are summed in a fixed order, so the result is the same bits on
 * every run.  Without it the GEMM runs single-pass.  One GEMM at a time may use a workspace. */
size_t eb_gemm_workspace_bytes(void);
int eb_gemm_bf16_tn(const void *A_bf16, int64_t lda, const void *B_bf16, int64_t ldb, float *C, int64_t ldc,
                    int M, int N, int K, const float *bias, float alpha, int act, void *workspace, size_t workspace_bytes,
                    void *stream);
/* The same contraction with either operand given "rows are K": a_rows_are_k != 0 means A is a [K][M] row-major matrix
 * (M contiguous, lda >= M), likewise B as [K][N].  The tensor cores read such tiles directly (MN-major shared-memory
 * descriptors), so the backward GEMMs dW = dY^T . X (K = batch) and dX = dY . W with W kept [K][N] need no transposed copies. */
int eb_gemm_bf16(const void *A_bf16, int64_t lda, int a_rows_are_k, const void *B_bf16, int64_t ldb, int b_rows_are_k,
                 float *C, int64_t ldc, int M, int N, int K, const float *bias, float alpha, int act, void *workspace,
                 size_t workspace_bytes, void *stream);
/* ... and with a second output: C_bf16 (row stride ldcb >= N) receives the same values as bf16 — the next layer's operand copy,
 * written from the epilogue's registers instead of by a conversion pass (not combined with split-K). */
int eb_gemm_bf16_out(const void *A_bf16, int64_t lda, int a_rows_are_k, const void *B_bf16, int64_t ldb, int b_rows_are_k,
                     float *C, int64_t ldc, void *C_bf16, int64_t ldcb, int M, int N, int K, const float *bias, float alpha,
                     int act, void *stream);
/* CHECKING path (tests only, slow): the same contraction with fp32 operands on the CUDA cores, fixed-order fp32 FMA
 * accumulation — lets the dense-layer models be compared with their fp64 restatements to 1e-5 instead of bf16's 1e-2. */
int eb_gemm_f32_ref(const float *A, int64_t lda, int a_rows_are_k, const float *B, int64_t ldb, int b_rows_are_k, float *C,
                    int64_t ldc, int M, int N, int K, const float *bias, float alpha, int act, void *stream);

/* Row-SHARDED tables (SURVEY.md §8e): owners gather requested rows / add returned deltas; the requester
 * runs the BPR update (BPRMF_model.py:91-117 arithmetic) against fetched item-row copies: user rows are
 * local and updated in place, item deltas dRi/dRj are written per triple.  If bias_col >= 0 that column
 * of the (padded) item rows carries the item bias.  The id exchange itself is an NCCL all-to-all done by
 * the host (elliot_b200/parallel.py::ShardedTable). */
int eb_gather_rows_f32(const float *table, int64_t ld, const int32_t *ids, int64_t n, int width, float *out, int64_t ldo,
                       void *stream);
int eb_scatter_add_rows_f32(float *table, int64_t ld, const int32_t *ids, int64_t n, int width, const float *rows,
                            int64_t ldr, void *stream);
int eb_bpr_step_rows_f32(float *U, int64_t ldu, const int32_t *tu, const float *Ri, const float *Rj, int64_t ldr, int64_t n,
                         int bias_col, float lr, float reg_u, float reg_b, float reg_pos, float reg_neg, float *dRi,
                         float *dRj, double *loss, void *stream);

/* ------------------------------------------------------------------------
 * GMF (neural/GeneralizedMF/generalized_matrix_factorization_model.py:18-92, is_edge_weight_train = True):
 * out = sigmoid((U[u]*I[i]).h), BinaryCrossentropy (mean over `mean_over` samples).  One fused kernel per batch gathers,
 * scores, and scatters the gradients into the dense tables dU/dI (+ dh, loss) for the dense Keras Adam that follows.
 * eb_pointwise_sample_philox: dataset/samplers/pointwise_pos_neg_sampler.py:24-48 (u uniform; a fair bit picks a train item
 * with label 1 or a non-train item with label 0), Philox stream.  eb_gmf_scale_rows: dst = src * h per column (scoring then
 * ranks plain dot products); eb_sigmoid_inplace: logits -> probabilities (-inf -> 0).
 * ------------------------------------------------------------------------ */
int eb_gmf_step_grads(const float *U, const float *I, int64_t ld, int f, const float *h, const int32_t *u, const int32_t *it,
                      const float *label, int64_t n, int64_t mean_over, float *dU, float *dI, float *dh, double *loss,
                      void *stream);
int eb_gmf_scale_rows(const float *src, int64_t ld, int64_t rows, int f, const float *h, float *dst, int64_t ldd, void *stream);
int eb_sigmoid_inplace(float *x, int64_t n, void *stream);
int eb_pointwise_sample_philox(int32_t n_users, int32_t n_items, const int64_t *csr_indptr, const int32_t *csr_indices,
                               const uint32_t *filter, int filter_words, int64_t n, uint64_t seed, uint64_t first,
                               int32_t *out_u, int32_t *out_i, float *out_label, void *stream);

/* ------------------------------------------------------------------------
 * Tables spread over the GPUs of one NVSwitch box, addressed DIRECTLY by the kernels (SURVEY.md §8e;
 * no reference counterpart: the reference is single-device).  One process per GPU: a rank allocates its
 * part with eb_peer_alloc (the one place this library allocates: the memory must be a plain cudaMalloc
 * block to be exportable; zero-filled), publishes its 64-byte CUDA IPC handle (eb_peer_export; the host
 * exchanges the handles, e.g. with torch.distributed.all_gather_object) and maps the other ranks' parts
 * (eb_peer_open, peer access enabled lazily).  `*_shards` / `slice_ptrs` arguments below are HOST arrays of
 * n device pointers, entry r = rank r's part as seen from the calling process (its own allocation for
 * r = own rank).  Row i of a sharded table lives in shard i / shard_rows at local row i % shard_rows.
 * ------------------------------------------------------------------------ */
#define EB_MAX_PEERS 8
int eb_peer_alloc(size_t bytes, void **dev_ptr);
int eb_peer_free(void *dev_ptr);
int eb_peer_export(const void *dev_ptr, void *handle64_host);
int eb_peer_open(const void *handle64_host, void **dev_ptr);
int eb_peer_close(void *dev_ptr);

/* BPR step (BPRMF_model.py:91-117 arithmetic, as eb_bpr_step_f32 / eb_bpr_step_sampled_f32) with the ITEM table and
 * item biases row-sharded over n_shards GPUs: user rows are local (a rank samples only for the users it owns,
 * custom_sampler.py:31-42 distribution over ITS users), item rows are loaded from and updated in their owner's
 * memory over NVLink (128-bit loads, system-scope red.add.v4.f32) inside the one training kernel — the
 * three all-to-alls of an NCCL formulation never happen.  ld in {32, 64, 128}. */
int eb_bpr_step_peer_f32(float *U, float *const *V_shards, float *const *b_shards, int n_shards, int32_t shard_rows,
                         int d, int ld, int32_t n_items, const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n,
                         float lr, float reg_u, float reg_b, float reg_pos, float reg_neg, double *loss, int flags,
                         void *stream);
int eb_bpr_step_sampled_peer_f32(float *U, float *const *V_shards, float *const *b_shards, int n_shards, int32_t shard_rows,
                                 int d, int ld, int32_t n_users, int32_t n_items, const int64_t *csr_indptr,
                                 const int32_t *csr_indices, const uint32_t *filter, int filter_words, int64_t n,
                                 uint64_t seed, uint64_t first_triple, float lr,
                                 float reg_u, float reg_b, float reg_pos, float reg_neg, double *loss, int32_t *out_u,
                                 int32_t *out_i, int32_t *out_j, int flags, void *stream);

/* REPLICATED table kept consistent without a collective: the caller owns one slice of the table; slice_ptrs[p] is
 * the address of that slice inside rank p's copy (n floats, n % 4 == 0), prev_slice the slice's last agreed value
 * (local, n floats).  One kernel: agreed = scale * sum_p (copy_p - prev); every copy += agreed - (copy_p - prev)
 * (vector atomics, so training kernels running on any copy at the same time lose nothing); prev += agreed.
 * scale = 1/n_peers averages the ranks' steps (local-SGD style), scale = 1 sums them.  max_ctas > 0 caps the grid
 * (to run beside a training kernel). */
int eb_table_reconcile_peer_f32(float *const *slice_ptrs, int n_peers, float *prev_slice, int64_t n, float scale,
                                int max_ctas, void *stream);

/* NeuMF (neural_matrix_factorization_model.py:74-106) with the two ITEM tables side by side in one row-sharded
 * [items, ldi >= 2f] table (row = [I_mf | I_mlp]) and user tables local: eb_neumf_gather / eb_neumf_scatter with the
 * item rows read from, and the item-row gradients added into, the owner's memory (GI_shards: the owners' dense
 * gradient shards, same layout). */
int eb_neumf_gather_peer(const float *Umf, const float *Umlp, int64_t ldu, float *const *I_shards, int n_shards,
                         int32_t shard_rows, int64_t ldi, int f, const int32_t *u, const int32_t *it, int64_t n, float *x0,
                         int64_t ldx, float *pm, int64_t ldp, void *stream);
int eb_neumf_scatter_peer(const float *Umf, int64_t ldu, float *const *I_shards, float *const *GI_shards, int n_shards,
                          int32_t shard_rows, int64_t ldi, int f, const int32_t *u, const int32_t *it, int64_t n,
                          const float *dpm, int64_t ldp, const float *dx0, int64_t ldx, float *dUmf, float *dUmlp,
                          void *stream);
/* Order a batch by the OWNER of the rows it touches before a peer kernel runs over it.  On 8 GPUs random rows fetched from 7
 * peers interleaved arrive at 44 GB/s, the same rows grouped by owner at 548 GB/s (tools/peer_fanout_probe.py); up to 3 peers
 * interleaved are fine.  a, b, c: up to three 32-bit arrays that travel together (b, c may be NULL with their outputs);
 * key1 (0..2) names the array of row ids, key2 (-1 or 0..2) an optional second one (BPR: positive and negative item).
 * Counting sort on ((owner - rank) mod world) — rank r starts at peer r+1, so no two ranks work on the same owner at the
 * same moment; order inside a group is arbitrary.  work: 128 int32 of device scratch.  world <= 8.  No reference
 * counterpart (the reference is single-process). */
int eb_group_by_owner_i32(const int32_t *a, const int32_t *b, const int32_t *c, int key1, int key2, int64_t n,
                          int32_t shard_rows, int rank, int world, int32_t *out_a, int32_t *out_b, int32_t *out_c,
                          int32_t *work, void *stream);
/* out[t][0..width) = row ids[t] of a sharded table (scoring over sharded item tables, tests) */
int eb_gather_rows_peer_f32(float *const *shards, int n_shards, int32_t shard_rows, int64_t ld, const int32_t *ids, int64_t n,
                            int width, float *out, int64_t ldo, void *stream);

/* Tensor-core path (wgmma + TMA, bf16 mainloop, exact fp32 re-rank).  Same contract and
 * same RESULT as eb_score_topk_f32 (identical index lists and scores): the kernel keeps the 32
 * best bf16-approximate candidates per user, re-scores them exactly in fp32 and certifies the
 * list with a rounding bound; users it cannot certify are re-done by the exact kernel inside
 * this call.  Contiguous user range only, k <= 16, d <= 256, mask rows sorted ascending.
 * dump (optional, tests): dense n_sel x n_items raw approximate scores.
 * stats_host (optional, host int64[16]): [0] users re-done exactly, [1] padded K, [2..15] cycle
 * counters of CTA 0 when the environment variable EB_TC_PROF is set (profiling aid).
 * Asynchronous unless stats_host is given (reading the statistics back is the only synchronisation): the exact
 * re-check runs over a device-side count.  K is padded to a multiple of 16 (full 64-column blocks with the 128-byte
 * swizzle plus one 16- or 32-column tail block with the 32-/64-byte swizzle), not to a multiple of 64. */
size_t eb_score_topk_tc_workspace_bytes(int64_t n_sel, int32_t n_items, int d);
int eb_score_topk_tc_f32(const float *U, const float *V, const float *item_bias, int32_t n_items, int d, int ld,
                         const int64_t *mask_indptr, const int32_t *mask_indices,
                         int32_t user_begin, int64_t n_sel, int k,
                         int32_t *out_idx, float *out_val, float *dump,
                         void *workspace, size_t workspace_bytes, int64_t *stats_host, void *stream);

/* ------------------------------------------------------------------------
 * ItemKNN / UserKNN, standard implementation (knn/item_knn/item_knn_similarity.py, knn/user_knn/user_knn_similarity.py).
 * eb_csr_to_dense_bf16: rows [row0, row0 + n_rows) of a CSR (values NULL: ones), times `scale`, into a bf16 matrix
 * [n_rows][ld] that the call zero-fills first; row_sq[r] / col_sq[c] (optional) receive the squared norms of the scaled
 * rows / columns.  With every scaled value an integer of magnitude <= 256 and every squared norm < 2^24, the operand is
 * exact and so is the Gram matrix eb_gemm_bf16 makes of it, and these norms are its diagonal.
 * eb_knn_neighbors_f32: per row s of a Gram slab (rows row0.. of G, n columns, row stride ld), replaces the row by its
 * similarity values, cosine = fp32((double)G_rc / sqrt((double)G_rr * (double)G_cc)) (0 when a norm is 0) or
 * dot = G_rc * dot_scale, and writes the k largest nonzero ones ordered by value desc, column asc: out_idx/out_val
 * [n_rows][k] (unused slots -1 / 0) and out_cnt[n_rows].  1 <= k <= 1024.
 * eb_knn_score_topk_f32: for output row q (user users[q], or user_begin + q when users is NULL) the scores
 * sum_j A[u, j] * B[j, :] over n_cols columns, each term rounded to a multiple of 2^-frac_bits and summed exactly in
 * int64 (the caller keeps max_u sum_j |A[u, j]| * max |B| * 2^frac_bits below 2^62), so the result does not depend on the
 * order of the sums; train items (mask CSR, rows sorted) are excluded; the k best by (score desc, column asc) go to
 * out_idx/out_val [n_sel][k], padded with -1 / -inf when fewer than k columns are unmasked.  B rows sorted by column.
 * The columns are processed in tiles of eb_knn_score_tile_cols() columns.  1 <= k <= 1024.
 * ------------------------------------------------------------------------ */
int eb_csr_to_dense_bf16(const int64_t *indptr, const int32_t *indices, const float *values, int32_t row0, int32_t n_rows,
                         int32_t n_cols, float scale, void *dst_bf16, int64_t ld, float *row_sq, float *col_sq, void *stream);
int eb_knn_neighbors_f32(float *slab, int64_t ld, int32_t n_rows, int32_t n, int32_t row0, const float *diag, int cosine,
                         float dot_scale, int k, int32_t *out_idx, float *out_val, int32_t *out_cnt, void *stream);
int eb_knn_score_tile_cols(void);
int eb_knn_score_topk_f32(const int64_t *a_indptr, const int32_t *a_indices, const float *a_values, const int64_t *b_indptr,
                          const int32_t *b_indices, const float *b_values, int32_t n_cols, const int64_t *mask_indptr,
                          const int32_t *mask_indices, const int32_t *users, int32_t user_begin, int64_t n_sel, int k,
                          int frac_bits, int32_t *out_idx, float *out_val, void *stream);

/* ------------------------------------------------------------------------
 * iALS / WRMF alternating least squares, fp64 (latent_factor_models/iALS/iALS_model.py:37-65,
 * latent_factor_models/WRMF/wrmf_model.py:41-58).  Tables are row-major fp64, 1 <= d <= 200.
 * eb_gram_f64: G[d][d] = Y^T Y over the n rows of Y (row stride ld).  The rows are split into a number of parts that
 * depends on n only, each summed in row order, and the parts are added in order, so the result is bit-reproducible.
 * workspace: at least eb_gram_f64_workspace_bytes(n, d) bytes, else EB_ERR_WORKSPACE.
 * eb_als_solve_f64: for s < n_rows and r = order[s], with the row's entries e in [indptr[r], indptr[r + 1]):
 *   A = G + sum_e w[e] y y^T + reg I,  b = sum_e c[e] y   (y = Y[indices[e]], row stride ld_y),
 *   X[r] = A^-1 b (Cholesky factorisation and two triangular solves; row stride ld_x, padding columns untouched).
 * Rows not listed in `order` are left untouched.  `order` only balances the load (longest rows first is best): the
 * result of a row does not depend on it, nor on which CTA solves it.  The rank-k updates run on the fp64 tensor cores.
 * d <= eb_als_small_d_max() solves one row per warp, larger d one row per CTA.  The call synchronises `stream`.  If a
 * pivot is <= 0 (A not positive definite) the row is not written and EB_ERR_DATA names the smallest such row.  Calls
 * must not run concurrently on one device (they share the status word).
 * ------------------------------------------------------------------------ */
size_t eb_gram_f64_workspace_bytes(int64_t n, int d);
int eb_gram_f64(const double *Y, int64_t n, int d, int64_t ld, double *G, void *workspace, size_t workspace_bytes,
                void *stream);
int eb_als_small_d_max(void);
int eb_als_solve_f64(const double *G, const double *Y, int64_t ld_y, int d, const int64_t *indptr, const int32_t *indices,
                     const double *w, const double *c, const int32_t *order, int64_t n_rows, double reg, double *X,
                     int64_t ld_x, void *stream);

/* ------------------------------------------------------------------------
 * EASE^R (autoencoders/EASE_R/ease_r.py:69-91) and the dense linear algebra it needs, fp64.
 * eb_inverse_f64: A[n][n] (row stride ld >= n; padding columns untouched) is replaced by its inverse.  Blocked
 * Gauss-Jordan elimination with partial pivoting: the pivot of a column is its largest |a| on or below the diagonal
 * (the lowest row on a tie); the trailing updates are fp64 tensor-core GEMMs.  Works for any nonsingular matrix, definite
 * or not.  Reruns are bit-identical.  workspace: at least eb_inverse_f64_workspace_bytes(n) bytes, else
 * EB_ERR_WORKSPACE.  A pivot that is exactly zero or not finite stops the call with EB_ERR_DATA naming the column (A is
 * then left partly transformed).  The call synchronises `stream`; calls must not run concurrently on one device (they
 * share the status word).  1 <= n <= 4 194 240.
 * eb_ease_normal_f64: rows row0 .. row0 + n_rows of EASE^R's normal matrix from the same rows of an fp32 Gram slab (row
 * stride ld_slab): A[i][j] = slab[i - row0][j] * scale for j != i and A[i][i] = (double)(float)(count[i] + l2_norm),
 * the fp64 sum rounded to fp32 as the reference stores it into its float32 matrix.
 * eb_ease_weights_f32: B[i][j] = (float)(-P[i][j] / P[j][j]) (one fp64 divide, one rounding) and B[j][j] = 0.  A zero
 * P[j][j] returns EB_ERR_DATA naming the smallest such j.  The call synchronises `stream`.
 * eb_dense_score_topk_f32: eb_knn_score_topk_f32 with a dense row-major B (row stride ldb): the same fixed-point terms,
 * mask and selection, so its output equals eb_knn_score_topk_f32's for the same B given as a CSR, bit for bit.
 * ------------------------------------------------------------------------ */
size_t eb_inverse_f64_workspace_bytes(int64_t n);
int eb_inverse_f64(double *A, int64_t n, int64_t ld, void *workspace, size_t workspace_bytes, void *stream);
int eb_ease_normal_f64(const float *slab, int64_t ld_slab, int32_t n_rows, int64_t n, int64_t row0, const int32_t *count,
                       double l2_norm, double scale, double *A, int64_t ld, void *stream);
int eb_ease_weights_f32(const double *P, int64_t ld_p, int64_t n, float *B, int64_t ld_b, void *stream);
int eb_dense_score_topk_f32(const int64_t *a_indptr, const int32_t *a_indices, const float *a_values, const float *b,
                            int64_t ldb, int32_t n_cols, const int64_t *mask_indptr, const int32_t *mask_indices,
                            const int32_t *users, int32_t user_begin, int64_t n_sel, int k, int frac_bits,
                            int32_t *out_idx, float *out_val, void *stream);

/* ------------------------------------------------------------------------
 * RP3beta (graph_based/RP3beta/rp3beta.py:73-176).  The float32 sparse products are SciPy's, bit for bit: output row r of
 * A . B is acc[c] = fp32(acc[c] + fp32(A[r, e] * B[e, c])) over A's row entries e in stored order (one rounded product,
 * one rounded add, no FMA, no atomics).  B's rows are sorted by column.  Output rows are visited in `order` (a
 * permutation of 0 .. n_sel - 1, NULL: ascending), which balances the load only.  Catalogues wider than
 * eb_rp3_tile_cols() columns are processed in column tiles and need a workspace of eb_rp3_row_workspace_bytes(n_cols)
 * bytes (0 otherwise), else EB_ERR_WORKSPACE.
 * eb_rp3_similarity_f32: row i of A . B (A = Piu, users ascending; B = Pui), each value times degree[c] in fp64 and the
 * diagonal zeroed; the min(k, n_items) largest nonzero fp64 values (ties: lowest column first) go to out_idx/out_val
 * [n_items][stride] as fp32, in column order, with out_cnt[n_items].
 * eb_rp3_l1_rows_f32: val[r][j] = fp32(val[r][j] / sum_j |val[r][j]|) for j < cnt[r], the sum in fp64 in stored order
 * (rows that sum to 0 are left alone).
 * eb_rp3_prune_cols_f32: W given as eb_rp3_similarity_f32's lists (nnz = sum of cnt); per column the k largest nonzero
 * values (ties: lowest row first) are kept and written as a CSR (out_indptr [n + 1], out_indices / out_values with room
 * for nnz entries, columns ascending in every row).  workspace: eb_rp3_prune_workspace_bytes(n, stride, nnz) bytes.
 * eb_rp3_score_topk_f32: for output row q (user users[q], or user_begin + q when users is NULL) the scores A[u] . B over
 * n_cols columns; train items (mask CSR) are excluded; the k best by (score desc, column asc) go to out_idx/out_val
 * [n_sel][k], padded with -1 / -inf when fewer than k columns are unmasked.  1 <= k <= 1024.
 * ------------------------------------------------------------------------ */
int eb_rp3_tile_cols(void);
size_t eb_rp3_row_workspace_bytes(int32_t n_cols);
int eb_rp3_similarity_f32(const int64_t *a_indptr, const int32_t *a_indices, const float *a_values, const int64_t *b_indptr,
                          const int32_t *b_indices, const float *b_values, const double *degree, int32_t n_items,
                          const int32_t *order, int k, int64_t stride, int32_t *out_idx, float *out_val, int32_t *out_cnt,
                          void *workspace, size_t workspace_bytes, void *stream);
int eb_rp3_l1_rows_f32(int32_t n_rows, int64_t stride, const int32_t *cnt, float *val, void *stream);
size_t eb_rp3_prune_workspace_bytes(int32_t n, int64_t stride, int64_t nnz);
int eb_rp3_prune_cols_f32(int32_t n, int64_t stride, const int32_t *cnt, const int32_t *idx, const float *val, int64_t nnz,
                          int k, int64_t *out_indptr, int32_t *out_indices, float *out_values, void *workspace,
                          size_t workspace_bytes, void *stream);
int eb_rp3_score_topk_f32(const int64_t *a_indptr, const int32_t *a_indices, const float *a_values, const int64_t *b_indptr,
                          const int32_t *b_indices, const float *b_values, int32_t n_cols, const int64_t *mask_indptr,
                          const int32_t *mask_indices, const int32_t *users, int32_t user_begin, int64_t n_sel,
                          const int32_t *order, int k, int32_t *out_idx, float *out_val, void *workspace,
                          size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------
 * SLIM (latent_factor_models/Slim/slim_model.py:44-113): per item p, sklearn's positive ElasticNet (fit_intercept=False,
 * selection='random') by sparse coordinate descent on X (CSC colptr/rows/vals, users ascending in every column; the CSR
 * pattern rowptr/cols gives user p's columns) with user row p read as zero and y = X[:, p].  l1 = fp32(alpha * l1_ratio *
 * n_users), l2 = fp32(alpha * (1 - l1_ratio) * n_users), tol (1e-4), seed: the xorshift state every fit starts from.
 * The coordinate updates reproduce the reference's float32 arithmetic; the gap's reductions run in fp64.
 * eb_slim_fit_f32 fits items item_begin .. item_begin + n_problems - 1, `slots` at a time (each slot holds one problem's
 * rows in the workspace, eb_slim_workspace_bytes(n_users, n_items, slots, shared_residual) bytes); the residual lives in
 * shared memory when shared_residual is 1 (eb_slim_shared_residual_fits(n_users)), otherwise in the workspace.
 * Outputs by item p: coef_t[i * n_items + p] = coefficient of item i, n_iter[p] (sklearn's n_iter_), gap[p] (sklearn's
 * dual_gap_), nnz[p] (nonzero coefficients) and drop[p]: the coefficient the min(nnz - 1, neighborhood) rule removes
 * when 1 <= nnz <= neighborhood (the smallest, ties: the highest item), else -1.  Requires n_items <= n_users.
 * eb_slim_slots: how many problems run at once on this device.
 * eb_slim_drop_f32: coef_t[drop[p] * n_items + p] = 0 wherever drop[p] >= 0.
 * ------------------------------------------------------------------------ */
int eb_slim_shared_residual_fits(int32_t n_users);
int eb_slim_slots(int32_t n_users, int shared_residual);
size_t eb_slim_workspace_bytes(int32_t n_users, int32_t n_items, int32_t slots, int shared_residual);
int eb_slim_fit_f32(const int64_t *colptr, const int32_t *rows, const float *vals, const int64_t *rowptr, const int32_t *cols,
                    int32_t n_users, int32_t n_items, int32_t item_begin, int32_t n_problems, float l1, float l2, float tol,
                    uint32_t seed, int max_iter, int neighborhood, int shared_residual, int32_t slots, float *coef_t,
                    int32_t *n_iter, float *gap, int32_t *nnz, int32_t *drop, void *workspace, size_t workspace_bytes,
                    void *stream);
int eb_slim_drop_f32(int32_t n_items, const int32_t *drop, float *coef_t, void *stream);

/* ------------------------------------------------------------------------
 * PureSVD (latent_factor_models/PureSVD/pure_svd_model.py:36-43: sklearn's randomized_svd), fp64.  Widths w and d are at
 * most eb_svd_max_width() (200, the limit of eb_gram_f64).
 * eb_csr_spmm_f64: Y[n_rows][w] (row stride ldy) = A X for a CSR A (int64 indptr, int32 indices, fp32 data) and X (row
 * stride ldx); element Y[r][c] is fma-summed over row r's entries in stored order from 0, so reruns are bit-identical.
 * Y must not be X.
 * eb_chol_pivoted_f64: for a symmetric positive semi-definite G[w][w] (G = X^T X), the Cholesky factorisation
 * P^T G P = L L^T with diagonal pivoting (the largest remaining diagonal entry; ties: the lowest index), stopped at the
 * first pivot <= w * 2^-52 * trace(G); writes M[w][w] = P L^-T with its columns past the numerical rank zero, and the rank
 * to *rank when rank is not NULL.  X M then has orthonormal columns spanning X's column space, followed by zero columns.
 * eb_tall_times_small_f64: Y[n][d] = X[n][w] M[w][d] (M row-major, row stride d), each element fma-summed over k in order.
 * Y may be X when d == w and ldy == ldx; otherwise they must not overlap.
 * eb_sym_eig_f64: eigenvalues (descending; ties: the lower diagonal index first) and eigenvectors (evecs[w][w], column k
 * for evals[k]) of a symmetric A[w][w], by cyclic Jacobi rotations in the parallel order; a pair is rotated while
 * |a_pq| > 2^-52 sqrt(|a_pp a_qq|) and |a_pq| > w 2^-52 sum_i |a_ii|.  workspace: at least
 * eb_sym_eig_f64_workspace_bytes(w) bytes, else EB_ERR_WORKSPACE.  The call synchronises `stream`; EB_ERR_DATA when it
 * does not converge.  Calls must not run concurrently on one device (they share the status word).
 * eb_svd_finish_f64: for k < d: s_out[k] = sqrt(max(evals[k], 0)); when scale_user_by_inv_s, user column k is
 * multiplied by 1 / s_out[k] (by 0 when evals[k] <= w * 2^-52 * sum_j max(evals[j], 0)) and item column k by s_out[k].
 * Then both columns are multiplied by the sign of the user column's largest-|.| entry (the first such row; +1 when the
 * column is zero), as sklearn's svd_flip does.
 * ------------------------------------------------------------------------ */
int eb_svd_max_width(void);
int eb_csr_spmm_f64(const int64_t *indptr, const int32_t *indices, const float *data, int64_t n_rows, const double *X, int w,
                    int64_t ldx, double *Y, int64_t ldy, void *stream);
int eb_chol_pivoted_f64(const double *G, int w, double *M, int32_t *rank, void *stream);
int eb_tall_times_small_f64(const double *X, int64_t n, int w, int64_t ldx, const double *M, int d, double *Y, int64_t ldy,
                            void *stream);
size_t eb_sym_eig_f64_workspace_bytes(int w);
int eb_sym_eig_f64(const double *A, int w, double *evals, double *evecs, void *workspace, size_t workspace_bytes, void *stream);
int eb_svd_finish_f64(const double *evals, int w, int d, double *user, int64_t n_user, int64_t ld_user, double *item,
                      int64_t n_item, int64_t ld_item, int scale_user_by_inv_s, double *s_out, void *stream);

/* ------------------------------------------------------------------------
 * SlopeOne (algebric/slope_one/slope_one_model.py:19-64), fp64.
 * eb_slope_one_dev_f64: for a row slab of the exact fp32 products F = B^T B, M1 = X^T B and M2 = B^T X (row stride
 * ld_in; X the ratings times 2^s, B the entry pattern, every entry an integer below 2^24), E[r][c] (row stride lde) =
 * ((double)M1 - (double)M2) * 2^-s / (double)F, divided with round-to-nearest, and NaN where F = 0.  0 <= s <= 30.
 * eb_slope_one_score_topk_f64: for output row q (user users[q], or user_begin + q when users is NULL), with the user's
 * train items j and ratings taken from the CSR indptr / items / ratings in stored order: mean = (sum of the ratings) / n
 * (the sum must be exact in fp64, as it is for ratings times 2^s that are integers), and for every item c the sum of
 * -E[j][c] over the j in stored order (sequential fp64 additions from 0, NaN entries skipped), divided by the number of
 * terms summed, plus the mean (the mean alone when there are none).  Items of the mask CSR (any order) are excluded; the
 * k best by (score desc, item asc) go to out_idx/out_val [n_sel][k], padded with -1 / -inf when fewer than k items are
 * left.  1 <= k <= 1024.  No workspace: the scores of one column tile live in shared memory.
 * ------------------------------------------------------------------------ */
int eb_slope_one_dev_f64(const float *F, const float *M1, const float *M2, int64_t ld_in, int32_t n_rows, int32_t n, int s,
                         double *E, int64_t lde, void *stream);
int eb_slope_one_score_topk_f64(const double *E, int64_t lde, int32_t n_items, const int64_t *indptr, const int32_t *items,
                                const float *ratings, const int64_t *mask_indptr, const int32_t *mask_indices,
                                const int32_t *users, int32_t user_begin, int64_t n_sel, int k, int32_t *out_idx,
                                double *out_val, void *stream);

/* ------------------------------------------------------------------------
 * NonNegMF (latent_factor_models/NonNegMF/non_negative_matrix_factorization_model.py:42-84), fp64, one epoch in three
 * steps; every product, sum and quotient is rounded on its own (no FMA), so the results equal the reference's bit for
 * bit.  The ratings k are those of a CSR indptr [n_users + 1] / items (users ascending, each user's items in the
 * reference's dict order); P [n_users][F] and Q [n_items][F] are dense with row stride F.
 * eb_nnmf_dots_f64: dots[k] = sum over f = 0..F-1 of Q[i][f] * P[u][f], summed in f order from +0.0.
 * eb_nnmf_bias_chain_f64: for k in order: est[k] = ((mu + bu[u]) + bi[i]) + dots[k], err = ratings[k] - est[k],
 *   bu[u] += lr * (err - reg * bu[u]), then bi[i] += lr * (err - reg * bi[i]).  bu and bi are updated in place; bu of a
 *   user without ratings is unchanged.  One thread walks the ratings; bi is staged in shared memory when n_items doubles
 *   fit the device's opt-in dynamic shared memory, and read and written in global memory otherwise.
 * eb_nnmf_row_update_f64: for every row r and f < F, over the row's entries e in stored order (k = pos[e], or e when
 *   pos is NULL): num = sum T[cols[e]][f] * ratings[k], den = sum T[cols[e]][f] * est[k], both from +0.0; then
 *   den += (n * reg) * S[r][f] with n the row's entry count, and S_out[r][f] = S[r][f] * (num / den) (IEEE inf / NaN
 *   when den is 0).  S_out may be S; it must not be T.  The user side passes the CSR above with T = Q, S = P; the item
 *   side the CSC (items' entries in ascending user order) with pos = each entry's k, T = P, S = Q.
 * ------------------------------------------------------------------------ */
int eb_nnmf_dots_f64(const double *P, const double *Q, int F, const int64_t *indptr, const int32_t *items, int32_t n_users,
                     double *dots, void *stream);
int eb_nnmf_bias_chain_f64(const int64_t *indptr, const int32_t *items, const double *ratings, const double *dots,
                           int32_t n_users, int32_t n_items, double mu, double lr, double reg, double *bu, double *bi,
                           double *est, void *stream);
int eb_nnmf_row_update_f64(const int64_t *indptr, const int32_t *cols, const int64_t *pos, int32_t n_rows,
                           const double *ratings, const double *est, const double *T, const double *S, double *S_out, int F,
                           double reg, void *stream);

/* ------------------------------------------------------------------------
 * SVD++ and FunkSVD (latent_factor_models/SVDpp/svdpp_model.py, FunkSVD/funk_svd_model.py) and the pair pass of the rating
 * metrics (evaluation/metrics/rating/{mae,mse,rmse}).  fp32 tables, row stride ld (multiple of 4), f % 4 == 0, f <= 128.
 * eb_rated_sample_philox: dataset/samplers/custom_pointwise_sparse_sampler.py:24-39 (u uniform, i uniform over u's train
 *   row, label = the train rating), the user and item draws of eb_bpr_sample_philox_filter's stream (counter first + t);
 *   csr_ratings [nnz] is aligned with the sorted train CSR.
 * eb_implicit_mean_f32: Z[r] (row stride ldz) = P[u] + (1/|N(u)|) sum_{j in N(u)} Y[j], N(u) = train row of u = users[r]
 *   (users NULL: u = r), fp32 sums of 128-bit row loads.
 * eb_rating_mf_step_f32: per sample s, out = z.q_i + b_u + b_i + g with z = Z[s] (SVD++) or P[u] (Z NULL: FunkSVD), g NULL
 *   for no global bias; loss += (out - y)^2 / mean_over (fp64 accumulator); the gradient e = 2 (out - y) / mean_over is
 *   added (vector atomics) to dQ[i] (e z), dP[u] (e q_i), dbu[u], dbi[i], dg[0] and, when dY is given (with Z and the train
 *   CSR), to dY[j] (e q_i / |N(u)|) for every j of u's train row.  The tables the dense Keras Adam then applies.
 * eb_score_pairs_f32: for every user w < n_users and relevant entry k of its row (rel CSR, rel_items -1 outside the
 *   catalogue): out[k] = (U[w].V[item] + item_bias[item]) + (user_off[w] + global_off[0]) (each term optional), -inf when
 *   item is in w's mask row (sorted), NaN when item = -1.  One warp per user.
 * eb_add_row_offset_f32: x[r][c] += row_off[r] + scalar_off[0] (scalar_off optional) for c < cols.
 * eb_rating_error_sums_f64: out[0] = sum |scores[e] - ratings[e]|, out[1] = sum (scores[e] - ratings[e])^2 over the
 *   entries with items[e] >= 0, in fp64, one CTA in a fixed order (the same bits every run).
 * ------------------------------------------------------------------------ */
int eb_rated_sample_philox(int32_t n_users, int32_t n_items, const int64_t *csr_indptr, const int32_t *csr_indices,
                           const float *csr_ratings, int64_t n, uint64_t seed, uint64_t first, int32_t *out_u, int32_t *out_i,
                           float *out_rating, void *stream);
int eb_implicit_mean_f32(const float *P, const float *Y, int64_t ld, int f, const int64_t *indptr, const int32_t *indices,
                         const int32_t *users, int64_t n, float *Z, int64_t ldz, void *stream);
int eb_rating_mf_step_f32(const float *P, const float *Q, int64_t ld, int f, const float *bu, const float *bi, const float *g,
                          const float *Z, int64_t ldz, const int64_t *indptr, const int32_t *indices, const int32_t *u,
                          const int32_t *it, const float *label, int64_t n, int64_t mean_over, float *dP, float *dQ, float *dY,
                          float *dbu, float *dbi, float *dg, double *loss, void *stream);
int eb_score_pairs_f32(const float *U, const float *V, int64_t ld, int f, const float *item_bias, const float *user_off,
                       const float *global_off, const int64_t *rel_indptr, const int32_t *rel_items, int32_t n_users,
                       const int64_t *mask_indptr, const int32_t *mask_indices, float *out, void *stream);
int eb_add_row_offset_f32(float *x, int64_t rows, int cols, int64_t ldx, const float *row_off, const float *scalar_off,
                          void *stream);
int eb_rating_error_sums_f64(const float *scores, const double *ratings, const int32_t *items, int64_t n, double *out,
                             void *stream);

/* ------------------------------------------------------------------------
 * CML (latent_factor_models/CML/CML_model.py:59-106), fp32 tables Gu, Gi (row stride ld, one of 8..256), Bi.
 * eb_cml_grad_f32 accumulates the gradient of the reference's broadcast B x B loss over n triples (see csrc/cml.cu):
 *   L = sum_a sum_b max(m - clip(D_a + E_b, -80, 1e8), 0) + l_w (|gu_a|^2 + |gi_a|^2 + |gj_a|^2)/2 + l_b bpos^2/2
 *       + l_b bneg^2/20,   D_a = |gu_a - gj_a|^2 - |gu_a - gi_a|^2,  E_b = Bi[pos_b] - Bi[neg_b]
 *   into dense gradient tables (duplicates summed), counting the active pairs (-80 < D_a + E_b <= m, fp64 sum of the fp32
 *   terms) by sorting instead of forming them.  loss (optional, device double[1]) += L.  terms [2n] receives D then E in
 *   triple order.  -80 < margin < 1e8; n < 2^31.  workspace: eb_cml_workspace_bytes(n) bytes, else EB_ERR_WORKSPACE.
 * eb_cml_score_operands_f32: U2 = 2 Gu (row stride ld), item_off[i] = Bi[i] - |Gi[i]|^2, user_off[u] = -|Gu[u]|^2, so
 *   that U2[u].Gi[i] + item_off[i] + user_off[u] = Bi[i] - |Gu[u] - Gi[i]|^2, the reference's predict.
 * ------------------------------------------------------------------------ */
size_t eb_cml_workspace_bytes(int64_t n);
int eb_cml_grad_f32(const float *Gu, const float *Gi, const float *Bi, float *dGu, float *dGi, float *dBi, int d, int ld,
                    const int32_t *tu, const int32_t *ti, const int32_t *tj, int64_t n, float l_w, float l_b, float margin,
                    float *terms, double *loss, void *workspace, size_t workspace_bytes, void *stream);
int eb_cml_score_operands_f32(const float *Gu, const float *Gi, const float *Bi, int ld, int32_t n_users, int32_t n_items,
                              float *U2, float *item_off, float *user_off, void *stream);

/* ------------------------------------------------------------------------
 * DMF (neural/DMF/deep_matrix_factorization_model.py), fp32.
 * eb_dmf_sparse_fwd_f32: h1[b][:H] = act(sum_p values[p] W1[indices[p]][:] + b1) over the CSR row rows[b] (act = ReLU
 *   if relu, else none); W1 [n_cols][H], H a multiple of 4 up to 1024, 16-byte aligned; row stride ldh; B < 2^31.
 * eb_dmf_sparse_bwd_f32: dW1[indices[p]][:] += values[p] dpre1[b][:] over the same rows (vector atomics).
 * eb_dmf_head_f32: one batch of B (user, item) tower outputs U, V [B][ld] (F columns) and ratings label[B].
 *   cosine: u^ = l2_normalize(U, axis 0) (each column over the batch: x / sqrt(max(sum_b x^2, 1e-12))), same for V;
 *   else u^ = U, v^ = V.  o_b = sum_f u^ v^, p_b = clip(o_b, 1e-7, 1 - 1e-7) (float32 bounds, as Keras), y_b = label_b / max_rating;
 *   loss (device double[1]) += mean_b -(y log(p + 1e-7) + (1 - y) log(1 - p + 1e-7)) (fp64, fixed order);
 *   dU, dV [B][ldg] = d mean / d(U, V) (clip passes the gradient on the closed interval; a column below the 1e-12
 *   floor gets only the direct term).  prob (optional) [B] = o.  F <= 256.  workspace: eb_dmf_head_workspace_bytes(B, F).
 * eb_dmf_score_operands_f32: tower outputs Uo [n_users] (stride ldu), Vo [n_items] (stride ldv) -> Uh [n_users][ld]
 *   with each user block [k block, (k+1) block) normalised by its own column norms, Vh [n_items][ld] = V / sqrt(max(
 *   block V^2, 1e-12)) and, when n_users % block != 0, Vh_last the same for the short last block (get_recs).  cosine = 0:
 *   Uh, Vh are Uo, Vo.  Padding columns [F, ld) are zero.  block > n_users means one block of every user.
 * ------------------------------------------------------------------------ */
int eb_dmf_sparse_fwd_f32(const float *W1, const float *b1, int H, const int64_t *indptr, const int32_t *indices,
                          const float *values, const int32_t *rows, int64_t B, int relu, float *h1, int64_t ldh,
                          void *stream);
int eb_dmf_sparse_bwd_f32(float *dW1, int H, const int64_t *indptr, const int32_t *indices, const float *values,
                          const int32_t *rows, int64_t B, const float *dpre1, int64_t ldd, void *stream);
size_t eb_dmf_head_workspace_bytes(int64_t B, int F);
int eb_dmf_head_f32(const float *U, const float *V, int64_t ld, int F, int64_t B, const float *label, float max_rating,
                    int cosine, double *loss, float *dU, float *dV, int64_t ldg, float *prob, void *workspace,
                    size_t workspace_bytes, void *stream);
int eb_dmf_score_operands_f32(const float *Uo, int64_t ldu, const float *Vo, int64_t ldv, int F, int32_t n_users,
                              int32_t n_items, int64_t block, int cosine, float *Uh, float *Vh, float *Vh_last, int64_t ld,
                              void *stream);

/* ------------------------------------------------------------------------
 * UserAutoRec / ItemAutoRec (neural/UserAutoRec/userautorec_model.py, neural/ItemAutoRec/itemautorec_model.py), fp32.
 * eb_autorec_decoder_f32: one training step's decoder and its backward over the OBSERVED entries of the batch rows
 *   rows[B] of the CSR (indptr, indices, values).  h [B][ldh] is the encoder output after its sigmoid, W2 [n_out][H] the
 *   decoder kernel stored output-major (Keras's [H][n_out] transposed), b2 [n_out]; act 0 = linear, 1 = sigmoid; scale =
 *   1 / B.  For every entry p of row rows[b], i = indices[p], x = values[p]:
 *     o = h_b . W2[i] + b2[i], r = act(o), e = x - r;  loss (device double[1]) += scale e^2 (fp64);
 *     g = -2 scale e act'(o);  dW2[i] += g h_b, db2[i] += g (vector / scalar reductions);  dh_b += g W2[i];
 *   then dpre1 [B][ldd] = dh ⊙ h ⊙ (1 - h) (an empty row gets 0).  dpre1 and the loss are combined in a fixed order (they
 *   do not depend on scheduling); dW2 / db2 may differ in the last bits from run to run.  H a multiple of 4 in [4, 1024];
 *   h, W2, dW2, dpre1 16-byte aligned.  The rows' entries must total at most max_entries (distinct rows of the CSR: its
 *   nnz).  workspace: eb_autorec_decoder_workspace_bytes(B, H, max_entries).  No host synchronisation.
 * ------------------------------------------------------------------------ */
size_t eb_autorec_decoder_workspace_bytes(int64_t B, int H, int64_t max_entries);
int eb_autorec_decoder_f32(const int64_t *indptr, const int32_t *indices, const float *values, const int32_t *rows, int64_t B,
                           int64_t max_entries, const float *h, int64_t ldh, const float *W2, const float *b2, int H, int act,
                           float scale, float *dW2, float *db2, float *dpre1, int64_t ldd, double *loss, void *workspace,
                           size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------
 * MostPop and Random (recommender/unpersonalized/most_popular/most_popular.py, random_recommender/Random.py).
 * The train CSR indptr [n_users + 1] / train (each row sorted ascending) is also the mask: a user's train items are
 * never listed.  Output row q is user users[q], or user_begin + q when users is NULL.
 * eb_item_pop: pop[i] = number of entries of item i among the nnz train indices (integer atomics; pop is zeroed first).
 * eb_mostpop_topk: order = every item by (pop desc, item asc).  Row q gets the first k items of that order outside the
 *   user's train row, out_val = their pop.  A user with |train_u| + k >= n_items gets a row of -1 (the reference lists
 *   nothing for it); *skipped (device int32) = the number of such rows.  Slots past the list: -1 / 0.  k >= 1.
 * eb_random_draws: the reference's np.random.randint(n_u) draws for every user in order (n_u = n_items - |train_u|,
 *   min(k, n_u) draws each, none when n_u <= 1), from the legacy MT19937 stream of eb_mt_seed / eb_mt_raw.  words
 *   [capacity] holds generated stream words; pos_host (HOST int64[2]) = (next unread word, words held) and is updated;
 *   when the held words run out, the buffer is refilled with the next `capacity` words of `state`.  r_out [n_users][k]
 *   gets the drawn values, -1 past min(k, n_u); *consumed_host (HOST) = the stream words this call used.  Synchronises
 *   the stream once per buffer's worth of words.  One warp walks the words: the walk is serial.
 * eb_complement_select: out[q][j] = the r-th (0-based) item outside the user's train row for r = r_in[u][j] (row u of
 *   [n_users][k]), -1 where r < 0.
 * ------------------------------------------------------------------------ */
int eb_item_pop(const int32_t *indices, int64_t nnz, int32_t n_items, int32_t *pop, void *stream);
int eb_mostpop_topk(const int32_t *order, const int32_t *pop, int32_t n_items, const int64_t *indptr, const int32_t *train,
                    const int32_t *users, int32_t user_begin, int64_t n_sel, int k, int32_t *out_idx, int32_t *out_val,
                    int32_t *skipped, void *stream);
size_t eb_random_workspace_bytes(void);
int eb_random_draws(uint32_t *state, uint32_t *words, int64_t capacity, int64_t *pos_host, int32_t n_users, int32_t n_items,
                    const int64_t *indptr, int k, int32_t *r_out, int64_t *consumed_host, void *workspace,
                    size_t workspace_bytes, void *stream);
int eb_complement_select(const int32_t *r_in, const int64_t *indptr, const int32_t *train, const int32_t *users,
                         int32_t user_begin, int64_t n_sel, int k, int32_t *out, void *stream);

#ifdef __cplusplus
}
#endif
#endif
