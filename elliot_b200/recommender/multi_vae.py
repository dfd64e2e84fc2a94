"""MultiVAE on the H100 behind the reference's model surface.

Mirrors elliot/recommender/autoencoders/vae/multi_vae.py:22-115 (params `intermediate_dim,
latent_dim, reg_lambda, lr, dropout_pkeep`, anneal schedule min(0.2, step/200000), per-epoch
shuffled user batches from sparse_sampler.py:13-25 — Python `random.seed(42)` stream, same as the
reference) and multi_vae_model.py:20-159.  Dense layers run on the tensor cores
(eb_gemm_bf16_tn, bf16 operands / fp32 accumulation); the I-wide input layer is a CSR gather-sum
and the dense B x I input batch of the reference is never built.  reg_lambda is accepted and inert,
as in the reference (its regulariser losses are never added, multi_vae_model.py:47-53 vs :136).
TensorFlow parity is UNPINNED (TF cannot run here); arithmetic is checked against
oracle/tf_models.py::multivae_forward_backward.
"""
import math
import os
import pickle
import random

import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import cuda_device, recs_dict


def _pad4(n):
    return (n + 3) // 4 * 4


class VariationalAutoEncoder:
    def __init__(self, original_dim, intermediate_dim, latent_dim, learning_rate, dropout_rate, regularization_lambda,
                 random_seed, indptr, indices, device):
        self.I, self.H, self.L = original_dim, intermediate_dim, latent_dim
        assert self.H % 8 == 0 and self.L % 8 == 0, "intermediate_dim and latent_dim must be multiples of 8 (TMA strides)"
        self.lr, self.drop, self.seed = learning_rate, float(dropout_rate), int(random_seed)
        self.indptr, self.indices, self.device = indptr, indices, torch.device(device)
        g = torch.Generator(device=self.device); g.manual_seed(self.seed)

        def glorot(rows, cols, fan_in, fan_out):       # GlorotNormal (truncated at 2 sigma), Keras layout [in][out] or [out][in]
            std = math.sqrt(2.0 / (fan_in + fan_out)) / 0.87962566103423978
            t = torch.empty((rows, cols), device=self.device)
            torch.nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=g)
            return t
        I, H, L = self.I, self.H, self.L
        Z = self._code_width()                         # 2L: mean | log-variance (one draw per Dense in the reference too)
        # W1 as [I][H] (gather-friendly); the other kernels as [out][in] = K-major GEMM B-operands
        self.P = {"W1": glorot(I, H, I, H), "b1": torch.zeros(_pad4(H), device=self.device),
                  "W2": glorot(Z, H, H, L), "b2": torch.zeros(_pad4(Z), device=self.device),
                  "W3": glorot(H, L, L, H), "b3": torch.zeros(_pad4(H), device=self.device),
                  "W4": glorot(I, H, H, I), "b4": torch.zeros(_pad4(I), device=self.device)}
        z = lambda t: torch.zeros_like(t)
        # gradients live in ONE flat buffer (views per parameter): data-parallel training all-reduces it in one call
        self._gflat = torch.zeros(sum(v.numel() for v in self.P.values()), device=self.device)
        self.G, off = {}, 0
        for k, v in self.P.items():
            self.G[k] = self._gflat[off:off + v.numel()].view_as(v); off += v.numel()
        self.dp, self._salt = None, 0
        self.native = True                                     # one native call per step phase (csrc/vae_step.cu)
        self.M = {k: z(v) for k, v in self.P.items()}
        self.V = {k: z(v) for k, v in self.P.items()}
        self.step = 0
        self._acc = torch.zeros(2, dtype=torch.float64, device=self.device)      # [kl_sum, nll_sum]
        self._refresh()

    def _code_width(self):
        return 2 * self.L

    def enable_data_parallel(self, group=None):
        """Replicated weights, batch split across the ranks of `group`, gradients averaged by one all-reduce
        (SURVEY.md §8e).  Every rank must be constructed with the same seed (same initial weights); the dropout and
        reparameterisation noise is salted with the rank so the slices draw independent noise."""
        import torch.distributed as dist
        from ..parallel import GradAllReduce
        self.dp = GradAllReduce(self._gflat, group, extra=self._acc)
        self._salt = 0x9E3779B1 * (dist.get_rank(group) if dist.is_initialized() else 0)

    def _refresh(self):
        """bf16 operand copies of the [out][in] weights (after every optimizer step); the buffers are allocated once so the
        native step can keep their addresses.  The backward GEMMs read the same copies as [K][N] matrices: there are no
        transposed copies."""
        P = self.P
        if not hasattr(self, "W2b"):
            self.W2b = self.W3b = self.W4b = None
        self.W2b, self.W3b, self.W4b = (ops.to_bf16(P["W2"], out=self.W2b), ops.to_bf16(P["W3"], out=self.W3b),
                                        ops.to_bf16(P["W4"], out=self.W4b))

    def _native_model(self):
        """The eb_vae_model struct (include/elliot_b200.h) over this model's tensors."""
        if getattr(self, "_cmodel", None) is None:
            self._cmodel = ops.vae_model_struct(self.I, self.H, self.L, self.P, self.G, self.M, self.V,
                                                (self.W2b, self.W3b, self.W4b),
                                                self.indptr, self.indices)
        return self._cmodel

    # ---- forward up to the logits (multi_vae_model.py:56-64,80-83,114-123)
    def _forward(self, rows, step_id, kl_sum=None, train=True):
        B, H, L, I = rows.numel(), self.H, self.L, self.I
        dev = self.device
        h1 = torch.empty((B, H), device=dev)
        ops.vae_embed_fwd(self.P["W1"], self.P["b1"], self.indptr, self.indices, rows, h1,
                          self.drop if train else 0.0, self.seed * 7919 + step_id + self._salt)
        ml = ops.gemm_bf16_tn(ops.to_bf16(h1), self.W2b, B, 2 * L, H, bias=self.P["b2"])
        z = torch.empty((B, L), device=dev)
        ops.vae_reparam_fwd(ml, L, z, self.seed + self._salt, step_id, kl_sum)
        h2 = ops.gemm_bf16_tn(ops.to_bf16(z), self.W3b, B, H, L, bias=self.P["b3"], act=1)
        logits = ops.gemm_bf16_tn(ops.to_bf16(h2), self.W4b, B, I, H, bias=self.P["b4"])
        return h1, ml, z, h2, logits

    def train_step(self, rows, anneal, global_batch=None):
        """rows: int32 device tensor of private user ids (data parallel: THIS rank's slice, possibly empty).
        global_batch: number of rows of the whole batch over all ranks (default: world x this slice).
        Returns the loss as a python float — the same value on every rank."""
        B, L = rows.numel(), self.L
        self.step += 1
        self._acc.zero_()
        if B > 0:
            self.compute_grads(rows, anneal, self.step)      # B == 0: the gradient buffer is already zero (Adam clears it)
        world = 1
        if self.dp is not None:
            import torch.distributed as dist
            world = dist.get_world_size(self.dp.group) if dist.is_initialized() else 1
            Bg = int(global_batch) if global_batch is not None else B * world
            self.dp.sync_weighted(B, Bg)                         # global-batch gradient (slices may be unequal or empty), loss terms summed
        else:
            Bg = B
        self.apply_grads()
        kl_sum, nll_sum = self._acc.tolist()
        return nll_sum / Bg + anneal * (-0.5 * kl_sum / (Bg * L))

    def compute_grads(self, rows, anneal, sid):
        """Forward + backward of one batch: gradients into self.G (views of one flat buffer), loss terms into _acc.
        native (default): one C-ABI call issues all ~33 kernels (eb_vae_train_step phase 1); the launch-by-launch
        Python sequence below is the same kernels in the same order and is kept as the readable specification
        (tests/test_gpu_multivae.py checks the two against each other)."""
        if self.native:
            ops.vae_train_step(self._native_model(), self.I, self.H, self.L, rows, self.drop, self.seed + self._salt,
                               self.seed * 7919 + sid + self._salt, sid, float(anneal), self.lr, self._acc, phase=1)
            return
        B, H, L, I = rows.numel(), self.H, self.L, self.I
        h1, ml, z, h2, logits = self._forward(rows, sid, self._acc[0:1])
        ops.vae_softmax(logits, self.indptr, self.indices, rows, nll_sum=self._acc[1:2], write_grad=True)
        dlogits = logits                                                       # in place
        # backward GEMMs read the row-major bf16 copies as they lie ("rows are K" operands): no transposed copies
        dl_b, G = ops.to_bf16(dlogits), self.G
        h1_b, z_b, h2_b = ops.to_bf16(h1), ops.to_bf16(z), ops.to_bf16(h2)
        ops.gemm_bf16(dl_b, h2_b, I, H, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W4"])
        ops.colsum(dlogits, G["b4"])
        dh2 = ops.gemm_bf16(dl_b, self.W4b, B, H, I, b_rows_are_k=True)
        dpre2 = ops.tanh_bwd(dh2, h2)
        dpre2_b = ops.to_bf16(dpre2)
        ops.gemm_bf16(dpre2_b, z_b, H, L, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W3"])
        ops.colsum(dpre2, G["b3"])
        dz = ops.gemm_bf16(dpre2_b, self.W3b, B, L, H, b_rows_are_k=True)
        dml = torch.empty((B, 2 * L), device=self.device)
        ops.vae_reparam_bwd(ml, L, dz, dml, self.seed + self._salt, sid, float(anneal))
        dml_b = ops.to_bf16(dml)
        ops.gemm_bf16(dml_b, h1_b, 2 * L, H, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W2"])
        ops.colsum(dml, G["b2"])
        dh1 = ops.gemm_bf16(dml_b, self.W2b, B, H, 2 * L, b_rows_are_k=True)
        dpre1 = ops.tanh_bwd(dh1, h1)
        ops.colsum(dpre1, G["b1"])
        ops.vae_embed_bwd(G["W1"], self.indptr, self.indices, rows, dpre1, self.drop, self.seed * 7919 + sid + self._salt)

    def apply_grads(self):
        """Keras Adam on every parameter (clears the gradients), then refresh the bf16 operand copies."""
        if self.native:
            ops.vae_train_step(self._native_model(), self.I, self.H, self.L, None, self.drop, 0, 0, self.step, 0.0, self.lr,
                               self._acc, phase=2)
            return
        for k in ("W1", "b1", "W2", "b2", "W3", "b3", "W4", "b4"):
            ops.adam_dense_f32(self.P[k], self.M[k], self.V[k], self.G[k], self.lr, self.step)
        self._refresh()

    def predict_topk(self, rows, k, mask_indptr, mask_indices):
        """log_softmax(decoder(z)) with the train mask -> top-k (multi_vae_model.py:144-159); note the
        reference samples z at predict time too (Sampling has no training guard, :63)."""
        self._pred_calls = getattr(self, "_pred_calls", 0) + 1
        _, _, _, _, logits = self._forward(rows, (1 << 40) + self._pred_calls, None, train=False)
        lse = torch.empty(rows.numel(), device=self.device)
        ops.vae_softmax(logits, self.indptr, self.indices, rows, lse_out=lse, write_grad=False)
        return ops.dense_topk(logits, k, mask_indptr, mask_indices, rows, shift=-lse)

    def get_model_state(self):
        return {"P": {k: v.cpu().numpy() for k, v in self.P.items()}, "step": self.step,
                "M": {k: v.cpu().numpy() for k, v in self.M.items()}, "V": {k: v.cpu().numpy() for k, v in self.V.items()}}

    def set_model_state(self, s):
        for k in self.P:
            self.P[k].copy_(torch.from_numpy(s["P"][k])); self.M[k].copy_(torch.from_numpy(s["M"][k])); self.V[k].copy_(torch.from_numpy(s["V"][k]))
        self.step = s["step"]; self._refresh()

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))


def epoch_user_order(num_users):
    """One epoch's user order: `random.sample(range(users), users)` on the global `random` stream seeded with 42
    at construction (sparse_sampler.py:10,18); pinned by tests/golden/samplers_tiny.npz."""
    return random.sample(range(num_users), num_users)


class MultiVAE(RecMixin, BaseRecommenderModel):
    r"""Variational Autoencoders for Collaborative Filtering (https://dl.acm.org/doi/10.1145/3178876.3186150).
    YAML keys as in the reference (multi_vae.py:42-52)."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_intermediate_dim", "intermediate_dim", "intermediate_dim", 600, int, None),
            ("_latent_dim", "latent_dim", "latent_dim", 200, int, None),
            ("_lambda", "reg_lambda", "reg_lambda", 0.01, None, None),
            ("_learning_rate", "lr", "lr", 0.001, None, None),
            ("_dropout_rate", "dropout_pkeep", "dropout_pkeep", 1, None, None),
        ]
        self.autoset_params()
        random.seed(42)                                              # sparse_sampler.py:10
        if self._batch_size < 1:
            self._batch_size = self._num_users
        self._dropout_rate = 1. - self._dropout_rate
        # b200_dp: true (under torchrun) -> data parallel: replicated weights, every batch split across the ranks,
        # gradients averaged by one all-reduce per step (SURVEY.md §8e); each rank drives the GPU of its LOCAL_RANK
        self._dp = bool(getattr(self._params, "b200_dp", False))
        default_dev = f"cuda:{os.environ.get('LOCAL_RANK', '0')}" if self._dp else "cuda:0"
        self._device = cuda_device(self._params, "MultiVAE", default_dev)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
        self._model = VariationalAutoEncoder(self._num_items, self._intermediate_dim, self._latent_dim, self._learning_rate,
                                             self._dropout_rate, self._lambda, self._seed, self._indptr, self._sorted_idx,
                                             self._device)
        self._total_anneal_steps = 200000
        self._anneal_cap = 0.2
        if self._dp:
            import torch.distributed as dist
            if not dist.is_initialized():
                raise Exception("b200_dp needs an initialised torch.distributed process group (launch with torchrun)")
            self._model.enable_data_parallel()

    @property
    def name(self):
        return "MultiVAE" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        self._update_count = 0
        for it in self.iterate(self._epochs):
            loss = 0
            order = epoch_user_order(self._num_users)
            order = torch.tensor(order, dtype=torch.int32, device=self._device)
            for s in range(0, self._num_users, self._batch_size):
                rows = order[s:s + self._batch_size].contiguous()
                n_batch = rows.numel()
                if self._dp:                                     # this rank's slice of the batch: sizes differ by <= 1, and a
                    import torch.distributed as dist             # tail batch smaller than the world leaves some ranks EMPTY
                    from ..parallel import shard_range
                    lo, hi = shard_range(n_batch, dist.get_rank(), dist.get_world_size())
                    rows = rows[lo:hi].contiguous()
                anneal = min(self._anneal_cap, 1. * self._update_count / self._total_anneal_steps) \
                    if self._total_anneal_steps > 0 else self._anneal_cap
                loss += self._model.train_step(rows, anneal, global_batch=n_batch)
                self._update_count += 1
            self.evaluate(it, loss / (it + 1))

    def get_recommendations(self, k: int = 100):
        if self._negative_sampling:
            raise NotImplementedError("evaluation-time negative sampling masks are outside this build's hot-path scope")
        out = {}
        for offset in range(0, self._num_users, self._batch_size):              # recommender_utils_mixin.py:63-73
            stop = min(offset + self._batch_size, self._num_users)
            rows = torch.arange(offset, stop, dtype=torch.int32, device=self._device)
            recs_dict(self._data, *self._model.predict_topk(rows, k, self._indptr, self._sorted_idx), first=offset, out=out)
        return out, out
