"""NeuMF on the H100 behind the reference's model surface.

Mirrors elliot/recommender/neural/NeuMF/neural_matrix_factorization.py:24-124 (params `mf_factors, lr, dropout,
is_mf_train, is_mlp_train, m`; MLP sizes forced to (4f, 2f, f) and mlp_factors = f, :71-72; pointwise BCE,
NOT BPR) and neural_matrix_factorization_model.py:18-148.  Embedding gathers / scatter-adds are CUDA-core
kernels, the MLP runs on the tensor cores (eb_gemm_bf16_tn), every variable is moved by dense Keras Adam.
get_recommendations evaluates the full MLP for every (user, item) pair of a user block like the reference
(:109-124), with the first layer factorised into per-user and per-item pre-activations.
Scope notes: dropout must be 0 (the reference default), both branches trained; f must be a multiple of 8.
The sampler draws the reference's distribution (each train pair once with label 1 + m uniform non-train
items with label 0, shuffled) from a Philox stream; the reference's np.random/`random`/set-order stream is
not replayed (its set-of-tuples iteration order is an implementation detail of CPython's tuple hash).
TensorFlow parity is UNPINNED (oracle/tf_models.py::neumf_forward_backward is the checker).
"""
import math
import pickle
import random

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import cuda_device, recs_dict


class ReferenceSampler:
    """Host replay of the reference's pointwise sampler (neural/NeuMF/custom_sampler.py:14-48): legacy
    np.random.seed(42) + random.seed(42); per epoch the SET of positives (u, i, 1), for each positive (in the
    set's iteration order) m negatives drawn with np.random.randint and redrawn while they hit a train item,
    collected in a SET (duplicates collapse), then `random.sample` shuffles positives + negatives.  The order
    depends on CPython's set iteration order for int tuples, so it has to run in Python like the reference;
    pinned by tests/golden/samplers_tiny.npz.  `b200_sampler: reference` selects it (small data only)."""

    def __init__(self, i_train_dict, m):
        np.random.seed(42)
        random.seed(42)
        self._rows = {u: list(set(i_train_dict[u])) for u in i_train_dict}
        self._n_items = len({k for a in i_train_dict.values() for k in a.keys()})
        self._m = m

    def epoch(self):
        draw, n_items = np.random.randint, self._n_items
        positives = {(u, i, 1) for u, items in self._rows.items() for i in items}
        negatives = set()
        for u, _, _ in positives:
            mine = self._rows[u]
            for _ in range(self._m):
                j = draw(n_items)
                while j in mine:
                    j = draw(n_items)
                negatives.add((u, j, 0))
        samples = list(positives)
        samples.extend(list(negatives))
        samples = random.sample(samples, len(samples))
        arr = np.array(samples, dtype=np.int64).reshape(-1, 3)
        return arr[:, 0], arr[:, 1], arr[:, 2]


class NeuralMatrixFactorizationModel:
    def __init__(self, num_users, num_items, f, learning_rate, random_seed, device):
        assert f % 8 == 0 and 8 <= f <= 128, "mf_factors must be a multiple of 8 in [8, 128] for the tensor-core path"
        self.nu, self.ni, self.f, self.lr = num_users, num_items, f, learning_rate
        self.device = torch.device(device)
        g = torch.Generator(device=self.device); g.manual_seed(int(random_seed))

        def glorot(rows, cols, fan_in, fan_out):                      # GlorotUniform (:38), Keras Dense default
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            return (torch.rand((rows, cols), device=self.device, generator=g) * 2 - 1) * lim
        z = lambda n: torch.zeros((n + 3) // 4 * 4, device=self.device)
        self.P = {"U_mf": glorot(num_users, f, num_users, f), "I_mf": glorot(num_items, f, num_items, f),
                  "U_mlp": glorot(num_users, f, num_users, f), "I_mlp": glorot(num_items, f, num_items, f),
                  "W1": glorot(4 * f, 2 * f, 2 * f, 4 * f), "b1": z(4 * f),     # Dense kernels kept [out][in]
                  "W2": glorot(2 * f, 4 * f, 4 * f, 2 * f), "b2": z(2 * f),
                  "W3": glorot(f, 2 * f, 2 * f, f), "b3": z(f),
                  "wp": glorot(1, 2 * f, 2 * f, 1).reshape(-1).contiguous(), "bp": z(1)}
        zl = lambda t: torch.zeros_like(t)
        self.G = {k: zl(v) for k, v in self.P.items()}
        self.M = {k: zl(v) for k, v in self.P.items()}
        self.V = {k: zl(v) for k, v in self.P.items()}
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        self._refresh()

    def _refresh(self):
        P = self.P
        self.Wb = {k: ops.to_bf16(P[k]) for k in ("W1", "W2", "W3")}

    def _mlp(self, x0):
        f, B = self.f, x0.shape[0]
        x0b = ops.to_bf16(x0)
        # each layer's epilogue writes the bf16 operand copy of its output beside the fp32 activations
        h1, h1b = ops.gemm_bf16_tn(x0b, self.Wb["W1"], B, 4 * f, 2 * f, bias=self.P["b1"], act=2, out_bf16=True)
        h2, h2b = ops.gemm_bf16_tn(h1b, self.Wb["W2"], B, 2 * f, 4 * f, bias=self.P["b2"], act=2, out_bf16=True)
        h3 = ops.gemm_bf16_tn(h2b, self.Wb["W3"], B, f, 2 * f, bias=self.P["b3"], act=2)
        self._act_b = (x0b, h1b, h2b)                     # row-major bf16 copies, read again ("rows are K") by the weight-gradient GEMMs
        return h1, h2, h3

    def train_step(self, batch):
        """batch = (user int32, item int32, label float32) device tensors; returns the batch loss tensor."""
        u, it, y = batch
        f, B, P, G = self.f, u.numel(), self.P, self.G
        dev = self.device
        x0 = torch.empty((B, 2 * f), device=dev); pm = torch.empty((B, f), device=dev)
        ops.neumf_gather(P["U_mf"], P["I_mf"], P["U_mlp"], P["I_mlp"], f, u, it, x0, pm)
        h1, h2, h3 = self._mlp(x0)
        dpm = torch.empty_like(pm); dpre3 = torch.empty_like(h3)
        self._loss.zero_()
        ops.neumf_head(pm, h3, f, P["wp"], P["bp"], label=y, dpm=dpm, dh3=dpre3, dwp=G["wp"], dbp=G["bp"], loss=self._loss)
        # backward: dW = dY^T . X contracts over the batch rows of both row-major operands, dX = dY . W reads the [out][in] kernel as
        # a [K][N] matrix — "rows are K" operands of eb_gemm_bf16, no transposed copies of activations or weights
        x0b, h1b, h2b = self._act_b
        d3b = ops.to_bf16(dpre3)
        ops.gemm_bf16(d3b, h2b, f, 2 * f, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W3"]); ops.colsum(dpre3, G["b3"])
        dpre2, d2b = ops.relu_bwd(ops.gemm_bf16(d3b, self.Wb["W3"], B, 2 * f, f, b_rows_are_k=True), h2, copy_bf16=True)
        ops.gemm_bf16(d2b, h1b, 2 * f, 4 * f, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W2"]); ops.colsum(dpre2, G["b2"])
        dpre1, d1b = ops.relu_bwd(ops.gemm_bf16(d2b, self.Wb["W2"], B, 4 * f, 2 * f, b_rows_are_k=True), h1, copy_bf16=True)
        ops.gemm_bf16(d1b, x0b, 4 * f, 2 * f, B, a_rows_are_k=True, b_rows_are_k=True, out=G["W1"]); ops.colsum(dpre1, G["b1"])
        dx0 = ops.gemm_bf16(d1b, self.Wb["W1"], B, 2 * f, 4 * f, b_rows_are_k=True)
        ops.neumf_scatter(P["U_mf"], P["I_mf"], f, u, it, dpm, dx0, G["U_mf"], G["I_mf"], G["U_mlp"], G["I_mlp"])
        self.step += 1
        for k in P:
            ops.adam_dense_f32(P[k], self.M[k], self.V[k], G[k], self.lr, self.step)
        self._refresh()
        return self._loss

    def get_recs_topk(self, u0, u1, k, mask_indptr, mask_indices):
        """sigmoid outputs for users [u0, u1) x all items -> masked top-k (get_recs/get_top_k, :119-148)."""
        f, P, ni, nb = self.f, self.P, self.ni, u1 - u0
        W1u = self.Wb["W1"][:, :f]; W1i = self.Wb["W1"][:, f:2 * f]                       # column halves of the first kernel
        Au = ops.gemm_bf16_tn(ops.to_bf16(P["U_mlp"][u0:u1]), W1u, nb, 4 * f, f)
        if getattr(self, "_Ai_step", None) != self.step:
            self._Ai = ops.gemm_bf16_tn(ops.to_bf16(P["I_mlp"]), W1i, ni, 4 * f, f); self._Ai_step = self.step
        pairs = nb * ni
        h1 = torch.empty((pairs, 4 * f), dtype=self.Wb["W2"].dtype, device=self.device)       # bf16 (fp32 in checking mode)
        ops.neumf_pair_h1(Au, self._Ai, P["b1"], nb, ni, 4 * f, h1)
        h2 = ops.gemm_bf16_tn(h1, self.Wb["W2"], pairs, 2 * f, 4 * f, bias=P["b2"], act=2)
        h3 = ops.gemm_bf16_tn(ops.to_bf16(h2), self.Wb["W3"], pairs, f, 2 * f, bias=P["b3"], act=2)
        prob = torch.empty((nb, ni), device=self.device)
        ops.neumf_pair_head(P["U_mf"], P["I_mf"], f, u0, nb, ni, h3, P["wp"], P["bp"], prob)
        rows = torch.arange(u0, u1, dtype=torch.int32, device=self.device)
        return ops.dense_topk(prob, k, mask_indptr, mask_indices, rows)

    def get_model_state(self):
        return {"P": {k: v.cpu().numpy() for k, v in self.P.items()}, "step": self.step,
                "M": {k: v.cpu().numpy() for k, v in self.M.items()}, "V": {k: v.cpu().numpy() for k, v in self.V.items()}}

    def set_model_state(self, s):
        for k in self.P:
            self.P[k].copy_(torch.from_numpy(s["P"][k])); self.M[k].copy_(torch.from_numpy(s["M"][k])); self.V[k].copy_(torch.from_numpy(s["V"][k]))
        self.step = s["step"]; self._refresh()

    def save_weights(self, path):
        with open(path, "wb") as fh:
            pickle.dump(self.get_model_state(), fh)

    def load_weights(self, path):
        with open(path, "rb") as fh:
            self.set_model_state(pickle.load(fh))


class NeuMF(RecMixin, BaseRecommenderModel):
    r"""Neural Collaborative Filtering (https://arxiv.org/abs/1708.05031).  YAML keys as in the reference."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_learning_rate", "lr", "lr", 0.001, None, None),
            ("_mf_factors", "mf_factors", "mffactors", 10, int, None),
            ("_dropout", "dropout", "drop", 0, None, None),
            ("_is_mf_train", "is_mf_train", "mftrain", True, None, None),
            ("_is_mlp_train", "is_mlp_train", "mlptrain", True, None, None),
            ("_m", "m", "m", 0, int, None),
        ]
        self.autoset_params()
        self._mlp_hidden_size = (self._mf_factors * 4, self._mf_factors * 2, self._mf_factors)     # :71
        self._mlp_factors = self._mf_factors
        if self._batch_size < 1:
            self._batch_size = self._data.transactions
        if self._dropout or not (self._is_mf_train and self._is_mlp_train):
            raise NotImplementedError("elliot_b200.NeuMF covers the default configuration: dropout 0, both branches trained")
        self._device = cuda_device(self._params, "NeuMF")
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
        self._model = NeuralMatrixFactorizationModel(self._num_users, self._num_items, self._mf_factors, self._learning_rate,
                                                     self._seed, self._device)
        self._gen = torch.Generator(device=self._device); self._gen.manual_seed(42)
        self._epoch = 0
        self._sampler_kind = getattr(self._params, "b200_sampler", "device")
        if self._sampler_kind not in ("device", "reference"):
            raise Exception("b200_sampler must be 'device' or 'reference'")
        self._ref_sampler = ReferenceSampler(self._data.i_train_dict, self._m) if self._sampler_kind == "reference" else None

    @property
    def name(self):
        return "NeuMF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        for it in self.iterate(self._epochs):
            loss, steps = 0.0, 0
            if self._ref_sampler is not None:                   # exact replay of the reference's epoch sample list
                hu, hi, hy = self._ref_sampler.epoch()
                u = torch.from_numpy(hu.astype(np.int32)).to(self._device); i = torch.from_numpy(hi.astype(np.int32)).to(self._device)
                y = torch.from_numpy(hy.astype(np.float32)).to(self._device)
            else:
                u, i, y = ops.neumf_sample(self._num_users, self._num_items, self._indptr, self._sorted_idx, self._m,
                                           42 + 1000003 * self._epoch)
                perm = torch.randperm(u.numel(), device=self._device, generator=self._gen)        # random.sample shuffle (:44)
                u, i, y = u[perm].contiguous(), i[perm].contiguous(), y[perm].contiguous()
            self._epoch += 1
            for s in range(0, u.numel(), self._batch_size):
                e = min(s + self._batch_size, u.numel())
                loss += float(self._model.train_step((u[s:e], i[s:e], y[s:e])).item()); steps += 1
            self.evaluate(it, loss / (it + 1))

    def get_recommendations(self, k: int = 100):
        if self._negative_sampling:
            raise NotImplementedError("evaluation-time negative sampling masks are outside this build's hot-path scope")
        out = {}
        f = self._mf_factors
        block = max(1, min(self._batch_size, (256 << 20) // max(1, self._num_items * 4 * f * 2)))   # <= 256 MB of layer-1 operand
        for u0 in range(0, self._num_users, block):
            u1 = min(u0 + block, self._num_users)
            recs_dict(self._data, *self._model.get_recs_topk(u0, u1, k, self._indptr, self._sorted_idx), first=u0, out=out)
        return out, out
