"""MF2020 — pointwise logistic matrix factorisation ("Neural Collaborative Filtering vs. Matrix Factorization
Revisited") on the H100: a sibling of BPRMF on the same gather / dot / scatter shape (SURVEY.md §8f #3).

Mirrors elliot/recommender/latent_factor_models/MF2020/MF.py:22-146 (class MF2020: `_params_list` keys/defaults
factors 10, lr 0.05, reg 0, m 0; name; train(); get_recommendations()), MF_model.py:14-174 (MFModel: init stream,
state dict incl. `_global_bias`, pickle weights) and custom_sampler_rendle.py:14-85 (the epoch sample list).

`b200_mode: exact` (default): the reference's run, reproduced — same init stream, the same epoch sample lists
(host: numpy's legacy stream for the negatives, Python's `random.sample` for the permutation, through private
generator objects seeded like the reference seeds the global ones), updates applied in the reference's order in
fp64 by `eb_mf_pointwise_exact_f64`, top-k by the exact fp64 scoring kernel.
`b200_mode: hogwild`: fp32 throughput mode, one fused launch per epoch (`eb_mf_pointwise_step_f32`), tensor-core
scoring; same distribution of samples, different stream.
"""
import pickle
import random

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger


class RendleSampler:
    """custom_sampler_rendle.Sampler: positives in `sp_i_train.nonzero()` order, each followed by m uniform items
    (label 0, not rejected against the train set), the whole list permuted by `random.sample` once per epoch."""

    def __init__(self, sparse_matrix, m, seed, np_stream):
        self._m = m
        rows, cols = sparse_matrix.nonzero()                          # custom_sampler_rendle.py:25-27
        self.pos_u, self.pos_i = rows.astype(np.int32), cols.astype(np.int32)
        self._nitems = len(set(self.pos_i.tolist()))                  # :20-21 distinct train items
        self._np = np_stream                                          # the process-wide legacy numpy stream (shared with init)
        self._py = random.Random(seed)                                # random.seed(seed) (:17)

    def epoch(self):
        n, m = len(self.pos_u), self._m
        mat = np.empty((n * (1 + m), 3), dtype=np.int32)
        mat[::1 + m, 0] = self.pos_u; mat[::1 + m, 1] = self.pos_i; mat[::1 + m, 2] = 1
        if m:
            neg = self._np.randint(self._nitems, size=n * m).reshape(n, m)      # one randint per negative, in order (:66-69)
            for q in range(m):
                mat[1 + q::1 + m, 0] = self.pos_u; mat[1 + q::1 + m, 1] = neg[:, q]; mat[1 + q::1 + m, 2] = 0
        return mat[self._py.sample(range(len(mat)), len(mat))]         # :80-81


class MF2020Model:
    """Device-resident tables with the reference MFModel's interface subset (MF_model.py:14-174)."""

    def __init__(self, F, data, lr, reg, random_seed, mode="exact", device="cuda:0"):
        self._factors, self._data, self._lr, self._reg, self._mode = F, data, lr, reg, mode
        self.device = torch.device(device)
        self.np_stream = np.random.RandomState(random_seed)           # np.random.seed(random_seed) (MF_model.py:21)
        nu, ni = len(data.users), len(data.items)
        U0 = self.np_stream.normal(loc=0, scale=0.1, size=(nu, F))    # MF_model.py:47-50: U first, then V
        V0 = self.np_stream.normal(loc=0, scale=0.1, size=(ni, F))
        self.set_model_state({"_global_bias": 0, "_user_bias": np.zeros(nu), "_item_bias": np.zeros(ni),
                              "_user_factors": U0, "_item_factors": V0})

    @property
    def name(self):
        return "MF2020"

    def set_model_state(self, s):
        F = self._factors
        dt = torch.float64 if self._mode == "exact" else torch.float32
        self.ld = F if self._mode == "exact" else ops.padded_dim(F)
        to = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(self.device, dt)
        nu, ni = s["_user_factors"].shape[0], s["_item_factors"].shape[0]
        self.U = torch.zeros((nu, self.ld), dtype=dt, device=self.device); self.U[:, :F] = to(s["_user_factors"])
        self.V = torch.zeros((ni, self.ld), dtype=dt, device=self.device); self.V[:, :F] = to(s["_item_factors"])
        self.ub, self.ib = to(s["_user_bias"]).contiguous(), to(s["_item_bias"]).contiguous()
        self.gb = torch.tensor([float(s["_global_bias"])], dtype=dt, device=self.device)

    def get_model_state(self):
        F = self._factors
        return {"_global_bias": float(self.gb.item()), "_user_bias": self.ub.double().cpu().numpy(),
                "_item_bias": self.ib.double().cpu().numpy(), "_user_factors": self.U[:, :F].double().cpu().numpy(),
                "_item_factors": self.V[:, :F].double().cpu().numpy()}

    def train_step(self, batch, batch_loss=None):
        """batch: (n, 3) int32 rows (user, item, label) in the order to apply (MF_model.py:80-112)."""
        t = torch.from_numpy(np.ascontiguousarray(batch.T)).to(self.device)
        ops.mf_pointwise_exact_f64(self.U, self.V, self.ub, self.ib, self.gb, self._factors, t[0], t[1], t[2],
                                   self._lr, self._reg, batch=100000, batch_loss=batch_loss)

    def topk(self, k, mask_indptr, mask_indices):
        """Scores gb + ub[u] + ib[i] + U[u].V[i] (MF_model.py:113-114); the per-user constant does not change the
        ranking, so the kernels rank ib + U.V and the constant is added to the returned values."""
        if self._mode != "exact" and k <= 16:
            idx, val, _ = ops.score_topk_tc(self.U, self.V, self.ib, self._factors, k, mask_indptr, mask_indices, stats=False)
        else:
            idx, val = ops.score_topk(self.U, self.V, self.ib, self._factors, k, mask_indptr, mask_indices)
        return idx, val + (self.ub + self.gb).to(val.dtype).unsqueeze(1)

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)


class MF2020(RecMixin, BaseRecommenderModel):
    r"""Matrix Factorization as in "NCF vs. MF Revisited" (https://dl.acm.org/doi/pdf/10.1145/3383313.3412488) on the H100.

    YAML block identical to the reference's (MF.py:41-52): MF2020: {meta: {...}, epochs, factors, lr, reg, m};
    optional keys `b200_mode` (exact | hogwild), `b200_batch` (samples per Hogwild launch), `b200_eval`,
    `b200_device`.
    """

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_factors", "factors", "f", 10, int, None),
            ("_learning_rate", "lr", "lr", 0.05, None, None),
            ("_regularization", "reg", "reg", 0, None, None),
            ("_m", "m", "m", 0, int, None),
        ]
        self.autoset_params()
        self._mode = getattr(self._params, "b200_mode", "exact")
        if self._mode not in ("exact", "hogwild"):
            raise Exception("b200_mode must be 'exact' or 'hogwild'")
        self._hog_batch = int(getattr(self._params, "b200_batch", 1 << 20))   # samples per Hogwild launch
        if self._mode == "hogwild" and not hasattr(self._params, "b200_eval"):
            self._params.b200_eval = "device"
        if not torch.cuda.is_available():
            raise RuntimeError("elliot_b200.MF2020 needs a CUDA device (there is no CPU fallback)")
        self._device = torch.device(getattr(self._params, "b200_device", "cuda:0"))
        self._batch_size = 100000                                     # MF.py:68-69 (progress-bar granularity only)
        # MF.py:65-76: the sampler is built first, the model second; both seed the global streams with the model
        # seed and only the model draws before training, so one numpy stream (init, then negatives) serves both
        self._model = MF2020Model(self._factors, self._data, self._learning_rate, self._regularization, self._seed,
                                  mode=self._mode, device=self._device)
        self._sampler = RendleSampler(self._data.sp_i_train, self._m, self._seed, self._model.np_stream)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
        self._pos_u = torch.from_numpy(self._sampler.pos_u).to(self._device)
        self._pos_i = torch.from_numpy(self._sampler.pos_i).to(self._device)
        self._loss_dev = torch.zeros(1, dtype=torch.float64, device=self._device)
        self._epoch_counter = 0

    @property
    def name(self):
        return "MF2020" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def get_recommendations(self, k: int = 10):
        recs_val, recs_test = self.process_protocol(k)
        return dict(recs_val), dict(recs_test)

    def get_recommendations_tensors(self, k: int = 10):
        return self._model.topk(k, self._indptr, self._sorted_idx)

    def get_single_recommendation(self, mask, k, *args):
        if self._negative_sampling:
            raise NotImplementedError("evaluation-time negative sampling masks are outside this build's hot-path scope")
        idx, val = self.get_recommendations_tensors(k)
        idx, val = idx.cpu().numpy(), val.cpu().numpy().astype(np.float64)
        items = np.array(self._data.items, dtype=object)
        out = {}
        for pu, u in enumerate(self._data.users):
            ok = idx[pu] >= 0
            out[u] = list(zip(items[idx[pu][ok]].tolist(), val[pu][ok].tolist()))
        return out

    def predict(self, u: int, i: int):
        """Score of a (public user, public item) pair (MF.py:96-103 / MF_model.py:60-62)."""
        pu, pi = self._data.public_users[u], self._data.public_items[i]
        m, F = self._model, self._factors
        return float(m.gb.item() + m.ub[pu].item() + m.ib[pi].item() + (m.U[pu, :F].double() @ m.V[pi, :F].double()).item())

    def train(self):
        if self._restore:
            return self.restore_weights()
        for it in self.iterate(self._epochs):
            if self._mode == "exact":
                samples = self._sampler.epoch()
                nb = (len(samples) + self._batch_size - 1) // self._batch_size
                bl = torch.zeros(nb, dtype=torch.float64, device=self._device)
                self._model.train_step(samples, batch_loss=bl)
                sizes = np.minimum(self._batch_size, len(samples) - self._batch_size * np.arange(nb))
                loss = float((bl.cpu().numpy() / sizes).sum())        # MF.py:120-124: sum over batches of mean loss
            else:
                self._loss_dev.zero_()
                m = self._model
                n = len(self._sampler.pos_u) * (1 + self._m)
                for first in range(0, n, self._hog_batch):
                    ops.mf_pointwise_step_f32(m.U, m.V, m.ub, m.ib, m.gb, self._factors, self._pos_u, self._pos_i, self._m,
                                              self._sampler._nitems, self._seed, self._epoch_counter, self._learning_rate,
                                              self._regularization, loss=self._loss_dev, first=first,
                                              count=min(self._hog_batch, n - first))
                self._epoch_counter += 1
                n = len(self._sampler.pos_u) * (1 + self._m)
                nb = (n + self._batch_size - 1) // self._batch_size
                loss = float(self._loss_dev.item()) / max(n, 1) * nb   # mean sample loss x batches, as MF.py:120-124 sums it
            self.evaluate(it, loss / (it + 1))
