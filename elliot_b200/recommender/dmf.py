"""DMF, deep matrix factorization (Xue et al., IJCAI 2017), on the H100 behind the reference's model surface.

Mirrors elliot/recommender/neural/DMF/deep_matrix_factorization.py:56-121 (params `lr, user_mlp, item_mlp, neg_ratio, reg,
similarity`, name "DMF", batch_size < 1 -> every sample of the epoch, transactions * (1 + neg_ratio) samples per epoch,
per-batch mean losses summed) and deep_matrix_factorization_model.py:18-132.

- Towers: the user tower reads the user's train rating ROW (n_items wide), the item tower the item's rating COLUMN
  (n_users wide), rating values, not 0/1 (the reference's frozen Embedding layers over sp_i_train_ratings).  Dense ReLU
  layers, then a linear last layer; kernels RandomNormal(0, 0.01) from a seeded torch generator, biases zero.  The first
  layer is a sparse product over the train CSR / CSC (csrc/dmf.cu), the others run on the tensor cores (eb_gemm_bf16_tn /
  eb_gemm_bf16, bf16 operands, fp32 accumulation) as NeuMF's do.  Every MLP weight is moved by dense Keras Adam.
- Head: `cosine` is tf.nn.l2_normalize(x, 0): each factor COLUMN is normalised over the batch, so every sample's output
  depends on the whole batch, and a user or item repeated in the batch counts once per occurrence.  `dot` skips it.
  Label r / max_ratings, Keras BinaryCrossentropy with its clip (csrc/dmf.cu, eb_dmf_head_f32).
- `reg` is parsed and, as in the reference, used nowhere.
- Recommendations score users in blocks [offset, offset + batch_size) as get_recommendations does, and with `cosine` a
  user's list depends on its block: the block's column norms scale its users, and every item factor becomes
  V / sqrt(block * V^2) (get_recs feeds B identical copies of each item).  eb_dmf_score_operands_f32 writes those
  operands and the existing scorers rank them; the towers run once per model state, not once per block.
- Samples are the reference's pointwise ratio sampler's stream, replayed bit for bit on the device
  (ops.MtPointwiseRatioSampler).

TensorFlow parity of the initial weights and of Adam is unpinned; the arithmetic is checked against the fp64
restatements in oracle/dmf.py.
"""
import ast
import pickle

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import RankRecs, TopKRecs, check_free, cuda_device


def _mlp_shortcut(x):
    """The reference's printer of user_mlp / item_mlp in the model name: "[64, 32]" -> "64-32"."""
    s = str(x)
    for c in " []":
        s = s.replace(c, "")
    return s.replace(",", "-")


def check_widths(user_mlp, item_mlp):
    for name, w in (("user_mlp", user_mlp), ("item_mlp", item_mlp)):
        if not w or any(int(x) != x or x < 8 or x > 256 or x % 8 for x in w):
            raise ValueError(f"DMF {name}={tuple(w)}: every width must be a multiple of 8 in [8, 256] (the tensor-core "
                             "GEMMs take bf16 rows of multiples of 8; the head takes at most 256 factors)")
    if user_mlp[-1] != item_mlp[-1]:
        raise ValueError(f"DMF needs the two towers to end at the same width (user_mlp {tuple(user_mlp)}, item_mlp "
                         f"{tuple(item_mlp)}): the head multiplies their outputs factor by factor")


class _Tower:
    """One MLP tower over the rows of a rating CSR (indptr, indices, values): W[0] is [n_in][w0] (gathered by row), W[l]
    for l >= 1 is [w_l][w_(l-1)] as the tensor-core GEMMs read it."""

    def __init__(self, n_in, widths, csr, gen, device):
        self.widths, self.csr, self.device = list(widths), csr, device
        dims = [n_in] + self.widths
        normal = lambda shape: torch.randn(shape, device=device, generator=gen) * 0.01      # RandomNormal(stddev=0.01)
        self.W = [normal((n_in, dims[1]))] + [normal((dims[l + 1], dims[l])) for l in range(1, len(self.widths))]
        self.b = [torch.zeros((w + 3) // 4 * 4, device=device) for w in self.widths]
        self.refresh()

    def params(self):
        return self.W + self.b

    def refresh(self):
        self.Wb = [None] + [ops.to_bf16(W) for W in self.W[1:]]

    def forward(self, rows):
        """Output [B][w_last] fp32 for int32 row ids; keeps what backward needs."""
        n, B = len(self.widths), rows.numel()
        h = torch.empty((B, self.widths[0]), device=self.device)
        ops.dmf_sparse_fwd(self.W[0], self.b[0], *self.csr, rows, h, relu=n > 1)
        self._rows, self._acts, self._acts_b = rows, [h], []
        for l in range(1, n):
            hb = ops.to_bf16(h)
            h = ops.gemm_bf16_tn(hb, self.Wb[l], B, self.widths[l], self.widths[l - 1], bias=self.b[l], act=2 if l < n - 1 else 0)
            self._acts.append(h); self._acts_b.append(hb)
        return h

    def backward(self, d, G):
        """Gradients of the last forward into G (lists like W and b) from d = dloss/doutput [B][w_last]."""
        B = d.shape[0]
        for l in range(len(self.widths) - 1, 0, -1):
            db = ops.to_bf16(d)
            ops.gemm_bf16(db, self._acts_b[l - 1], self.widths[l], self.widths[l - 1], B, a_rows_are_k=True, b_rows_are_k=True,
                          out=G["W"][l])
            ops.colsum(d, G["b"][l])
            d = ops.relu_bwd(ops.gemm_bf16(db, self.Wb[l], B, self.widths[l - 1], self.widths[l], b_rows_are_k=True),
                             self._acts[l - 1])
        ops.dmf_sparse_bwd(G["W"][0], *self.csr, self._rows, d)
        ops.colsum(d, G["b"][0])


class DMFModel:
    def __init__(self, num_users, num_items, user_mlp, item_mlp, similarity, max_ratings, learning_rate, random_seed, device,
                 user_csr, item_csr, block):
        check_widths(user_mlp, item_mlp)
        if similarity not in ("cosine", "dot"):
            raise NotImplementedError(f"DMF similarity must be 'cosine' or 'dot' (got {similarity!r})")
        self.nu, self.ni, self.F = num_users, num_items, int(user_mlp[-1])
        self.cosine, self.max_ratings, self.lr, self.block = similarity == "cosine", float(max_ratings), learning_rate, block
        self.device = torch.device(device)
        g = torch.Generator(device=self.device); g.manual_seed(int(random_seed))
        self.user = _Tower(num_items, user_mlp, user_csr, g, self.device)
        self.item = _Tower(num_users, item_mlp, item_csr, g, self.device)
        self.P = self.user.params() + self.item.params()
        z = lambda: [torch.zeros_like(t) for t in self.P]
        self.G, self.M, self.V = z(), z(), z()
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        self._ops_step = None

    def _grads_of(self, tower):
        nw, off = len(tower.W), 0 if tower is self.user else len(self.user.params())
        return {"W": self.G[off:off + nw], "b": self.G[off + nw:off + 2 * nw]}

    def grads(self, batch):
        """Adds the batch's mean loss to self._loss and writes its gradients into self.G."""
        u, it, r = batch
        Uo, Vo = self.user.forward(u), self.item.forward(it)
        dU, dV = torch.empty_like(Uo), torch.empty_like(Vo)
        ops.dmf_head_f32(Uo, Vo, self.F, r, self.max_ratings, self.cosine, self._loss, dU, dV)
        self.user.backward(dU, self._grads_of(self.user))
        self.item.backward(dV, self._grads_of(self.item))

    def adam(self):
        """One Keras Adam step on every MLP weight; clears self.G."""
        self.step += 1
        for p, m, v, gr in zip(self.P, self.M, self.V, self.G):
            ops.adam_dense_f32(p, m, v, gr, self.lr, self.step)
        self.user.refresh(); self.item.refresh()

    def train_step(self, batch):
        """batch = (user int32, item int32, rating float32) device tensors; adds the batch loss to the running sum and returns
        it (fp64 device tensor)."""
        self.grads(batch)
        self.adam()
        return self._loss

    def tower_outputs(self):
        """(every user's, every item's) tower output, computed once per model state."""
        if self._ops_step != self.step:
            self._outs = (self.user.forward(torch.arange(self.nu, dtype=torch.int32, device=self.device)),
                          self.item.forward(torch.arange(self.ni, dtype=torch.int32, device=self.device)))
            self._ops_step = self.step
        return self._outs

    def _blocks(self):
        """[(user_begin, n_sel, item operand)] over the reference's user blocks: the full blocks share one operand, the
        short last block has its own."""
        Uh, Vh, Vl = ops.dmf_score_operands_f32(*self.tower_outputs(), self.F, self.block, self.cosine)
        bl = min(self.block, self.nu)
        n_full = self.nu // bl * bl
        parts = [(0, n_full, Vh)] if n_full else []
        if n_full < self.nu:
            parts.append((n_full, self.nu - n_full, Vl if Vl is not None else Vh))
        return Uh, parts

    def topk(self, k, mask_indptr, mask_indices, tensor_cores=True):
        """masked top-k of the block-normalised scores of every user (get_recs + get_top_k, model.py:106-132)."""
        Uh, parts = self._blocks()
        idx, val = [], []
        for u0, n, V in parts:
            if tensor_cores and k <= 16:
                i, v, _ = ops.score_topk_tc(Uh, V, None, self.F, k, mask_indptr, mask_indices, user_begin=u0, n_sel=n, stats=False)
            else:
                i, v = ops.score_topk(Uh, V, None, self.F, k, mask_indptr, mask_indices, user_begin=u0, n_sel=n)
            idx.append(i); val.append(v)
        return torch.cat(idx), torch.cat(val)

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """The lists topk() selects from, ranked for AUC / GAUC."""
        Uh, parts = self._blocks()
        outs = [ops.score_rank(Uh, V, None, self.F, rel_indptr, rel_items, mask_indptr, mask_indices, user_begin=u0, n_sel=n)
                for u0, n, V in parts]
        return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])

    def get_model_state(self):
        host = lambda ts: [t.cpu().numpy() for t in ts]
        return {"P": host(self.P), "M": host(self.M), "V": host(self.V), "step": self.step}

    def set_model_state(self, s):
        for dst, key in ((self.P, "P"), (self.M, "M"), (self.V, "V")):
            for t, a in zip(dst, s[key]):
                t.copy_(torch.from_numpy(a))
        self.step = s["step"]
        self.user.refresh(); self.item.refresh()
        self._ops_step = None

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))


def rating_csrs(data, device):
    """((indptr, item, rating) of the train rating rows, (indptr, user, rating) of its columns), sorted, on `device`."""
    import scipy.sparse as sp
    R = sp.csr_matrix(data.sp_i_train_ratings, dtype=np.float32)
    R.sort_indices()
    C = R.T.tocsr()
    C.sort_indices()
    up = lambda M: (torch.from_numpy(M.indptr.astype(np.int64)).to(device), torch.from_numpy(M.indices.astype(np.int32)).to(device),
                    torch.from_numpy(M.data.astype(np.float32)).to(device))
    return up(R), up(C)


def set_order_ratings(indptr, set_idx, sorted_idx, sorted_vals, n_items):
    """The rating of every set-order entry: its row's sorted entry of the same item."""
    rows = torch.repeat_interleave(torch.arange(indptr.numel() - 1, device=indptr.device), indptr[1:] - indptr[:-1])
    keys = rows * n_items + sorted_idx.long()
    pos = torch.searchsorted(keys, rows * n_items + set_idx.long())
    return sorted_vals[pos].contiguous()


class DMF(TopKRecs, RankRecs, RecMixin, BaseRecommenderModel):
    r"""Deep Matrix Factorization (https://www.ijcai.org/Proceedings/2017/0447.pdf).  YAML keys as in the reference
    (deep_matrix_factorization.py:56-63): `epochs, batch_size, lr, user_mlp, item_mlp, neg_ratio, reg, similarity`;
    optional key `b200_device`.  `reg` has no effect, as in the reference."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_learning_rate", "lr", "lr", 0.0001, None, None),
            ("_user_mlp", "user_mlp", "umlp", "(64,32)", lambda x: list(ast.literal_eval(str(x))), _mlp_shortcut),
            ("_item_mlp", "item_mlp", "imlp", "(64,32)", lambda x: list(ast.literal_eval(str(x))), _mlp_shortcut),
            ("_neg_ratio", "neg_ratio", "negratio", 5, None, None),
            ("_reg", "reg", "reg", 0.001, None, None),
            ("_similarity", "similarity", "sim", "cosine", None, None),
        ]
        self.autoset_params()
        if self._similarity not in ("cosine", "dot"):
            raise NotImplementedError(f"DMF similarity must be 'cosine' or 'dot' (got {self._similarity!r})")
        check_widths(self._user_mlp, self._item_mlp)
        T = self._data.transactions
        self._transactions_per_epoch = T + self._neg_ratio * T                        # :66-72
        if self._batch_size < 1:
            self._batch_size = self._transactions_per_epoch
        self._device = cuda_device(self._params, "DMF")
        self._indptr, self._set_idx, self._sorted_idx = train_csr_of(self._data, self._device)
        lui = (self._indptr[1:] - self._indptr[:-1]).max().item()
        if lui >= self._num_items:
            raise ValueError("DMF: a user has rated every item, so the reference's sampler never finds it a negative "
                             "(its negative draw loops forever)")
        user_csr, item_csr = rating_csrs(self._data, self._device)
        self._max_ratings = float(user_csr[2].max().item())
        B = min(self._batch_size, self._transactions_per_epoch)
        per_sample = 16 * (sum(self._user_mlp) + sum(self._item_mlp)) + 64
        check_free("DMF", self._device, B * per_sample + self._transactions_per_epoch * 12,
                   f"one batch of {B} samples through both towers and the epoch's samples")
        self._sampler = ops.MtPointwiseRatioSampler(
            self._num_users, self._num_items, self._indptr, self._set_idx,
            set_order_ratings(self._indptr, self._set_idx, user_csr[1], user_csr[2], self._num_items), self._sorted_idx,
            self._neg_ratio, seed=42)
        self._model = DMFModel(self._num_users, self._num_items, self._user_mlp, self._item_mlp, self._similarity,
                               self._max_ratings, self._learning_rate, self._seed, self._device, user_csr, item_csr,
                               self._batch_size)

    @property
    def name(self):
        return "DMF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        E, B = self._transactions_per_epoch, self._batch_size
        for it in self.iterate(self._epochs):
            self._model._loss.zero_()
            self._sampler.epoch()                                      # each Sampler.step() call rebuilds the list
            u, i, r = self._sampler.step(E)
            for s in range(0, E, B):
                e = min(s + B, E)
                self._model.train_step((u[s:e], i[s:e], r[s:e]))
            self.evaluate(it, float(self._model._loss.item()) / (it + 1))

    def get_recommendations(self, k: int = 100):
        return super().get_recommendations(k)
