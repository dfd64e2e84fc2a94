"""ConvNeuMF, outer-product-based neural collaborative filtering (He et al., IJCAI 2018), on the H100 behind the
reference's model surface.

Mirrors elliot/recommender/neural/ConvNeuMF/convolutional_neural_matrix_factorization.py:59-131 (params `lr,
embedding_size, cnn_channels, cnn_kernels, cnn_strides, dropout_prob, l_w, l_b`, name "ConvNeuMF", batch_size < 1 ->
`transactions`, per-batch losses summed and reported over it + 1) and convolutional_neural_matrix_factorization_model.py:
the outer product u (x) i of each (user, item) pair through Conv2D(2, c_l, stride 2, 'valid', relu) layers, summed over
both spatial axes, then Dropout -> Dense(c_L) -> Dropout -> Dense(1); pairwise BPR loss with the l_w regulariser on the
three embedding rows.  `l_b` is parsed and, as in the reference, used nowhere.

With kernels and strides 2 the network is a quad-tree (csrc/convneumf.cu): level 1 is generated from the user's
S = W1 u terms and the item row, levels >= 2 are tensor-core GEMMs over Z-ordered rows (eb_gemm_bf16_tn / eb_gemm_bf16,
as NeuMF's layers), and scoring runs every (user, item) pair of the catalogue through one fused kernel that keeps every
activation on chip (eb_convneumf_score), then the existing dense top-k and the dense rank pass.  Only the first
m = 2^L floor(f / 2^L) coordinates of an embedding reach the network; the others get only the regulariser's gradient.

Triples are the reference's custom_sampler stream, replayed bit for bit on the device (ops.MtSampler, as CML).  Weights
start GlorotUniform (conv fans k^2 c_in and k^2 c_out) from a seeded torch generator, biases zero; dropout draws its
masks from a Philox stream.  TensorFlow parity of those streams is unpinned; the arithmetic is checked against the fp64
restatements in oracle/convneumf.py.
"""
import ast
import math
import pickle

import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import RankRecs, TopKRecs, cuda_device

SCORER_SMEM_MAX = 227 * 1024


def _list_shortcut(x):
    """The reference's printer of cnn_channels / cnn_kernels / cnn_strides in the model name: "[1, 32, 32]" -> "1-32-32"."""
    s = str(x)
    for c in " []":
        s = s.replace(c, "")
    return s.replace(",", "-")


def check_config(embedding_size, cnn_channels, cnn_kernels, cnn_strides):
    """Refuses what the device path does not take; returns the widths c_1 .. c_L."""
    if len(cnn_kernels) != len(cnn_strides) or len(cnn_channels) - 1 != len(cnn_kernels):
        raise RuntimeError("channels, kernels and strides don't match")               # the reference's check, model.py:27-28
    if any(k != 2 for k in cnn_kernels) or any(s != 2 for s in cnn_strides):
        raise NotImplementedError(f"ConvNeuMF covers kernels and strides of 2 (got kernels {tuple(cnn_kernels)}, strides "
                                  f"{tuple(cnn_strides)}): the device network is the quad-tree they make")
    widths = [int(c) for c in cnn_channels[1:]]
    if any(c != w or w < 8 or w > 64 or w % 8 for c, w in zip(cnn_channels[1:], widths)):
        raise ValueError(f"ConvNeuMF cnn_channels={tuple(cnn_channels)}: every width after the first must be a multiple of 8 "
                         "in [8, 64] (the tensor-core layers take bf16 rows of multiples of 8)")
    L, f = len(widths), int(embedding_size)
    if f != embedding_size or f < (1 << L) or f > 256:
        raise ValueError(f"ConvNeuMF embedding_size={embedding_size} with {L} layers: need 2^{L} <= embedding_size <= 256 (the "
                         "map must hold one final position, and the scorer keeps a user's terms on chip)")
    need = ops.convneumf_score_smem_bytes(f, L, f >> L, widths)
    if need > SCORER_SMEM_MAX:
        raise ValueError(f"ConvNeuMF embedding_size={f}, widths {tuple(widths)}: the fused scorer would need {need} bytes of "
                         f"shared memory per CTA, more than the H100's {SCORER_SMEM_MAX}")
    return widths


class ConvNeuMFModel:
    ACT_BUDGET = 1 << 30           # bytes of activations and their gradients one chunk of a training batch may hold
    SCORE_BUDGET = 256 << 20       # bytes of one dense score block

    def __init__(self, num_users, num_items, embedding_size, learning_rate, widths, dropout_prob, l_w, l_b, random_seed,
                 device):
        self.nu, self.ni, self.f = num_users, num_items, int(embedding_size)
        self.c = [1] + list(widths)
        self.L = len(widths)
        self.HL = self.f >> self.L
        self.R = [None] + [self.HL * self.HL << (2 * (self.L - l)) for l in range(1, self.L + 1)]     # rows per pair
        self.lr, self.p_drop, self.l_w, self.l_b, self.seed = learning_rate, float(dropout_prob), l_w, l_b, int(random_seed)
        self.device = torch.device(device)
        self.ld = (self.f + 3) // 4 * 4
        g = torch.Generator(device=self.device); g.manual_seed(self.seed)

        def glorot(shape, fan_in, fan_out):
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            return (torch.rand(shape, device=self.device, generator=g) * 2 - 1) * lim

        def table(n):                                      # Embedding(GlorotUniform): fans (n, f)
            t = torch.zeros((n, self.ld), device=self.device)
            t[:, :self.f] = glorot((n, self.f), n, self.f)
            return t
        c, L = self.c, self.L
        self.P = {"U": table(num_users), "I": table(num_items),
                  "W1": glorot((4 * c[1],), 4 * c[0], 4 * c[1]), "b1": torch.zeros(c[1], device=self.device)}
        for l in range(2, L + 1):                          # kept [c_l][4 c_(l-1)]: the transposed Keras [2, 2, c_in, c_out]
            self.P[f"W{l}"] = glorot((4 * c[l - 1], c[l]), 4 * c[l - 1], 4 * c[l]).t().contiguous()
            self.P[f"b{l}"] = torch.zeros(c[l], device=self.device)
        self.P.update({"Wd1": glorot((c[L], c[L]), c[L], c[L]).reshape(-1).contiguous(), "bd1": torch.zeros(c[L], device=self.device),
                       "wd2": glorot((c[L],), c[L], 1), "bd2": torch.zeros(4, device=self.device)})
        z = lambda: {k: torch.zeros_like(v) for k, v in self.P.items()}
        self.G, self.M, self.V = z(), z(), z()
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        self._refresh()

    def _refresh(self):
        self.Wb = {l: ops.to_bf16(self.P[f"W{l}"]) for l in range(2, self.L + 1)}
        self._packed = None

    def _triple_bytes(self):
        """Activation bytes of one triple (two pairs): bf16 and fp32 copies of every level and of its gradient."""
        return 2 * sum(self.R[l] * self.c[l] for l in range(1, self.L + 1)) * 16

    def _add(self, key, fresh, out):
        """G[key] += out when fresh is False (a later chunk of the batch), else the result already went to G[key]."""
        if not fresh:
            ops.table_apply_delta_f32(self.G[key], self.G[key], out)

    def grads(self, tu, ti, tj, chunk=None, y_out=None, mask_out=None):
        """Adds the batch's loss to self._loss and its gradients to self.G, in chunks of at most `chunk` triples (default:
        what ACT_BUDGET holds).  The loss is a sum over triples, so the chunks add up to the batch's gradient."""
        n, P, G, c, L, R = tu.numel(), self.P, self.G, self.c, self.L, self.R
        chunk = int(chunk or max(1, self.ACT_BUDGET // self._triple_bytes()))
        seed = self.seed * 1000003 + self.step
        dt = torch.float32 if L == 1 else self.Wb[2].dtype              # bf16, or fp32 in the exact_gemm checking mode
        for s in range(0, n, chunk):
            e = min(n, s + chunk)
            nc, fresh = e - s, s == 0
            cu, ci, cj = tu[s:e], ti[s:e], tj[s:e]
            pu, pi = torch.cat([cu, cu]), torch.cat([ci, cj])
            x = torch.empty((2 * nc * R[1], c[1]), dtype=dt, device=self.device)
            ops.convneumf_l1_fwd(P["U"], P["I"], self.f, pu, pi, L, self.HL, P["W1"], P["b1"], c[1], x)
            ins, outs = {}, {}
            for l in range(2, L + 1):
                rows = 2 * nc * R[l]
                ins[l] = x.view(rows, 4 * c[l - 1])
                if l < L:
                    outs[l], x = ops.gemm_bf16_tn(ins[l], self.Wb[l], rows, c[l], 4 * c[l - 1], bias=P[f"b{l}"], act=2,
                                                  out_bf16=True)
                else:
                    outs[l] = x = ops.gemm_bf16_tn(ins[l], self.Wb[l], rows, c[l], 4 * c[l - 1], bias=P[f"b{l}"], act=2)
            dpre = torch.empty_like(x)
            ops.convneumf_head(x, R[L], c[L], P["Wd1"], P["bd1"], P["wd2"], P["bd2"], P["U"], P["I"], self.f, cu, ci, cj, s, n,
                               self.p_drop, seed, self.l_w, self._loss, G["Wd1"], G["bd1"], G["wd2"], G["bd2"], dpre,
                               y_out=y_out, mask_out=mask_out)
            for l in range(L, 1, -1):
                rows = 2 * nc * R[l]
                dpre_b = ops.to_bf16(dpre) if l == L else dpre_b
                wk, bk = f"W{l}", f"b{l}"
                out = G[wk] if fresh else torch.empty_like(G[wk])
                ops.gemm_bf16(dpre_b, ins[l], c[l], 4 * c[l - 1], rows, a_rows_are_k=True, b_rows_are_k=True, out=out)
                self._add(wk, fresh, out)
                out = G[bk] if fresh else torch.empty_like(G[bk])
                ops.colsum(dpre, out)
                self._add(bk, fresh, out)
                dx = ops.gemm_bf16(dpre_b, self.Wb[l], rows, 4 * c[l - 1], c[l], b_rows_are_k=True)
                if l > 2:
                    dpre, dpre_b = ops.relu_bwd(dx.view(-1, c[l - 1]), outs[l - 1], copy_bf16=True)
                else:
                    dpre = dx
            ops.convneumf_l1_bwd(P["U"], P["I"], self.f, pu, pi, nc, L, self.HL, P["W1"], P["b1"], c[1], dpre.view(-1, c[1]),
                                 self.l_w, G["U"], G["I"], G["W1"], G["b1"])

    def adam(self):
        """One Keras Adam step on every trainable weight; clears self.G."""
        self.step += 1
        for k in self.P:
            ops.adam_dense_f32(self.P[k], self.M[k], self.V[k], self.G[k], self.lr, self.step)
        self._refresh()

    def train_step(self, batch, chunk=None):
        """batch = (user, pos, neg) int32 device tensors; adds the batch loss to self._loss and returns it (fp64 tensor)."""
        self.grads(*batch, chunk=chunk)
        self.adam()
        return self._loss

    def _score_operands(self):
        if self._packed is None:
            with ops.exact_gemm(False):                    # the scorer always reads bf16 layers
                if self.L > 1:
                    flat = torch.cat([self.P[f"W{l}"].reshape(-1) for l in range(2, self.L + 1)]).view(1, -1)
                    Wp = ops.to_bf16(flat).view(-1)
                    bp = torch.cat([self.P[f"b{l}"] for l in range(2, self.L + 1)])
                else:
                    Wp = bp = None
            self._packed = (Wp, bp)
        return self._packed

    def scores(self, u0, u1, out=None):
        """Dense [u1 - u0][n_items] fp32 scores of users u0 .. u1 - 1 (get_recs with dropout off)."""
        Wp, bp = self._score_operands()
        P = self.P
        return ops.convneumf_score(P["U"], P["I"], self.f, self.L, self.HL, self.c[1:], P["W1"], P["b1"], Wp, bp, P["Wd1"],
                                   P["bd1"], P["wd2"], P["bd2"], u0, u1 - u0, self.ni, out=out)

    def _blocks(self):
        b = max(1, min(self.nu, self.SCORE_BUDGET // (4 * self.ni), 65535))
        return [(u0, min(u0 + b, self.nu)) for u0 in range(0, self.nu, b)]

    def topk(self, k, mask_indptr, mask_indices):
        """masked top-k of every user's scores (get_recs + get_top_k, model.py:158-187)."""
        idx, val = [], []
        for u0, u1 in self._blocks():
            rows = torch.arange(u0, u1, dtype=torch.int32, device=self.device)
            i, v = ops.dense_topk(self.scores(u0, u1), k, mask_indptr, mask_indices, rows)
            idx.append(i); val.append(v)
        return torch.cat(idx), torch.cat(val)

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """The lists topk() selects from, ranked for AUC / GAUC."""
        outs = [ops.dense_rank(self.scores(u0, u1), rel_indptr, rel_items, mask_indptr, mask_indices, row_begin=u0)
                for u0, u1 in self._blocks()]
        return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])

    def get_model_state(self):
        host = lambda d: {k: v.cpu().numpy() for k, v in d.items()}
        return {"P": host(self.P), "M": host(self.M), "V": host(self.V), "step": self.step}

    def set_model_state(self, s):
        for dst, key in ((self.P, "P"), (self.M, "M"), (self.V, "V")):
            for k, t in dst.items():
                t.copy_(torch.from_numpy(s[key][k]))
        self.step = s["step"]
        self._refresh()

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))


class ConvNeuMF(TopKRecs, RankRecs, RecMixin, BaseRecommenderModel):
    r"""Outer Product-based Neural Collaborative Filtering (https://arxiv.org/abs/1808.03912).  YAML keys as in the
    reference (convolutional_neural_matrix_factorization.py:65-77): `epochs, batch_size, embedding_size, lr, l_w, l_b,
    cnn_channels, cnn_kernels, cnn_strides, dropout_prob`; optional keys `b200_eval` and `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        as_list = lambda x: list(ast.literal_eval(str(x)))
        self._params_list = [
            ("_lr", "lr", "lr", 0.001, None, None),
            ("_embedding_size", "embedding_size", "embedding_size", 100, None, None),
            ("_cnn_channels", "cnn_channels", "cnn_channels", "(1, 32, 32)", as_list, _list_shortcut),
            ("_cnn_kernels", "cnn_kernels", "cnn_kernels", "(2,2)", as_list, _list_shortcut),
            ("_cnn_strides", "cnn_strides", "cnn_strides", "(2,2)", as_list, _list_shortcut),
            ("_dropout_prob", "dropout_prob", "dropout_prob", 0, None, None),
            ("_l_w", "l_w", "l_w", 0.005, None, None),
            ("_l_b", "l_b", "l_b", 0.0005, None, None),
        ]
        self.autoset_params()
        if self._negative_sampling:
            raise NotImplementedError("ConvNeuMF: evaluation-time negative sampling masks are outside this build's hot-path "
                                      "scope")
        widths = check_config(self._embedding_size, self._cnn_channels, self._cnn_kernels, self._cnn_strides)
        if not 0 <= float(self._dropout_prob) < 1:
            raise ValueError(f"ConvNeuMF dropout_prob={self._dropout_prob}: need 0 <= dropout_prob < 1")
        if self._batch_size < 1:
            self._batch_size = self._data.transactions                 # :79-80
        self._device = cuda_device(self._params, "ConvNeuMF")
        self._indptr, self._set_idx, self._sorted_idx = train_csr_of(self._data, self._device)
        self._sampler = ops.MtSampler(self._num_users, self._num_items, self._indptr, self._set_idx, self._sorted_idx, seed=42)
        self._model = ConvNeuMFModel(self._num_users, self._num_items, self._embedding_size, self._lr, widths,
                                     self._dropout_prob, self._l_w, self._l_b, self._seed, self._device)

    @property
    def name(self):
        return "ConvNeuMF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        T = self._data.transactions
        for it in self.iterate(self._epochs):
            self._model._loss.zero_()
            tu, ti, tj = self._sampler.step(T)                           # the triples of the reference's Sampler.step
            for s in range(0, T, self._batch_size):
                e = min(s + self._batch_size, T)
                self._model.train_step((tu[s:e], ti[s:e], tj[s:e]))
            self.evaluate(it, float(self._model._loss.item()) / (it + 1))

    def get_recommendations(self, k: int = 100):
        return super().get_recommendations(k)
