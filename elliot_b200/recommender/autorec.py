"""UserAutoRec and ItemAutoRec (Sedhain et al., WWW 2015) on the H100 behind the reference's model surface.

Mirrors elliot/recommender/neural/UserAutoRec/userautorec.py:59-98 and userautorec_model.py:19-123, and
neural/ItemAutoRec/itemautorec.py:58-108 and itemautorec_model.py:18-131 (params `lr, hidden_neuron, l_w`; batch_size < 1
-> `transactions`; rows in the order of sparse_sampler.py's `random.sample`, seeded with 42 at construction; the epoch's
summed batch losses reported as sum / (epoch + 1)).

- Network: Dense(H, sigmoid) then Dense(n_out) (UserAutoRec: linear; ItemAutoRec: sigmoid), GlorotNormal kernels
  (truncated at 2 sigma, from a seeded torch generator) and Ones biases.  UserAutoRec reads rows of the binary train
  matrix (users, n_in = n_out = items), ItemAutoRec rows of its transpose (items, n_in = n_out = users).
- Loss: mean over the batch rows (empty rows included) of sum_cols (x - act(o) sign(x))^2.  Only a row's train entries
  carry a gradient, so the decoder runs over those entries only (eb_autorec_decoder_f32): the dense rows x catalogue
  input and reconstruction of the reference are never formed.  The encoder is the sparse product of eb_dmf_sparse_fwd_f32
  and eb_sigmoid_inplace; dW1 is eb_dmf_sparse_bwd_f32, db1 eb_colsum; Keras Adam moves all four variables.
- `l_w` is parsed and, as in the reference, never applied: its Keras regularisation losses are not added to the
  train_step loss.
- UserAutoRec's score h_u . W2[:, i] + b2[i] factorises, so the encoder runs once per model state over every user and
  the existing scorers rank h . W2^T + b2 under the train mask.
- ItemAutoRec's get_recommendations draws `perm = random.sample(range(I), I)` from the training stream (so evaluating
  shifts the next epoch's order), reconstructs every item's column in perm order and treats column j as item j: user u's
  score of item j is sigmoid(W2[u] . g_perm[j] + b2[u]) with g_i the encoder output of item i.  That is mirrored, not
  fixed.  The rank pass ranks the lists the next get_recommendations will return: it takes the permutation that call
  will draw and leaves the stream as it was.

TensorFlow parity of the initial weights and of Adam is unpinned; the arithmetic is checked against the fp64
restatements in oracle/autorec.py.
"""
import math
import pickle
import random

import numpy as np
import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import RankRecs, TopKRecs, cuda_device

LINEAR, SIGMOID = 0, 1


def check_hidden(hidden_neuron):
    if int(hidden_neuron) != hidden_neuron or not 4 <= hidden_neuron <= 1024 or hidden_neuron % 4:
        raise ValueError(f"AutoRec hidden_neuron={hidden_neuron}: must be a multiple of 4 in [4, 1024] (the sparse encoder "
                         "and the decoder kernel take rows of float4 chunks, up to 1024 wide)")


class AutoRecModel:
    """The autoencoder over the rows of a binary CSR (indptr, indices, values).  W1 is Keras's [n_in][H] kernel (gathered
    by row), W2 Keras's [H][n_out] kernel stored [n_out][H] so that each output's weights are one contiguous row; b2 is
    padded to a multiple of 4 (the padding stays 0)."""

    def __init__(self, n_in, n_out, hidden_neuron, learning_rate, act, random_seed, device, csr):
        check_hidden(hidden_neuron)
        self.n_in, self.n_out, self.H, self.lr, self.act = n_in, n_out, int(hidden_neuron), learning_rate, act
        self.csr, self.device = csr, torch.device(device)
        g = torch.Generator(device=self.device); g.manual_seed(int(random_seed))

        def glorot(rows, cols, fan_in, fan_out):       # GlorotNormal (truncated at 2 sigma)
            std = math.sqrt(2.0 / (fan_in + fan_out)) / 0.87962566103423978
            t = torch.empty((rows, cols), device=self.device)
            torch.nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=g)
            return t
        H = self.H
        b2 = torch.zeros((n_out + 3) // 4 * 4, device=self.device)
        b2[:n_out] = 1.0
        self.P = [glorot(n_in, H, n_in, H), torch.ones(H, device=self.device), glorot(n_out, H, H, n_out), b2]
        z = lambda: [torch.zeros_like(t) for t in self.P]
        self.G, self.M, self.V = z(), z(), z()
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        self._h_step = None

    def encode(self, rows):
        """sigmoid(X[rows] W1 + b1) [B][H] for int32 row ids of the CSR."""
        h = torch.empty((rows.numel(), self.H), device=self.device)
        ops.dmf_sparse_fwd(self.P[0], self.P[1], *self.csr, rows, h, relu=False)
        return ops.sigmoid_(h)

    def grads(self, rows):
        """Adds the batch's loss to self._loss and its gradients to self.G; returns (h, dpre1)."""
        h = self.encode(rows)
        dpre1 = torch.empty_like(h)
        ops.autorec_decoder_f32(*self.csr, rows, h, self.P[2], self.P[3], self.act, self._loss, self.G[2], self.G[3], dpre1)
        ops.dmf_sparse_bwd(self.G[0], *self.csr, rows, dpre1)
        ops.colsum(dpre1, self.G[1])
        return h, dpre1

    def adam(self):
        """One Keras Adam step on W1, b1, W2, b2; clears self.G."""
        self.step += 1
        for p, m, v, gr in zip(self.P, self.M, self.V, self.G):
            ops.adam_dense_f32(p, m, v, gr, self.lr, self.step)

    def train_step(self, rows):
        """rows: int32 device tensor of CSR row ids.  Returns the batch loss (fp64 device tensor [1])."""
        self._loss.zero_()
        if rows.numel():
            self.grads(rows)
        self.adam()
        return self._loss

    def hidden(self):
        """The encoder output of every row, computed once per model state."""
        if self._h_step != self.step:
            self._h = self.encode(torch.arange(self.n_rows(), dtype=torch.int32, device=self.device))
            self._h_step = self.step
        return self._h

    def n_rows(self):
        return self.csr[0].numel() - 1

    def _scorer(self, U, V, bias, k, mask_indptr, mask_indices):
        if self.H <= 256 and k <= 16:
            return ops.score_topk_tc(U, V, bias, self.H, k, mask_indptr, mask_indices, stats=False)[:2]
        return ops.score_topk(U, V, bias, self.H, k, mask_indptr, mask_indices)

    # ---- UserAutoRec: rows are users, outputs items
    def topk(self, k, mask_indptr, mask_indices):
        """masked top-k of h . W2^T + b2 for every user (RecMixin.get_recommendations + get_top_k)."""
        return self._scorer(self.hidden(), self.P[2], self.P[3], k, mask_indptr, mask_indices)

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """The lists topk() selects from, ranked for AUC / GAUC."""
        return ops.score_rank(self.hidden(), self.P[2], self.P[3], self.H, rel_indptr, rel_items, mask_indptr, mask_indices)

    # ---- ItemAutoRec: rows are items, outputs users
    def item_operand(self, perm):
        """V[j] = g_perm[j], the encoder output of item perm[j]."""
        return self.encode(torch.as_tensor(np.asarray(perm, np.int32), device=self.device))

    def item_topk(self, perm, k, mask_indptr, mask_indices):
        """masked top-k of sigmoid(W2[u] . g_perm[j] + b2[u]) (itemautorec.py:99-108): selected on the logit, the bias and
        the sigmoid applied to the kept values."""
        idx, val = self._scorer(self.P[2], self.item_operand(perm), None, k, mask_indptr, mask_indices)
        return idx, ops.sigmoid_(ops.add_row_offset_(val.contiguous(), self.P[3]))

    def item_rank(self, perm, rel_indptr, rel_items, mask_indptr, mask_indices):
        return ops.score_rank(self.P[2], self.item_operand(perm), None, self.H, rel_indptr, rel_items, mask_indptr,
                              mask_indices)

    def get_model_state(self):
        host = lambda ts: [t.cpu().numpy() for t in ts]
        return {"P": host(self.P), "M": host(self.M), "V": host(self.V), "step": self.step}

    def set_model_state(self, s):
        for dst, key in ((self.P, "P"), (self.M, "M"), (self.V, "V")):
            for t, a in zip(dst, s[key]):
                t.copy_(torch.from_numpy(a))
        self.step = s["step"]
        self._h_step = None

    def save_weights(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.get_model_state(), f)

    def load_weights(self, path):
        with open(path, "rb") as f:
            self.set_model_state(pickle.load(f))


def binary_csr(m, device):
    """(indptr int64, indices int32 sorted per row, values float32) of a scipy matrix's rows on `device`."""
    import scipy.sparse as sp
    m = sp.csr_matrix(m, dtype=np.float32)
    m.sort_indices()
    return (torch.from_numpy(m.indptr.astype(np.int64)).to(device), torch.from_numpy(m.indices.astype(np.int32)).to(device),
            torch.from_numpy(m.data.astype(np.float32)).to(device))


def epoch_order(n_rows):
    """One epoch's row order: `random.sample(range(n), n)` on the global stream (sparse_sampler.py:17-18)."""
    return random.sample(range(n_rows), n_rows)


class _AutoRec(TopKRecs, RankRecs, RecMixin, BaseRecommenderModel):
    _ACT = LINEAR

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._params_list = [
            ("_lr", "lr", "lr", 0.0001, None, None),
            ("_hidden_neuron", "hidden_neuron", "hidden_neuron", 500, None, None),
            ("_l_w", "l_w", "l_w", 0.001, None, None),
        ]
        self.autoset_params()
        check_hidden(self._hidden_neuron)
        if self._negative_sampling:
            raise NotImplementedError(f"{type(self).__name__}: evaluation-time negative sampling masks are outside this "
                                      "build's hot-path scope")
        if self._batch_size < 1:
            self._batch_size = self._data.transactions
        self._device = cuda_device(self._params, type(self).__name__)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
        train = self._data.sp_i_train
        csr = binary_csr(train.T if self._ACT == SIGMOID else train, self._device)
        n = train.shape[0] if self._ACT == SIGMOID else train.shape[1]           # the outputs: users (Item), items (User)
        random.seed(42)                                                         # sparse_sampler.py:16
        self._model = AutoRecModel(n, n, self._hidden_neuron, self._lr, self._ACT, self._seed, self._device, csr)

    @property
    def name(self):
        return type(self).__name__ + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def train(self):
        if self._restore:
            return self.restore_weights()
        n = self._model.n_rows()
        for it in self.iterate(self._epochs):
            loss = torch.zeros(1, dtype=torch.float64, device=self._device)
            order = torch.tensor(epoch_order(n), dtype=torch.int32, device=self._device)
            for s in range(0, n, self._batch_size):
                loss += self._model.train_step(order[s:s + self._batch_size].contiguous())
            self.evaluate(it, float(loss.item()) / (it + 1))


class UserAutoRec(_AutoRec):
    r"""AutoRec, user-based (https://users.cecs.anu.edu.au/~akmenon/papers/autorec/autorec-paper.pdf).  YAML keys as in
    the reference (userautorec.py:59-63): `epochs, batch_size, lr, hidden_neuron, l_w`; optional key `b200_device`.
    `l_w` has no effect, as in the reference."""
    _ACT = LINEAR


class ItemAutoRec(_AutoRec):
    r"""AutoRec, item-based (https://users.cecs.anu.edu.au/~akmenon/papers/autorec/autorec-paper.pdf).  YAML keys as in
    the reference (itemautorec.py:58-62): `epochs, batch_size, lr, hidden_neuron, l_w`; optional key `b200_device`.
    `l_w` has no effect, as in the reference.

    As in the reference, every evaluation draws a permutation of the items from the training row stream and scores
    user u's item j with item perm[j]'s reconstruction: sigmoid(W2[u] . g_perm[j] + b2[u]).  Evaluating therefore shifts
    the next epoch's row order, and the lists are not those of the unpermuted model.  Both are kept for parity."""
    _ACT = SIGMOID

    def get_recommendations_tensors(self, k: int = 10):
        """(idx, val) device tensors, rows = private users; draws the evaluation's permutation (itemautorec.py:102)."""
        perm = epoch_order(self._num_items)
        return self._model.item_topk(perm, k, self._indptr, self._sorted_idx)

    def get_rank_tensors(self, rel_indptr, rel_items):
        """The rank pass runs before the lists are drawn (RecMixin.evaluate): it ranks under the permutation the next
        get_recommendations_tensors will draw, and leaves the stream where it was."""
        state = random.getstate()
        perm = epoch_order(self._num_items)
        random.setstate(state)
        return self._model.item_rank(perm, rel_indptr, rel_items, self._indptr, self._sorted_idx)
