"""SVD++ and FunkSVD, the reference's rating-prediction factor models, on the H100 behind the reference's model surface.

Mirrors latent_factor_models/SVDpp/svdpp.py + svdpp_model.py: out = (p_u + mean_{j in N(u)} y_j) . q_i + b_u + b_i + g,
N(u) the user's train row (a MEAN, not Koren's |N(u)|^-1/2), GlorotUniform tables (an [n, 1] bias table has fan_in n,
fan_out 1), g = 0 at the start; `transactions` samples per epoch from custom_pointwise_sparse_sampler.py (u uniform, i
uniform over u's train row, label = its train rating); Keras MeanSquaredError (batch mean; the last batch may be short) and
Keras Adam over P, Q, Y, b_u, b_i and g.  And FunkSVD/funk_svd.py + funk_svd_model.py: out = p_u . q_i + b_u + b_i, the
pointwise pos/neg sampler with labels 0/1, MSE and Adam; its model is built without `random_seed`, so it always starts
from seed 42.

`reg_w` and `reg_b` are parsed and have no effect: the reference attaches them as Embedding regularizers, but its
train_step differentiates `self.loss(label, output)` alone, so they never reach a gradient.

Per batch: eb_implicit_mean_f32 forms the batch's user vectors z (SVD++), ONE fused kernel (eb_rating_mf_step_f32) does
gather -> predict -> error -> loss -> gradient scatter (dY over each sample's train row for SVD++), and the dense Keras Adam
(eb_adam_dense_f32) moves every table.  Recommendations score z . q_i + b_i for every user with the scoring kernels and
add b_u + g to the kept values only (a per-user constant changes no ranking); the rank pass (AUC / GAUC) ranks the same
scores and the pair pass (MAE / MSE / RMSE) scores every relevant test item as the full list would.  The initial tables
come from a torch generator and the samples from a Philox stream: TensorFlow's streams are not replayed, and TensorFlow
parity is UNPINNED (checker: oracle/rating_mf.py).  `factors` is padded to the kernels' row stride; it must be <= 128.

MF, PMF and FM (latent_factor_models/MF, PMF, FM without side information) are configurations of the same model: MF has
no bias tables, PMF adds RandomNormal(0.01) tables and a sigmoid head (eb_pointwise_mf_step_f32; its scores get the
sigmoid after selection), FM has zero-initialised biases and g and takes the pointwise sampler's labels with each
positive's train rating written in (eb_rating_labels_f32).  DESIGN §4.20; checker: oracle/pointwise_mf.py.
"""
import math
import pickle

import torch

from .. import ops
from ..dataset import train_csr_of
from ._bases import BaseRecommenderModel, RecMixin, init_charger
from ._device import PairScoreRecs, RankRecs, TopKRecs, cuda_device, upload


def _pad4(n):
    return (n + 3) // 4 * 4


class RatingMFModel:
    """The tables, the training step and the scoring of SVD++ (implicit=True) and FunkSVD (implicit=False), and of MF,
    PMF and FM, which configure:
      bias         "glorot" (SVD++, FunkSVD), "zero" (FM) or "none" (MF, PMF): the b_u / b_i tables
      global_bias  the scalar g (SVD++, FM); defaults to `implicit`
      init         "glorot" (GlorotUniform) or "normal" (PMF's RandomNormal(stddev=0.01)) for the factor tables
      head         "linear" (out = z.q + biases) or "sigmoid" (PMF: out = sigmoid(p.q), eb_pointwise_mf_step_f32)
    The train CSR (indptr int64, sorted indices int32) is the user rows N(u) of SVD++ and the mask of every scoring pass."""

    def __init__(self, num_users, num_items, factors, learning_rate, random_seed, indptr, indices, implicit, device,
                 bias="glorot", global_bias=None, init="glorot", head="linear"):
        assert 1 <= factors <= 128, "factors must be <= 128"
        assert bias in ("glorot", "zero", "none") and init in ("glorot", "normal") and head in ("linear", "sigmoid")
        assert head == "linear" or (bias == "none" and not global_bias and not implicit), "the sigmoid head is PMF's: p.q only"
        self.nu, self.ni, self.f, self.lr, self.implicit = num_users, num_items, factors, learning_rate, implicit
        self.head = head
        self.fp = (factors + 3) // 4 * 4                                # kernels work on float4 columns; padding stays zero
        self.ld = ops.padded_dim(self.fp)
        self.device = torch.device(device)
        self.indptr, self.indices = indptr, indices
        g = torch.Generator(device=self.device); g.manual_seed(int(random_seed))

        def glorot(rows, cols, fan_in, fan_out, shape):                 # tf.initializers.GlorotUniform
            lim = math.sqrt(6.0 / (fan_in + fan_out))
            t = torch.zeros(shape, device=self.device)
            t.view(-1, shape[-1] if len(shape) == 2 else 1)[:rows, :cols] = \
                (torch.rand((rows, cols), device=self.device, generator=g) * 2 - 1) * lim
            return t
        def normal(rows, cols, shape):                                   # tf.initializers.RandomNormal(stddev=0.01)
            t = torch.zeros(shape, device=self.device)
            t[:rows, :cols] = torch.randn((rows, cols), device=self.device, generator=g) * 0.01
            return t
        f, ld = factors, self.ld
        table = (lambda n: glorot(n, f, n, f, (n, ld))) if init == "glorot" else (lambda n: normal(n, f, (n, ld)))
        self.P = {"P": table(num_users), "Q": table(num_items)}
        if implicit:
            self.P["Y"] = table(num_items)
        # bias vectors (and g) padded to a multiple of 4 for the vector Adam; the padding has no gradient and stays zero
        if bias == "glorot":
            self.P["bu"] = glorot(num_users, 1, num_users, 1, (_pad4(num_users),))
            self.P["bi"] = glorot(num_items, 1, num_items, 1, (_pad4(num_items),))
        elif bias == "zero":
            self.P["bu"] = torch.zeros(_pad4(num_users), device=self.device)
            self.P["bi"] = torch.zeros(_pad4(num_items), device=self.device)
        if implicit if global_bias is None else global_bias:
            self.P["g"] = torch.zeros(4, device=self.device)
        z = lambda t: torch.zeros_like(t)
        self.G = {k: z(v) for k, v in self.P.items()}
        self.M = {k: z(v) for k, v in self.P.items()}
        self.V = {k: z(v) for k, v in self.P.items()}
        self.step = 0
        self._loss = torch.zeros(1, dtype=torch.float64, device=self.device)
        self._z = None

    def batch_means(self, u):
        """SVD++ user vectors of a batch: Z[s] = P[u_s] + mean over u_s's train row of Y."""
        if self._z is None or self._z.shape[0] < u.numel():
            self._z = torch.zeros((u.numel(), self.ld), device=self.device)
        return ops.implicit_mean_f32(self.P["P"], self.P["Y"], self.fp, self.indptr, self.indices, users=u, out=self._z)

    def grads(self, batch, z=None):
        """Add the batch's gradients to self.G and its loss to self._loss; z: the batch's implicit means (SVD++)."""
        u, it, y = batch
        P, G = self.P, self.G
        if self.head == "sigmoid":
            ops.pointwise_mf_step_f32(P["P"], P["Q"], self.fp, u, it, y, G["Q"], ops.PMF_MSE, dP=G["P"], loss=self._loss)
            return
        ops.rating_mf_step_f32(P["P"], P["Q"], P.get("bu"), P.get("bi"), P.get("g"), self.fp, u, it, y, G["P"], G["Q"], G.get("bu"),
                               G.get("bi"), G.get("g"), Z=z, indptr=self.indptr if self.implicit else None,
                               indices=self.indices if self.implicit else None, dY=G.get("Y"), loss=self._loss)

    def adam(self):
        self.step += 1
        for k in self.P:
            ops.adam_dense_f32(self.P[k], self.M[k], self.V[k], self.G[k], self.lr, self.step)

    def train_step(self, batch):
        """batch = (user int32, item int32, label float32) device tensors; returns the batch loss tensor (device)."""
        self._loss.zero_()
        self.grads(batch, self.batch_means(batch[0]) if self.implicit else None)
        self.adam()
        return self._loss

    def user_vectors(self):
        """z_u of every user: p_u + mean of y_j over N(u) (SVD++), p_u (FunkSVD)."""
        if not self.implicit:
            return self.P["P"]
        return ops.implicit_mean_f32(self.P["P"], self.P["Y"], self.fp, self.indptr, self.indices)

    def topk(self, k, mask_indptr, mask_indices):
        """masked top-k of z_u . q_i + b_i + b_u + g for all users (get_recs / get_top_k); PMF: selected on p.q, the
        sigmoid applied to the kept values (it is monotone)."""
        Z = self.user_vectors()
        if k <= 16:
            idx, val, _ = ops.score_topk_tc(Z, self.P["Q"], self.P.get("bi"), self.f, k, mask_indptr, mask_indices, stats=False)
        else:
            idx, val = ops.score_topk(Z, self.P["Q"], self.P.get("bi"), self.f, k, mask_indptr, mask_indices)
        if self.head == "sigmoid":
            return idx, ops.sigmoid_scores_(val.contiguous())
        if "bu" not in self.P:
            return idx, val
        return idx, ops.add_row_offset_(val, self.P["bu"], self.P.get("g"))

    def rank(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """The lists topk() selects from, without b_u + g (a per-user constant) and before PMF's sigmoid (monotone)."""
        return ops.score_rank(self.user_vectors(), self.P["Q"], self.P.get("bi"), self.f, rel_indptr, rel_items, mask_indptr,
                              mask_indices)

    def pair_scores(self, rel_indptr, rel_items, mask_indptr, mask_indices):
        """Each relevant entry's score in the user's full list (-inf for a train item, NaN outside the catalogue)."""
        s = ops.score_pairs_f32(self.user_vectors(), self.P["Q"], self.fp, rel_indptr, rel_items, item_bias=self.P.get("bi"),
                                user_off=self.P.get("bu"), global_off=self.P.get("g"), mask_indptr=mask_indptr,
                                mask_indices=mask_indices)
        return ops.sigmoid_scores_(s) if self.head == "sigmoid" else s

    def get_model_state(self):
        return {"P": {k: v.cpu().numpy() for k, v in self.P.items()}, "step": self.step,
                "M": {k: v.cpu().numpy() for k, v in self.M.items()}, "V": {k: v.cpu().numpy() for k, v in self.V.items()}}

    def set_model_state(self, s):
        for k in self.P:
            self.P[k].copy_(torch.from_numpy(s["P"][k])); self.M[k].copy_(torch.from_numpy(s["M"][k])); self.V[k].copy_(torch.from_numpy(s["V"][k]))
        self.step = s["step"]

    def save_weights(self, path):
        with open(path, "wb") as fh:
            pickle.dump(self.get_model_state(), fh)

    def load_weights(self, path):
        with open(path, "rb") as fh:
            self.set_model_state(pickle.load(fh))


class _RatingMF(TopKRecs, RankRecs, PairScoreRecs, RecMixin, BaseRecommenderModel):
    """What SVDpp and FunkSVD share: the reference's parameters (factors, lr, reg_w, reg_b), the batch size, the tables."""

    _implicit = False
    _param_rows = [
        ("_factors", "factors", "factors", 10, None, None),
        ("_learning_rate", "lr", "lr", 0.001, None, None),
        ("_lambda_weights", "reg_w", "reg_w", 0.1, None, None),
        ("_lambda_bias", "reg_b", "reg_b", 0.001, None, None),
    ]
    _model_kwargs = {}                                                    # RatingMFModel's bias / global_bias / init / head

    def _setup(self, who, seed, check_factors=False):
        self._params_list = list(self._param_rows)
        self.autoset_params()
        if check_factors and not 1 <= int(self._factors) <= 128:
            raise ValueError(f"{who}: factors={self._factors} is outside [1, 128], the widths the step and scoring kernels take")
        if self._batch_size < 1:
            self._batch_size = self._data.transactions
        self._device = cuda_device(self._params, who)
        self._indptr, _, self._sorted_idx = train_csr_of(self._data, self._device, set_order=False)
        self._model = RatingMFModel(self._num_users, self._num_items, int(self._factors), self._learning_rate, seed,
                                    self._indptr, self._sorted_idx, self._implicit, self._device, **self._model_kwargs)
        self._drawn = 0

    def _train_ratings(self):
        """The train ratings on the device, aligned with the sorted train CSR."""
        m = self._data.sp_i_train_ratings.tocsr()
        if not m.has_sorted_indices:
            m = m.sorted_indices()
        assert m.nnz == self._sorted_idx.numel(), "sp_i_train_ratings and sp_i_train disagree"
        return upload(m.data, self._device, torch.float32)

    def _samples(self, T):
        raise NotImplementedError

    def train(self):
        if self._restore:
            return self.restore_weights()
        T = self._data.transactions
        for it in self.iterate(self._epochs):
            loss = 0.0
            u, i, y = self._samples(T)
            self._drawn += T
            for s in range(0, T, self._batch_size):
                e = min(s + self._batch_size, T)
                loss += float(self._model.train_step((u[s:e], i[s:e], y[s:e])).item())
            self.evaluate(it, loss / (it + 1))


class SVDpp(_RatingMF):
    r"""SVD++ (https://dl.acm.org/doi/10.1145/1401890.1401944).  YAML keys as in the reference (factors, lr, reg_w,
    reg_b); optional keys `b200_eval` and `b200_device`."""

    _implicit = True

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._setup("SVDpp", self._seed)
        self._ratings = self._train_ratings()

    @property
    def name(self):
        return "SVDpp" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def _samples(self, T):
        return ops.rated_sample_philox(self._num_users, self._num_items, self._indptr, self._sorted_idx, self._ratings, T, 42,
                                       first=self._drawn)


class FunkSVD(_RatingMF):
    r"""FunkSVD (https://sifter.org/~simon/journal/20061211.html).  YAML keys as in the reference (factors, lr, reg_w,
    reg_b); optional keys `b200_eval` and `b200_device`."""

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._setup("FunkSVD", 42)                                        # FunkSVDModel is built without random_seed
        self._filter = ops.bloom_build(self._indptr, self._sorted_idx, self._num_users)

    @property
    def name(self):
        return "FunkSVD" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def _samples(self, T):
        return ops.pointwise_sample_philox(self._num_users, self._num_items, self._indptr, self._sorted_idx, T, 42,
                                           first=self._drawn, filter=self._filter)


class MF(_RatingMF):
    r"""Matrix Factorization (latent_factor_models/MF): out = p_u . q_i, GlorotUniform tables, no biases, Keras MSE and
    Adam, the pointwise pos/neg sampler (labels 0 / 1).  YAML keys as in the reference (factors, lr, reg); `reg` is parsed
    and has no effect, as in the reference.  Optional keys `b200_eval` and `b200_device`."""

    _param_rows = [
        ("_factors", "factors", "factors", 10, None, None),
        ("_learning_rate", "lr", "lr", 0.001, None, None),
        ("_l_w", "reg", "reg", 0.1, None, None),
    ]
    _model_kwargs = {"bias": "none"}

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._setup(type(self).__name__, self._seed, check_factors=True)
        self._filter = ops.bloom_build(self._indptr, self._sorted_idx, self._num_users)

    @property
    def name(self):
        return "MF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def _samples(self, T):
        return ops.pointwise_sample_philox(self._num_users, self._num_items, self._indptr, self._sorted_idx, T, 42,
                                           first=self._drawn, filter=self._filter)


class PMF(MF):
    r"""Probabilistic Matrix Factorization (latent_factor_models/PMF): out = sigmoid(p_u . q_i), RandomNormal(stddev=0.01)
    tables, Keras MSE of the sigmoid and Adam, the pointwise pos/neg sampler.  YAML keys as in the reference (lr, factors,
    reg, gaussian_variance); `reg` and `gaussian_variance` are parsed and have no effect, as in the reference (its
    GaussianNoise layer is called outside training mode, DESIGN §4.20).  Optional keys `b200_eval` and `b200_device`."""

    _param_rows = [
        ("_learning_rate", "lr", "lr", 0.001, None, None),
        ("_factors", "factors", "factors", 50, None, None),
        ("_l_w", "reg", "reg", 0.0025, None, None),
        ("_gvar", "gaussian_variance", "gvar", 0.1, None, None),
    ]
    _model_kwargs = {"bias": "none", "init": "normal", "head": "sigmoid"}

    @property
    def name(self):
        return "PMF" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"


class FM(_RatingMF):
    r"""Factorization Machines without side information (latent_factor_models/FM with MatrixFactorizationLayer):
    out = p_u . q_i + b_u + b_i + g, GlorotUniform tables, zero biases, g = 0, Keras MSE and Adam over all five, the
    pointwise pos/neg ratings sampler (a positive carries its train rating, a negative 0).  YAML keys as in the reference
    (factors, lr, reg, loader); `reg` is parsed and has no effect.  A dataset whose `loader` side information has features
    is refused: the feature model is outside this build.  Optional keys `b200_eval` and `b200_device`."""

    _param_rows = [
        ("_factors", "factors", "factors", 10, int, None),
        ("_learning_rate", "lr", "lr", 0.001, float, None),
        ("_l_w", "reg", "reg", 0.1, float, None),
        ("_loader", "loader", "load", "ItemAttributes", None, None),
    ]
    _model_kwargs = {"bias": "zero", "global_bias": True}

    @init_charger
    def __init__(self, data, config, params, *args, **kwargs):
        self._setup(type(self).__name__, self._seed, check_factors=True)
        side = getattr(getattr(self._data, "side_information", None), self._loader, None)
        if hasattr(side, "nfeatures") and hasattr(side, "feature_map"):
            raise NotImplementedError(f"{type(self).__name__}: side information ({self._loader}) is not supported: the "
                                      "FactorizationMachineLayer over item features is outside this build; run FM without it")
        self._filter = ops.bloom_build(self._indptr, self._sorted_idx, self._num_users)
        self._ratings = self._train_ratings()

    @property
    def name(self):
        return "FM" + f"_{self.get_base_params_shortcut()}" + f"_{self.get_params_shortcut()}"

    def _samples(self, T):
        u, i, y = ops.pointwise_sample_philox(self._num_users, self._num_items, self._indptr, self._sorted_idx, T, 42,
                                              first=self._drawn, filter=self._filter)
        return u, i, ops.rating_labels_(self._indptr, self._sorted_idx, self._ratings, u, i, y)
