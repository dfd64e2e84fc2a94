"""The `mark(phase)` hook of every device model that the benchmarks under tools/ time: a build with a recording mark
gives the same bits as a build without one (weights or factor tables and the top-10 lists), and the phases arrive in the
documented order."""
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from c1_harness import DEV
from elliot_b200.recommender import knn
from elliot_b200.recommender.als import ALSModel
from elliot_b200.recommender.ease import EASEModel
from elliot_b200.recommender.knn import KNNModel
from elliot_b200.recommender.nonneg_mf import NonNegMFModel
from elliot_b200.recommender.pure_svd import PureSVDModel
from elliot_b200.recommender.rp3beta import RP3Model
from elliot_b200.recommender.slim import SlimModel
from elliot_b200.recommender.slope_one import SlopeOneModel

pytestmark = pytest.mark.gpu
U, I = 60, 40


def _case(seed=3):
    """A seeded 60 x 40 case with ratings 1-5 on a quarter of the pairs, and its train mask on the device."""
    g = np.random.default_rng(seed)
    u, i = np.nonzero(g.random((U, I)) < 0.25)
    r = g.integers(1, 6, u.size).astype(np.float32)
    ratings = sp.csr_matrix((r, (u, i)), shape=(U, I), dtype=np.float32)
    data = SimpleNamespace(sp_i_train_ratings=ratings, sp_i_train=sp.csr_matrix((np.ones_like(r), (u, i)), shape=(U, I)),
                           users=range(U), items=range(I), _tr=(u.astype(np.int64), i.astype(np.int64), r.astype(np.float64)))
    mask = (torch.from_numpy(ratings.indptr).to(DEV, torch.int64), torch.from_numpy(ratings.indices).to(DEV, torch.int32))
    return data, mask


def _check(build, outputs, phases):
    """Builds once without a mark and once with a recording one; both must give the same bits, the second `phases`."""
    plain = [t.cpu().numpy() for t in outputs(build(None))]
    seen = []
    marked = [t.cpu().numpy() for t in outputs(build(seen.append))]
    assert seen == phases
    for a, b in zip(plain, marked, strict=True):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("over", ["items", "users"])
def test_knn_phases(over):
    data, mask = _case()

    def build(mark):
        m = KNNModel(data, 7, "cosine", False, over, DEV)
        m.initialize(mark)
        return m
    _check(build, lambda m: [*m.A, *m.B, *m.topk(10, *mask)], ["densify", "gram", "neighbours", "transpose"])


def test_knn_neighbours_marks_every_slab():
    data, _ = _case()
    m = KNNModel(data, 7, "cosine", False, "items", DEV)
    _check(lambda mark: knn.neighbours(m.urm, U, I, "items", 7, True, slab_rows=8, mark=mark), list,
           ["densify"] + ["gram", "neighbours"] * 5)


def test_ease_phases():
    data, mask = _case()

    def build(mark):
        m = EASEModel(data, 100.0, DEV)
        m.initialize(mark)
        return m
    _check(build, lambda m: [m.B, *m.topk(10, *mask)], ["gram", "inverse", "weights"])


@pytest.mark.parametrize("normalize", [True, False])
def test_rp3beta_phases(normalize):
    data, mask = _case()

    def build(mark):
        m = RP3Model(data, 10, 0.9, 0.6, normalize, DEV)
        m.initialize(mark)
        return m
    _check(build, lambda m: [*m.W, *m.topk(10, *mask)],
           ["host_prepare", "upload", "similarity"] + ["normalize"] * normalize + ["prune"])


def test_slim_phases():
    data, mask = _case()

    def build(mark):
        m = SlimModel(data, 0.01, 0.1, 10, 42, DEV)
        m.initialize(mark=mark)
        return m
    _check(build, lambda m: [*m.W, m.coef_t, m.n_iter, *m.topk(10, *mask)], ["operands", "fit", "weights"])


@pytest.mark.parametrize("kind,phases", [("iALS", ["gram", "user_half", "gram", "item_half"]),
                                         ("WRMF", ["gram", "gram", "user_half", "item_half"])])
def test_als_phases(kind, phases):
    data, mask = _case()

    def build(mark):
        np.random.seed(42)
        m = ALSModel(kind, 8, data, 1.0, 0.1, 1.0, "linear", DEV)
        m.train_step(mark)
        return m
    _check(build, lambda m: [m.X, m.Y, *m.topk(10, *mask)], phases)


def test_slope_one_phases():
    data, mask = _case()

    def build(mark):
        m = SlopeOneModel(data, DEV)
        m.initialize(mark)
        return m
    _check(build, lambda m: [m.E, *m.topk(10, *mask)], ["upload", "operands", "products", "dev"])


def test_pure_svd_phases():
    data, mask = _case()

    def build(mark):
        m = PureSVDModel(5, data, 42, DEV)
        m.train_step(mark)
        return m
    n_iter = PureSVDModel(5, data, 42, DEV).n_iter
    _check(build, lambda m: [m.user_vec, m.item_vec, m.s, *m.topk(10, *mask)],
           ["upload"] + ["spmm", "orth"] * (2 * n_iter + 1) + ["spmm", "eig", "spmm", "finish"])


def test_nonneg_mf_phases():
    data, mask = _case()

    def build(mark):
        m = NonNegMFModel(data, U, I, 0.5, 4, 0.1, 0.001, random_seed=42, device=DEV)
        m.train_step(mark)
        return m
    _check(build, lambda m: [m.P, m.Q, m.bu, m.bi, *m.topk(10, *mask)], ["dots", "chain", "items", "users"])
