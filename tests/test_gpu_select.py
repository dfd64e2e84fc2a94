"""The block-wide top-k select (csrc/block_select.cuh) through every entry point that uses it, on rows built to stress
it: many exact ties straddling the k-th place across 512-candidate chunks and column tiles, values whose keys agree in
every radix digit but the last, negative values and subnormals, and k = 1, k = the number of candidates, k above it and
k = 1024.  Each result is checked exactly against a numpy lexsort on (value desc, index asc)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from elliot_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _t(a, dt=None):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)


def _dev_csr(M):
    M = sp.csr_matrix(M)
    M.sort_indices()
    return _t(M.indptr, torch.int64), _t(M.indices, torch.int32), _t(M.data.astype(np.float32))


def _bits(u):
    return np.asarray(u, np.uint32).view(np.float32)


def _row(kind, n, g):
    """One row of n fp32 values; zeros mark columns that are not candidates (neighbours) or score 0 (scores)."""
    if kind == "ties":            # four values, each repeated hundreds of times, across every chunk and tile
        v = g.choice(np.float32([3.0, 2.0, 0.5, -1.0]), n)
    elif kind == "last_digit":    # every key shares its top 22 bits, and duplicates tie as well
        v = _bits(0x3F800000 + g.integers(0, 1024, n))
    elif kind == "negsub":        # negative normals and subnormals of both signs
        v = np.where(g.random(n) < 0.5, _bits(g.integers(1, 0x800000, n)), -g.random(n).astype(np.float32))
        v = np.where(g.random(n) < 0.3, -v, v)
    elif kind == "tiny":          # subnormals and small normals of both signs, with ties
        v = _bits(g.choice(np.uint32([1, 2, 3, 0x7FFFFF, 0x800000, 0x1000000]), n)) * np.where(g.random(n) < 0.3, -1, 1)
    else:                         # "sparse": a few values, so the zeros (or the few candidates) decide the tail
        v = np.zeros(n, np.float32)
        on = g.random(n) < 0.02
        v[on] = g.choice(np.float32([1.0, 2.0, -2.0]), int(on.sum()))
    v = v.astype(np.float32)
    v[g.random(n) < 0.1] = 0.0
    return v


def _expect(vals, cand, k):
    """Indices and values of the k best candidates by (value desc, index asc)."""
    idx = np.nonzero(cand)[0]
    o = np.lexsort((idx, -vals[idx].astype(np.float64)))[:k]
    return idx[o], vals[idx[o]]


def _check(gi, gv, vals, cand, k, pad_val):
    ei, ev = _expect(vals, cand, k)
    m = len(ei)
    assert np.array_equal(gi[:m], ei)
    assert np.array_equal(gv[:m].view(np.uint32), ev.view(np.uint32))
    assert np.all(gi[m:] == -1) and np.all(gv[m:] == pad_val)
    return m


# ---------------------------------------------------------------- neighbours: u32 keys, 11 + 11 + 10 bits
KINDS = ["ties", "last_digit", "negsub", "tiny", "sparse"]


@pytest.mark.parametrize("k", [1, 60, 1024, 1000])
def test_knn_neighbors_select(k):
    g = np.random.default_rng(k)
    n = 3000 if k != 1000 else 900                                           # k = 1000: more than the candidates
    rows = np.stack([_row(kind, n, g) for kind in KINDS])
    exact = np.zeros(n, np.float32)                                          # exactly min(k, n) candidates
    exact[g.choice(n, min(k, n), replace=False)] = 1.5
    rows = np.vstack([rows, exact[None, :]])
    diag = _t(np.ones(n, np.float32))
    idx, val, cnt = ops.knn_neighbors(_t(rows), n, 0, diag, k, cosine=False, dot_scale=1.0)
    idx, val, cnt = idx.cpu().numpy(), val.cpu().numpy(), cnt.cpu().numpy()
    for r in range(rows.shape[0]):
        m = _check(idx[r], val[r], rows[r], rows[r] != 0, k, 0.0)
        assert cnt[r] == m
    assert cnt[-1] == min(k, n)


# ---------------------------------------------------------------- scores: identity A, so a score row is a B row
def _score_case(n_cols, n_masked, seed):
    g = np.random.default_rng(seed)
    R = np.stack([_row(kind, n_cols, g) for kind in KINDS])
    mask = np.zeros(R.shape, bool)
    for r in range(R.shape[0]):
        mask[r, g.choice(n_cols, n_masked, replace=False)] = True
    n = R.shape[0]
    A = _dev_csr(sp.identity(n, np.float32, format="csr"))
    M = _dev_csr(mask)
    return R, mask, A, M


SCORE_CASES = [                   # (n_cols, masked columns per row, k)
    (3000, 100, 1),
    (3000, 100, 1024),
    (700, 100, 600),              # k = the number of candidates
    (300, 20, 1024),              # k above it
    (60000, 500, 1024),           # wider than one column tile of either kernel
    (60000, 1, 77),
]


@pytest.mark.parametrize("n_cols,n_masked,k", SCORE_CASES)
@pytest.mark.parametrize("masked", [False, True])
def test_rp3_score_topk_select(n_cols, n_masked, k, masked):
    R, mask, A, M = _score_case(n_cols, n_masked, n_cols + k)
    if n_cols > 3000:
        assert n_cols > ops.rp3_tile_cols()
    kw = dict(mask_indptr=M[0], mask_indices=M[1]) if masked else {}
    idx, val = ops.rp3_score_topk(A, _dev_csr(R), n_cols, k, **kw)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    for r in range(R.shape[0]):
        # a score is 0 + 1 * b in fp32: b itself (+0.0 where B has no entry)
        _check(idx[r], val[r], R[r] + np.float32(0.0), ~mask[r] if masked else np.ones(n_cols, bool), k, -np.inf)


@pytest.mark.parametrize("n_cols,n_masked,k", SCORE_CASES)
@pytest.mark.parametrize("frac_bits", [24, 170])
def test_knn_and_dense_score_topk_select(n_cols, n_masked, k, frac_bits):
    R, mask, A, M = _score_case(n_cols, n_masked, n_cols + k + frac_bits)
    if frac_bits == 24:
        R[3] = R[0]                                                          # no subnormals: they vanish at 2^-24
    else:
        R = np.where(np.abs(R) < 2.0 ** -100, R, R * np.float32(2.0 ** -111)).astype(np.float32)
    # B on the 2^-f grid (every |b| 2^f an integer below 2^61), so each score is fp32(rint(b 2^f) 2^-f) = b
    R = (np.rint(R.astype(np.float64) * 2.0 ** frac_bits) * 2.0 ** -frac_bits).astype(np.float32)
    assert np.abs(R.astype(np.float64)).max() * 2.0 ** frac_bits < 2.0 ** 61
    if n_cols > 3000:
        assert n_cols > ops.knn_score_tile_cols()
    ki, kv = ops.knn_score_topk(A, _dev_csr(R), n_cols, k, frac_bits, M[0], M[1])
    di, dv = ops.dense_score_topk(A, _t(R), k, frac_bits, M[0], M[1])
    ki, kv, di, dv = (x.cpu().numpy() for x in (ki, kv, di, dv))
    for r in range(R.shape[0]):
        _check(ki[r], kv[r], R[r] + np.float32(0.0), ~mask[r], k, -np.inf)
    assert np.array_equal(di, ki) and np.array_equal(dv.view(np.uint32), kv.view(np.uint32))


# ---------------------------------------------------------------- column prune: u64 (value, row) keys per column
@pytest.mark.parametrize("k", [1, 7, 1024, 5000])
def test_rp3_prune_cols_select(k):
    g = np.random.default_rng(k)
    n, stride = 2000, 160
    hot = {0: "ties", 1: "last_digit", 2: "negsub", 3: "tiny", 4: "ties"}    # every row lists these columns
    cols_val = {c: _row(kind, n, g) for c, kind in hot.items()}
    exact = np.zeros(n, np.float32)
    exact[g.choice(n, 1024, replace=False)] = 0.25                           # column 5: exactly 1 024 candidates
    cols_val[5] = exact
    D = np.zeros((n, n), np.float32)
    for c, v in cols_val.items():
        D[:, c] = v
    for r in range(n):                                                       # and a few random others, ties included
        c = g.choice(np.arange(6, n), 40, replace=False)
        D[r, c] = g.choice(np.float32([1.0, 0.5, 0.0, -3.0]), 40)
    idx = np.full((n, stride), -1, np.int32)
    val = np.zeros((n, stride), np.float32)
    cnt = np.zeros(n, np.int32)
    for r in range(n):                                                       # zeros stay listed: the prune drops them
        c = np.nonzero((D[r] != 0) | (np.arange(n) < 6))[0]
        cnt[r] = len(c)
        idx[r, :len(c)], val[r, :len(c)] = c, D[r, c]
    ip, ii, iv = ops.rp3_prune_cols(_t(idx), _t(val), _t(cnt), k)
    got = sp.csr_matrix((iv.cpu().numpy(), ii.cpu().numpy(), ip.cpu().numpy()), shape=(n, n))
    keep = np.zeros((n, n), bool)
    for c in range(n):
        rows, _ = _expect(D[:, c], D[:, c] != 0, k)
        keep[rows, c] = True
    want = sp.csr_matrix(np.where(keep, D, 0))
    assert np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
    assert np.array_equal(got.data.view(np.uint32), want.data.view(np.uint32))
    assert keep[:, 5].sum() == min(k, 1024)
