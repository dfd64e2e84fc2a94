"""GPU parity tests for full-catalogue scoring + mask + top-k through the C ABI."""
import numpy as np
import pytest
import torch

import oracle
from elliot_b200 import ops
from oracle.topk_bound import check_topk_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _mask_dev(g):
    return (torch.from_numpy(g["ui_indptr"].astype(np.int64)).to(DEV),
            torch.from_numpy(g["ui_indices"].astype(np.int32)).to(DEV))


def test_topk_f64_equals_reference_lists(golden):
    """fp64 tables: index lists identical to MFModel.get_user_predictions, scores within 1e-12."""
    g = golden
    d, k = int(g["d"]), int(g["k"])
    U = torch.from_numpy(g["U"]).to(DEV); V = torch.from_numpy(g["V"]).to(DEV); b = torch.from_numpy(g["b"]).to(DEV)
    mp, mi = _mask_dev(g)
    idx, val = ops.score_topk(U, V, b, d, k, mp, mi)
    torch.cuda.synchronize()
    assert np.array_equal(idx.cpu().numpy(), g["rec_idx"])
    fin = np.isfinite(g["rec_val"])
    assert np.abs(val.cpu().numpy() - g["rec_val"])[fin].max() < 1e-12


def test_topk_f32_padded_tables(golden):
    """fp32 padded tables vs the oracle run on the SAME fp32-rounded values: identical lists
    wherever the oracle's gap between consecutive scores exceeds 1e-5 (fp32 dot noise)."""
    g = golden
    d, k = int(g["d"]), int(g["k"]); ld = ops.padded_dim(d)
    nu, ni = len(g["users"]), len(g["items"])
    U32 = np.zeros((nu, ld), np.float32); U32[:, :d] = g["U"]
    V32 = np.zeros((ni, ld), np.float32); V32[:, :d] = g["V"]
    b32 = g["b"].astype(np.float32)
    mp, mi = _mask_dev(g)
    idx, val = ops.score_topk(torch.from_numpy(U32).to(DEV), torch.from_numpy(V32).to(DEV),
                              torch.from_numpy(b32).to(DEV), d, k, mp, mi)
    torch.cuda.synchronize()
    oi, ov = oracle.user_topk(U32[:, :d].astype(np.float64), V32[:, :d].astype(np.float64), b32.astype(np.float64),
                              g["ui_indptr"], g["ui_indices"], np.arange(nu), k + 1)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    gaps = np.abs(np.diff(ov, axis=1))
    safe = np.all(~np.isfinite(gaps) | (gaps > 1e-5), axis=1)
    assert safe.mean() > 0.9
    assert np.array_equal(idx[safe], oi[safe, :k])
    fin = np.isfinite(ov[:, :k])
    assert np.abs(val - ov[:, :k])[fin].max() < 1e-5


def test_topk_user_subset_and_no_mask(golden_small):
    g = golden_small
    d = int(g["d"])
    U = torch.from_numpy(g["U"]).to(DEV); V = torch.from_numpy(g["V"]).to(DEV)
    users = np.array([5, 0, 399, 17, 17], np.int32)
    idx, val = ops.score_topk(U, V, None, d, 7, users=torch.from_numpy(users).to(DEV))
    oi, ov = oracle.user_topk(g["U"], g["V"], None, None, None, users, 7)
    assert np.array_equal(idx.cpu().numpy(), oi) and np.abs(val.cpu().numpy() - ov).max() < 1e-12


def test_topk_fewer_candidates_than_k():
    """A user who rated all but 3 items: 3 finite entries, then idx -1 / -inf padding; exact ties
    resolve to the lower item index."""
    ni, d, k = 12, 8, 5
    rs = np.random.RandomState(3)
    U = rs.normal(size=(2, d)); V = rs.normal(size=(ni, d))
    V[7] = V[4]                                   # exact tie between items 4 and 7
    indptr = np.array([0, ni - 3, ni - 3], np.int64)
    indices = np.array([x for x in range(ni) if x not in (2, 4, 7)], np.int32)
    idx, val = ops.score_topk(torch.from_numpy(U).to(DEV), torch.from_numpy(V).to(DEV), None, d, k,
                              torch.from_numpy(indptr).to(DEV), torch.from_numpy(indices).to(DEV))
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    oi, ov = oracle.user_topk(U, V, None, indptr, indices, np.arange(2), k)
    assert np.array_equal(idx, oi)
    assert set(idx[0, :3]) == {2, 4, 7} and list(idx[0, 3:]) == [-1, -1] and np.isinf(val[0, 3:]).all()
    p4, p7 = list(idx[0]).index(4), list(idx[0]).index(7)
    assert p4 + 1 == p7


@pytest.mark.parametrize("k", [17, 50, 100])
@pytest.mark.parametrize("d", [1, 3, 33, 255])
@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_topk_long_lists_vs_fp64_oracle(dtype, d, k):
    """Lists longer than the tensor-core kernel keeps (k > 16 goes to this kernel), against the fp64 oracle on the same
    tables: a `users` list with repeated ids, k + 8 copies of one item row that the even users rank first (exact ties
    across rank k, lower index first), then a catalogue smaller than k (-1 / -inf padding)."""
    nu, ni, ld = 60, 700, ops.padded_dim(d)
    rs = np.random.RandomState(1000 * d + k)
    U = np.zeros((nu, ld)); V = np.zeros((ni, ld))
    U[:, :d] = rs.normal(0, 0.1, (nu, d)); V[:, :d] = rs.normal(0, 0.1, (ni, d))
    b = rs.normal(0, 0.05, ni)
    U[::2, 0] = 1.0
    dup = np.sort(rs.choice(ni, size=k + 8, replace=False))
    V[dup, :d] = V[dup[0], :d]; V[dup, 0] = 0.5; b[dup] = b[dup[0]]
    rows = [np.sort(rs.choice(ni, size=rs.randint(0, 30), replace=False)).astype(np.int32) for _ in range(nu)]
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    indices = np.concatenate(rows)
    users = np.concatenate([[7, 7, 0, nu - 1, 8, 7], rs.randint(0, nu, 34)]).astype(np.int32)
    U, V, b = U.astype(dtype), V.astype(dtype), b.astype(dtype)
    unit = 2.0 ** -24 if dtype == np.float32 else 2.0 ** -53
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)

    idx, val = ops.score_topk(dev(U), dev(V), dev(b), d, k, dev(indptr), dev(indices), users=dev(users))
    q, n = check_topk_fp64(U, V, b, d, k, indptr, indices, users, idx.cpu().numpy(), val.cpu().numpy(), unit)
    assert q >= 0.9 * n, (q, n)
    assert np.array_equal(idx[0].cpu().numpy(), idx[1].cpu().numpy())   # repeated user id: the same list

    small = k // 2                                    # fewer items than k
    idx, val = ops.score_topk(dev(U), dev(V[:small]), dev(b[:small]), d, k, users=dev(users))
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    assert (idx[:, small:] == -1).all() and np.isneginf(val[:, small:]).all()
    q, n = check_topk_fp64(U, V[:small], b[:small], d, k, None, None, users, idx, val, unit)
    assert q >= 0.9 * n, (q, n)


def _dense_topk_reference(scores, k, indptr, indices, rows, shift):
    """stable arg-sort of the masked scores, -inf never returned, padded with -1 / -inf; values score + shift in fp32"""
    n, ni = scores.shape
    idx = np.full((n, k), -1, np.int32); val = np.full((n, k), -np.inf, np.float32)
    for r in range(n):
        s = scores[r].copy()
        if indptr is not None:
            s[indices[indptr[rows[r]]:indptr[rows[r] + 1]]] = -np.inf
        order = np.argsort(-s, kind="stable")
        order = order[np.isfinite(s[order])][:k]
        idx[r, :len(order)] = order
        val[r, :len(order)] = s[order] + shift[r]
    return idx, val


@pytest.mark.parametrize("with_shift", [False, True], ids=["no_shift", "shift"])
@pytest.mark.parametrize("k", [1, 10, 100, "all+1"])
@pytest.mark.parametrize("ni", [1, 255, 256, 257, 26744])
def test_dense_topk_equals_stable_argsort(ni, k, with_shift):
    """ops.dense_topk (MultiVAE / NeuMF lists) does no arithmetic but `+ shift`, so the numpy reference is exact: the same
    indices (ties -> lower index) and bit-identical values.  Scores on a coarse grid tie often; some are -inf on input; the
    block is a strided view (ld > n_items) and its rows map to other users' mask rows."""
    k = ni + 1 if k == "all+1" else k
    rs = np.random.RandomState(ni + (k % 1000))
    n, n_users, ld = 7, 12, ni + 37
    rows = np.array([5, 0, 11, 3, 3, 9, 1], np.int32)
    buf = np.full((n, ld), 7.0, np.float32)           # columns past n_items: never ranked, never written
    buf[:, :ni] = np.round(rs.normal(size=(n, ni)) * 8) / 8
    buf[:, :ni][rs.random_sample((n, ni)) < 0.02] = -np.inf
    mrows = []
    for u in range(n_users):
        if u == 9:
            mrows.append(np.arange(ni))                # row 5: nothing left
        elif u == 11:
            mrows.append(np.setdiff1d(np.arange(ni), rs.choice(ni, size=min(4, ni), replace=False)))   # row 2: <= 4 left
        else:
            mrows.append(np.sort(rs.choice(ni, size=rs.randint(0, ni // 3 + 1), replace=False)))
    indptr = np.zeros(n_users + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in mrows])
    indices = np.concatenate(mrows).astype(np.int32)
    shift = (rs.normal(size=n) * 3).astype(np.float32) if with_shift else np.zeros(n, np.float32)

    block = torch.from_numpy(buf).to(DEV)              # the kernel overwrites it; the reference reads the host copy
    scores = block[:, :ni]
    assert scores.stride(0) == ld
    idx, val = ops.dense_topk(scores, k, torch.from_numpy(indptr).to(DEV),
                              torch.from_numpy(indices).to(DEV), torch.from_numpy(rows).to(DEV),
                              shift=torch.from_numpy(shift).to(DEV) if with_shift else None)
    ri, rv = _dense_topk_reference(buf[:, :ni], k, indptr, indices, rows, shift)
    assert np.array_equal(idx.cpu().numpy(), ri)
    assert np.array_equal(val.cpu().numpy().view(np.int32), rv.view(np.int32))
    assert (block[:, ni:] == 7.0).all()
