"""Top-k lists computed in fp32 or fp64 against the fp64 oracle, with a rounding-error bound per user.  TEST INFRASTRUCTURE.

A kernel that scores user u against item i in a table precision with unit roundoff `unit` (2^-24 for fp32, 2^-53 for fp64)
is off the exact score by at most

    B_u = (d + 2) * unit * (||u|| * max_i ||v_i|| + max_i |b_i|)

(d products and sums plus the bias addition).  So, for the oracle run on the same tables widened to fp64:
  - every returned value lies within B_u of the fp64 score of the returned item;
  - the returned items' fp64 scores, sorted, lie within 2 B_u of the oracle's top k;
  - an oracle item whose score is more than 2 B_u away from both neighbours in the oracle's top k + 1 has exactly that rank
    in the kernel's list too: every item above it scores more than its own fp32 score, every item below it less.
Identical item rows (and biases) get identical scores in any kernel that scores every item with the same operations, so
a zero gap between two of them separates them as well as a wide one: both lists put the lower index first.
"""
import numpy as np

from . import user_topk


def _masked(mask_indptr, mask_indices, users, idx):
    """(n, k) bool: idx[r, j] is a train item of users[r]"""
    out = np.zeros(idx.shape, bool)
    if mask_indptr is None:
        return out
    for r, u in enumerate(users):
        out[r] = np.isin(idx[r], mask_indices[mask_indptr[u]:mask_indptr[u + 1]])
    return out


def check_topk_fp64(U, V, b, d, k, mask_indptr, mask_indices, users, idx, val, unit):
    """U, V, b: the tables the kernel scored (numpy; columns past d ignored; b may be None).  users: the user id of every output
    row.  idx, val: the kernel's (len(users), k) lists.  Asserts the three properties above and returns
    (filled ranks that qualified for the exact index check, filled ranks) so that the caller can make sure the check was
    not empty."""
    U = np.asarray(U, np.float64)[:, :d]
    V = np.asarray(V, np.float64)[:, :d]
    bb = np.zeros(len(V)) if b is None else np.asarray(b, np.float64)
    users = np.asarray(users, np.int64)
    idx = np.asarray(idx); val = np.asarray(val, np.float64)
    if mask_indptr is not None:
        mask_indptr = np.asarray(mask_indptr, np.int64); mask_indices = np.asarray(mask_indices, np.int32)
    n = len(users)
    assert idx.shape == (n, k) and val.shape == (n, k)
    oi, ov = user_topk(U, V, None if b is None else bb, mask_indptr, mask_indices, users, k + 1)
    vmax = np.sqrt((V * V).sum(1)).max()
    B = (d + 2) * unit * (np.sqrt((U[users] ** 2).sum(1)) * vmax + (np.abs(bb).max() if b is not None else 0.0))
    B = B[:, None]

    # padding: -1 / -inf exactly where the oracle ran out of candidates; no train item, no repeated item
    got = idx >= 0
    assert np.array_equal(got, np.isfinite(ov[:, :k])), "list lengths differ from the oracle's"
    assert np.all(np.isneginf(val[~got])), "padding values must be -inf"
    assert not (_masked(mask_indptr, mask_indices, users, idx) & got).any(), "a train item was returned"
    for r in range(n):
        assert len(np.unique(idx[r, got[r]])) == got[r].sum(), f"row {r} repeats an item"

    # values: within B_u of the returned item's fp64 score
    j = np.where(got, idx, 0)
    s = np.einsum("nd,nkd->nk", U[users], V[j]) + bb[j]
    err = np.where(got, np.abs(val - s), 0.0)
    assert (err <= B).all(), f"value off its fp64 score by {(err / B).max():.3g} B_u"

    # the returned set: its sorted fp64 scores match the oracle's top k to 2 B_u
    srt = -np.sort(-np.where(got, s, -np.inf), axis=1)
    with np.errstate(invalid="ignore"):
        gap = np.where(got, np.abs(srt - ov[:, :k]), 0.0)
    assert (gap <= 2 * B).all(), f"returned set off the oracle's top k by {(gap / B).max():.3g} B_u"

    # ranks: exact index wherever the oracle's score is isolated by more than 2 B_u (or by an identical row) on both sides
    oj = np.where(oi >= 0, oi, 0)
    same = np.all(V[oj[:, :-1]] == V[oj[:, 1:]], axis=2) & (bb[oj[:, :-1]] == bb[oj[:, 1:]])
    with np.errstate(invalid="ignore"):
        d_ov = ov[:, :-1] - ov[:, 1:]                       # k gaps of the k + 1 oracle scores; inf / nan next to padding
    sep = ~np.isfinite(d_ov) | (d_ov > 2 * B) | same
    ok = sep & np.concatenate([np.ones((n, 1), bool), sep[:, :-1]], axis=1)
    bad = ok & (idx != oi[:, :k])
    assert not bad.any(), f"{bad.sum()} isolated ranks differ from the oracle, first at {np.argwhere(bad)[0].tolist()}"
    return int((ok & got).sum()), int(got.sum())
