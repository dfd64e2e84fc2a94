"""numpy restatement of the reference's SLIM (latent_factor_models/Slim/slim_model.py:44-113) with sklearn's
ElasticNet(positive=True, fit_intercept=False, selection='random', max_iter=100, tol=1e-4) on a float32 sparse X, i.e.
`sparse_enet_coordinate_descent` of sklearn/linear_model/_cd_fast.pyx:

  problem p   (one per item) y = X[:, p] taken first, then user row p of X zeroed (the reference indexes the CSR's
              indptr with the item id), item column p kept: item p also regresses on itself;
  l1, l2      fp32(alpha * l1_ratio * n_users), fp32(alpha * (1 - l1_ratio) * n_users), computed in fp64 first;
  norms       per column the fp32 sum of x^2 in CSC (user) order;
  coordinate  j = active[xorshift(state) % 2^31 % n_active]; tmp = sum_i R[i] * x_ij in fp32, users ascending, one
              rounding per product and per add; tmp += w_j * norm_j; w_j = 0 if tmp < 0 else
              fp32((fp64(|tmp|) - l1) / fp64(norm_j + l2)): Cython binds the fused `fmax` of `fabs(tmp) - alpha` (a
              double) to its double version, so the soft threshold and the division run in fp64 and round once; the
              residual R[i] += x_ij * (w_old - w_new) in fp32;
  epoch stop  w_max == 0 or d_w_max / w_max <= tol (fp32), or the last epoch: then the duality gap, stop when
              gap <= tol * (y . y); otherwise gap-safe screening rebuilds the active set.

The stream of the xorshift state is the same for every problem (the ElasticNet gets an int random_state, so every fit
starts from RandomState(seed).randint(0, 2**31 - 1)).  The BLAS reductions of the gap (R.R, R.y, w.w, sum |w|, y.y)
run in fp64 here and on the device; sklearn runs them as float32 BLAS calls.  XtA = X^T R - l2 * w is the ordered
fp32 loop of the reference.

All problems advance in lockstep: coordinate step f of an epoch runs for every problem with f < n_active, as one
vectorised update over padded columns.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import numpy as np
import scipy.sparse as sp

MAX_ITER, TOL = 100, 1e-4


def seed_state(seed):
    """The xorshift seed every fit starts from (sparse_enet_coordinate_descent: rng.randint(0, RAND_R_MAX))."""
    return int(np.random.RandomState(seed).randint(0, 2 ** 31 - 1))


def xorshift(s):
    """our_rand_r on a uint32 array in place; returns the draws (before the % n_active)."""
    s[s == 0] = 1
    s ^= s << np.uint32(13)
    s ^= s >> np.uint32(17)
    s ^= s << np.uint32(5)
    return s % np.uint32(2 ** 31)


def regs(alpha, l1_ratio, n_users):
    return np.float32(alpha * l1_ratio * n_users), np.float32(alpha * (1.0 - l1_ratio) * n_users)


class Padded:
    """X's columns padded to one length: index n_users (a residual slot that stays 0) and value 0 past the end."""

    def __init__(self, X):
        C = sp.csc_matrix(X, dtype=np.float32)
        C.sort_indices()
        self.n_users, self.n_items = C.shape
        lens = np.diff(C.indptr)
        L = max(int(lens.max()) if len(lens) else 0, 1)
        self.idx = np.full((self.n_items, L), self.n_users, np.int64)
        self.val = np.zeros((self.n_items, L), np.float32)
        pos = np.arange(C.nnz) - np.repeat(C.indptr[:-1], lens)
        col = np.repeat(np.arange(self.n_items), lens)
        self.idx[col, pos] = C.indices
        self.val[col, pos] = C.data
        self.C = C


def _seq(a, axis=-1):
    """Sequential fp32 sum along `axis` (add.accumulate rounds after every add, in order)."""
    return np.take(np.add.accumulate(a, axis=axis, dtype=np.float32), -1, axis=axis)


def _gap(pd, probs, w, R, y, l1, l2, tol_eff):
    """(gap as fp32, XtA, dual_norm_XtA) for the problems `probs` (rows of w / R / y)."""
    idx, val = pd.idx, pd.val
    v = np.where(idx[None] == probs[:, None, None], np.float32(0), val[None])                  # (P, n, L)
    rows = np.arange(len(probs))[:, None, None]
    xta = _seq(v * R[rows, idx[None]])                                                        # ordered fp32
    xta = (xta - l2 * w).astype(np.float32)
    dual = xta.max(1)
    w64, R64 = w.astype(np.float64), R[:, :-1].astype(np.float64)
    primal_r = (R64 * R64).sum(1) + float(l2) * (w64 * w64).sum(1)
    ry = (R64 * y.astype(np.float64)).sum(1)
    l1n = np.abs(w64).sum(1)
    a = float(l1)
    scale = np.where(dual > a, a / np.maximum(dual.astype(np.float64), 1e-300), 1.0)
    gap = 0.5 * primal_r + a * l1n - (-0.5 * scale ** 2 * primal_r + scale * ry)
    return gap.astype(np.float32), xta, dual


def _screen(xta, dual, norm, gap, l1, l2, excl):
    """Gap-safe screening (Eq. 11 of arXiv:1802.07481) as _cd_fast.pyx computes it: the test in fp64 of fp32 terms."""
    xj = (xta / np.maximum(np.float32(l1), dual)[:, None]).astype(np.float32)
    dj = ((1.0 - np.abs(xj.astype(np.float64))) / np.sqrt((norm + l2).astype(np.float64))).astype(np.float32)
    bound = np.sqrt(2.0 * gap.astype(np.float64)) / float(l1)
    return (dj.astype(np.float64) <= bound[:, None]) & ~excl


def fit(X, alpha, l1_ratio, seed, items=None, max_iter=MAX_ITER, tol=TOL):
    """Every item's ElasticNet as the reference fits it.  Returns (coef [len(items), n_items] fp32, n_iter int, gap
    fp32 as sklearn's dual_gap_ (the solver's gap / n_users))."""
    pd = Padded(X)
    U, n = pd.n_users, pd.n_items
    if n > U:
        raise ValueError(f"SLIM zeroes user row p for item p: it needs num_items <= num_users, got {n} > {U}")
    probs = np.arange(n) if items is None else np.asarray(items, np.int64)
    P = len(probs)
    l1, l2 = regs(alpha, l1_ratio, U)
    C = pd.C
    # y, and the residual (its last slot is the padding target and stays 0)
    y = np.zeros((P, U), np.float32)
    for q, p in enumerate(probs):
        y[q, C.indices[C.indptr[p]:C.indptr[p + 1]]] = C.data[C.indptr[p]:C.indptr[p + 1]]
    R = np.zeros((P, U + 1), np.float32)
    R[:, :U] = y
    v = np.where(pd.idx[None] == probs[:, None, None], np.float32(0), pd.val[None])
    norm = _seq(v * v)                                                                        # (P, n) fp32
    del v
    w = np.zeros((P, n), np.float32)
    y64 = y.astype(np.float64)
    tol_eff = np.float32(tol) * (y64 * y64).sum(1).astype(np.float32)
    n_iter = np.zeros(P, np.int64)
    gap = np.zeros(P, np.float32)
    excl = np.zeros((P, n), bool)
    alive = np.ones(P, bool)
    rows_all = np.arange(P)

    g, xta, dual = _gap(pd, probs, w, R, y, l1, l2, tol_eff)
    gap[:] = g
    alive &= ~(g <= tol_eff)
    # initial screening: zero-norm columns always go
    keep = _screen(xta, dual, norm, g, l1, l2, excl) & (norm != 0)
    excl = ~keep
    active = [np.flatnonzero(keep[q]) for q in range(P)]
    n_active = np.array([len(a) for a in active], np.int64)
    act = np.zeros((P, n), np.int64)
    for q in range(P):
        act[q, :n_active[q]] = active[q]
    state = np.full(P, seed_state_value(seed), np.uint32)

    for it in range(max_iter):
        if not alive.any():
            break
        w_max = np.zeros(P, np.float32)
        d_max = np.zeros(P, np.float32)
        steps = int(n_active[alive].max()) if alive.any() else 0
        for f in range(steps):
            m = alive & (f < n_active)
            q = rows_all[m]
            if len(q) == 0:
                break
            s = state[q]
            r = xorshift(s)
            state[q] = s
            j = act[q, (r % n_active[q].astype(np.uint32)).astype(np.int64)]
            nj = norm[q, j]
            ok = nj != 0
            q, j, nj = q[ok], j[ok], nj[ok]
            idx = pd.idx[j]                                                                   # (Q, L)
            xv = np.where(idx == probs[q, None], np.float32(0), pd.val[j])
            wj = w[q, j]
            tmp = _seq(R[q[:, None], idx] * xv)
            tmp = (tmp + wj * nj).astype(np.float32)
            num = np.maximum(np.abs(tmp).astype(np.float64) - float(l1), 0.0)
            sign = np.sign(tmp).astype(np.float32)
            wn = np.where(tmp < 0, np.float32(0), (sign.astype(np.float64) * num) / (nj + l2).astype(np.float64)).astype(np.float32)
            ch = wn != wj
            if ch.any():
                qc, d = q[ch], (wj - wn)[ch]
                ic = idx[ch]
                R[qc[:, None], ic] = (R[qc[:, None], ic] + xv[ch] * d[:, None]).astype(np.float32)
                R[:, U] = 0
            w[q, j] = wn
            d_max[q] = np.maximum(d_max[q], np.abs(wn - wj))
            w_max[q] = np.maximum(w_max[q], np.abs(wn))
        with np.errstate(divide="ignore", invalid="ignore"):
            check = alive & ((w_max == 0) | (d_max / w_max <= np.float32(tol)) | (it == max_iter - 1))
        n_iter[alive] = it + 1
        if check.any():
            q = rows_all[check]
            g, xta, dual = _gap(pd, probs[q], w[q], R[q], y[q], l1, l2, tol_eff[q])
            gap[q] = g
            stop = g <= tol_eff[q]
            alive[q[stop]] = False
            # screening for the problems that go on
            go = ~stop
            if go.any():
                qg = q[go]
                keep = _screen(xta[go], dual[go], norm[qg], g[go], l1, l2, excl[qg])
                for t, qq in enumerate(qg):
                    drop = ~keep[t] & ~excl[qq]
                    for jj in np.flatnonzero(drop & (w[qq] != 0)):
                        ii = pd.idx[jj]
                        xv = np.where(ii == probs[qq], np.float32(0), pd.val[jj])
                        R[qq, ii] = (R[qq, ii] + xv * w[qq, jj]).astype(np.float32)
                        R[qq, U] = 0
                        w[qq, jj] = 0
                    excl[qq] |= drop
                    a = np.flatnonzero(keep[t])
                    n_active[qq] = len(a)
                    act[qq, :len(a)] = a
    return w, n_iter, (gap / np.float32(U)).astype(np.float32)


def seed_state_value(seed):
    return seed_state(seed)


def select(coef, neighborhood):
    """W (float32 CSR, coefficient item x target item) by the reference's rule: per column p the local_topK =
    min(nnz - 1, neighborhood) largest nonzero coefficients, ties to the lowest index.  A column without nonzeros stays
    empty (argpartition(-1) of an empty array returns nothing)."""
    n = coef.shape[1]
    rows, cols, vals = [], [], []
    for p in range(coef.shape[0]):
        nz = np.flatnonzero(coef[p])
        k = min(len(nz) - 1, int(neighborhood))
        if k <= 0:
            continue
        order = np.lexsort((nz, -coef[p, nz].astype(np.float64)))[:k]
        rows.append(nz[order])
        cols.append(np.full(k, p))
        vals.append(coef[p, nz[order]])
    if not rows:
        return sp.csr_matrix((n, coef.shape[0]), dtype=np.float32)
    W = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, coef.shape[0]),
                      dtype=np.float32)
    W.sort_indices()
    return W


def preds(X, W):
    """sp_i_train_ratings . W as the reference computes it (SciPy float32 csr * csr), dense."""
    return (sp.csr_matrix(X, dtype=np.float32) @ W).toarray()


def golden_W(g, name):
    n = g[f"{name}_R"].shape[1]
    return sp.csr_matrix((g[f"{name}_w_data"], g[f"{name}_w_indices"], g[f"{name}_w_indptr"]), shape=(n, n))


def w_equal_except_ties(W, Wg, coef, rel=1e-5):
    """W == Wg as matrices, except at entries whose value lies within rel * max|coef_p| of column p's last kept value
    or of zero (where two selections may differ by a tie).  Returns the number of differing entries excused."""
    A, B = W.toarray(), Wg.toarray()
    diff = A != B
    excused = 0
    for p in np.flatnonzero(diff.any(0)):
        tol = rel * max(float(np.abs(coef[p]).max()), 1e-30)
        kept = B[:, p][B[:, p] != 0]
        edge = kept.min() if len(kept) else 0.0
        for i in np.flatnonzero(diff[:, p]):
            v = max(abs(A[i, p]), abs(B[i, p]))
            assert abs(v - edge) <= tol or v <= tol, (p, i, A[i, p], B[i, p], edge)
            excused += 1
    return excused


def check_case(g, name, coef=None, n_iter=None):
    """The checks of tests/test_oracle_slim.py for one golden case (coef / n_iter: this side's results, default: the
    oracle's).  Returns a short summary; raises AssertionError on a mismatch."""
    from oracle.knn import isolated, topk as knn_topk
    from oracle.rp3beta import preds_digest
    R = g[f"{name}_R"].astype(np.float32)
    if coef is None:
        coef, n_iter, _ = fit(R, float(g[f"{name}_alpha"]), float(g[f"{name}_l1_ratio"]), int(g["seed"]))
    cg, ig = g[f"{name}_coef"], g[f"{name}_n_iter"]
    scale = np.maximum(np.abs(cg).max(1), 1e-30)
    rel = (np.abs(coef - cg).max(1) / scale)
    assert rel.max() <= 1e-5, (name, float(rel.max()))
    bad_it = np.flatnonzero(np.asarray(n_iter) != ig)
    assert len(bad_it) == 0, (name, bad_it[:10], np.asarray(n_iter)[bad_it[:10]], ig[bad_it[:10]])
    Wg = golden_W(g, name)
    W = select(coef, int(g[f"{name}_neighborhood"]))
    excused = w_equal_except_ties(W, Wg, cg)
    P = preds(R, Wg)
    assert preds_digest(P) == str(g[f"{name}_preds_sha256"]), name
    k = int(g["topk"])
    ti, tv = knn_topk(P, R != 0, k + 1)
    ref = g[f"{name}_topk_idx"].astype(np.int64)
    iso = isolated(tv[:, :k], tv[:, k])
    assert (ti[:, :k][iso] == ref[iso]).all(), name
    return (f"coef bit-exact {int((coef == cg).all(1).sum())}/{len(cg)} (max rel {rel.max():.1e}), n_iter equal, "
            f"W entries excused {excused}, preds sha ok, isolated ranks {int(iso.sum())}/{iso.size}")
