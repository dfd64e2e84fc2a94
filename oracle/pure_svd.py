"""fp64 numpy restatement of the device PureSVD (elliot_b200/recommender/pure_svd.py, csrc/pure_svd.cu).  TEST
INFRASTRUCTURE.

The same start block as sklearn's randomized_svd (RandomState(seed).normal, cast to float32), the same orientation and
iteration count, pivoted CholeskyQR2 as the normaliser (the device's pivot rule and rank tolerance), and the SVD of B
through the eigen-decomposition of B B^T (numpy's eigh here, Jacobi on the device), with the device's scaling and
svd_flip epilogue.  The reference's LU / QR normalisers span the same subspaces, so this agrees with the reference to
its float32 rounding."""
import numpy as np
import scipy.sparse as sp

EPS = 2.0 ** -52
OVERSAMPLES = 10


def chol_pivoted(G):
    """(M = P L^-T with zero columns past the rank, rank) for P^T G P = L L^T, pivoting on the largest remaining
    diagonal entry (ties: the lowest index), stopping at the first pivot <= w eps trace(G)."""
    w = G.shape[0]
    S = np.array(G, dtype=np.float64)
    tol = w * EPS * sum(S[i, i] for i in range(w))
    rem, piv = list(range(w)), []
    Lo = np.zeros((w, w))                                  # column k of L by original row index
    for k in range(w):
        diag = np.array([S[q, q] for q in rem])
        a = int(np.argmax(diag))
        if not diag[a] > tol:
            break
        p = rem.pop(a)
        piv.append(p)
        l = np.sqrt(S[p, p])
        col = np.array([S[q, p] / l for q in rem])
        for i, q in enumerate(rem):
            S[q, rem] -= col[i] * col
        Lo[p, k] = l
        Lo[rem, k] = col
    r = len(piv)
    M = np.zeros((w, w))
    if r:
        Linv = np.linalg.inv(np.tril(Lo[piv, :r]))
        M[np.array(piv), :r] = Linv.T
    return M, r


def orth(X):
    """Pivoted CholeskyQR2."""
    for _ in range(2):
        X = X @ chol_pivoted(X.T @ X)[0]
    return X


def fit(R, factors, seed=42):
    """(user_vec [U][d], item_vec [I][d], s [d]) of the device algorithm for the dense or sparse train matrix R."""
    A = sp.csr_matrix(R, dtype=np.float64)
    U, I = A.shape
    w = factors + OVERSAMPLES
    transpose = U < I
    M = A.T.tocsr() if transpose else A
    small = min(U, I)
    n_iter = 7 if factors < 0.1 * small else 4
    d = min(factors, small)
    Q = np.random.RandomState(seed).normal(size=(M.shape[1], w)).astype(np.float32).astype(np.float64)
    for _ in range(n_iter):
        Y = orth(M @ Q)
        Q = orth(M.T @ Y)
    Y = orth(M @ Q)
    Z = M.T @ Y
    G = Z.T @ Z
    lam, W = np.linalg.eigh(G)
    order = np.argsort(-lam, kind="stable")
    lam, W = lam[order], W[:, order]
    UM = Y @ W[:, :d]
    other = M.T @ UM
    s = np.sqrt(np.maximum(lam[:d], 0.0))
    if transpose:
        keep = lam[:d] > w * EPS * np.maximum(lam, 0.0).sum()
        user = other * np.where(keep, 1.0 / np.where(keep, s, 1.0), 0.0)
        item = UM * s
    else:
        user, item = UM, other
    rows = np.argmax(np.abs(user), axis=0)
    sign = np.where(user[rows, np.arange(d)] < 0, -1.0, 1.0)
    return user * sign, item * sign, s


def scores(user, item):
    return user @ item.T


def isolated_abs(v, v_next, tol):
    """Ranks of (n, k) top-k values whose value is more than 2 tol away from both neighbours (v_next: the (k+1)-th)."""
    w = np.concatenate([v, v_next[:, None]], 1)
    with np.errstate(invalid="ignore"):
        ok = np.abs(w[:, :-1] - w[:, 1:]) > 2 * tol
    iso = np.isfinite(v) & ok
    iso[:, 1:] &= ok[:, :-1]
    return iso


def clear_columns(s, user, rel=1e-3):
    """Columns whose singular value is well separated from its neighbours and from zero and whose user-side largest
    entry is unambiguous: their vectors, and signs, are determined."""
    d = len(s)
    ok = s > rel * s[0]
    gaps = np.abs(np.diff(s)) > rel * s[0]
    ok[:-1] &= gaps
    ok[1:] &= gaps
    a = np.sort(np.abs(user), axis=0)
    if user.shape[0] > 1:
        ok &= a[-2] < (1 - rel) * a[-1]
    return ok[:d]


def check_against(case, user, item, s, tol=1e-5):
    """Asserts (user, item, s) agree with a golden case: s within tol of the largest, scores within tol max |P|, the
    same orientation (positive inner product) of every clear user-side column, and the top-k lists at isolated ranks.  Returns (max |dP| / max |P|,
    isolated ranks checked)."""
    s_ref = case["s"]
    assert s.shape == s_ref.shape, (s.shape, s_ref.shape)
    assert np.abs(s - s_ref).max() <= tol * s_ref[0], np.abs(s - s_ref).max() / s_ref[0]
    P_ref = case["user_vec"].astype(np.float64) @ case["item_vec"].astype(np.float64).T
    P = scores(user, item)
    scale = np.abs(P_ref).max()
    err = np.abs(P - P_ref).max() / scale
    assert err <= tol, err
    ref_u = case["user_vec"].astype(np.float64)
    cc = clear_columns(s_ref, ref_u)
    assert np.all((user[:, cc] * ref_u[:, cc]).sum(0) > 0), "a determined user-side column has the other sign"
    k = case["topk_idx"].shape[1]
    mask = case["R"] != 0
    Pm = np.where(mask, -np.inf, P)
    order = np.argsort(-Pm, axis=1, kind="stable")[:, :k + 1]
    ov = np.take_along_axis(Pm, order, 1)
    iso = isolated_abs(ov[:, :k], ov[:, k], tol * scale)
    assert np.array_equal(order[:, :k][iso], case["topk_idx"][iso])
    return err, int(iso.sum())

