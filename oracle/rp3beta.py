"""numpy restatement of the reference's RP3beta (graph_based/RP3beta/rp3beta.py:73-176) that reproduces its float32
arithmetic bit for bit, with the tie rules of the device kernels:

  Pui         fp32(r / sum |r|) per user row, the sum in fp64 in stored order (sklearn's l1 `normalize`);
  Piu         fp32(1 / count_i) per item row of the binarised transpose, users ascending;
  degree      fp64(fp32 count_i ** -beta), 0 for items without ratings;
  alpha != 1  both raised to alpha in float32;
  similarity  row i = Piu[i] . Pui in float32, SciPy's order: acc[j] = fp32(acc[j] + fp32(a_e * b_ej)) over the left row's
              entries e in stored order; then fp64(row) * degree with the diagonal zeroed, and the k largest nonzero
              values by (value desc, column asc), kept as fp32;
  normalise   W rows l1-normalised like Pui, the sum in column order (SciPy's COO -> CSR sorts the columns);
  prune       per column the k largest nonzero values by (value desc, row asc);
  preds       R . W in float32, SciPy's order over R's stored entries;
  topk        oracle.knn.topk: train items -> -inf, (score desc, column asc).

Every float32 sum runs per left entry over that entry's right row; the columns of one right row are distinct, so each
entry is one vectorised update.  TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import hashlib

import numpy as np
import scipy.sparse as sp


def l1_rows(indptr, data):
    """fp32(v / sum |v|) per row, the sum accumulated in fp64 in stored order; rows that sum to 0 are left alone."""
    out = np.array(data, dtype=np.float32, copy=True)
    for r in range(len(indptr) - 1):
        seg = slice(indptr[r], indptr[r + 1])
        if indptr[r + 1] == indptr[r]:
            continue
        s = np.add.accumulate(np.abs(out[seg].astype(np.float64)))[-1]
        if s != 0.0:
            out[seg] = (out[seg].astype(np.float64) / s).astype(np.float32)
    return out


def prepare(R, alpha, beta):
    """(Pui, Piu, degree) of a float32 CSR R [users][items] (stored order kept): Pui, Piu float32 CSRs, degree fp64."""
    R = sp.csr_matrix(R, dtype=np.float32)
    n_items = R.shape[1]
    Pui = sp.csr_matrix((l1_rows(R.indptr, R.data), R.indices.copy(), R.indptr.copy()), shape=R.shape)
    Piu = sp.csr_matrix(R.T.astype(np.float32))
    Piu.sort_indices()
    count = np.diff(Piu.indptr)
    Piu.data = np.repeat((1.0 / np.maximum(count, 1)).astype(np.float32), count)
    degree = np.zeros(n_items)
    nz = count != 0
    degree[nz] = np.power(count[nz].astype(np.float32), -float(beta))
    if float(alpha) != 1.0:
        Pui.data = np.power(Pui.data, float(alpha))
        Piu.data = np.power(Piu.data, float(alpha))
    return Pui, Piu, degree


def ordered_row(A, r, B, n_cols):
    """Row r of the float32 product A . B in SciPy's order."""
    acc = np.zeros(n_cols, np.float32)
    for e in range(A.indptr[r], A.indptr[r + 1]):
        a = np.float32(A.data[e])
        seg = slice(B.indptr[A.indices[e]], B.indptr[A.indices[e] + 1])
        cols = B.indices[seg]
        acc[cols] = acc[cols] + a * B.data[seg]
    return acc


def top_nonzero(v, k):
    """Columns of the k largest nonzero values of v, (value desc, column asc), returned in column order."""
    nz = np.flatnonzero(v != 0)
    sel = nz[np.lexsort((nz, -v[nz]))][:k]
    return np.sort(sel)


def similarity_lists(Pui, Piu, degree, k, rows=None):
    """{i: (columns ascending, fp32 values)} of RP3beta's similarity lists before normalisation."""
    n = len(degree)
    out = {}
    for i in (range(n) if rows is None else rows):
        row = ordered_row(Piu, i, Pui, n).astype(np.float64) * degree
        row[i] = 0.0
        c = top_nonzero(row, min(k, n))
        out[int(i)] = (c, row[c].astype(np.float32))
    return out


def lists_to_csr(lists, n):
    indptr = np.zeros(n + 1, np.int64)
    for i, (c, _) in lists.items():
        indptr[i + 1] = len(c)
    indptr = np.cumsum(indptr)
    idx = np.concatenate([lists[i][0] for i in range(n)] or [np.zeros(0, np.int64)]).astype(np.int32)
    val = np.concatenate([lists[i][1] for i in range(n)] or [np.zeros(0, np.float32)]).astype(np.float32)
    return sp.csr_matrix((val, idx, indptr), shape=(n, n))


def prune_cols(W, k):
    """Per column of the float32 CSR W the k largest nonzero values, (value desc, row asc); a CSR with sorted columns."""
    C = sp.csc_matrix(W)
    C.sort_indices()
    rows, cols, vals = [], [], []
    for c in range(C.shape[1]):
        seg = slice(C.indptr[c], C.indptr[c + 1])
        r, v = C.indices[seg], C.data[seg]
        ok = v != 0
        r, v = r[ok], v[ok]
        o = np.lexsort((r, -v.astype(np.float64)))[:k]
        rows.append(r[o]); cols.append(np.full(len(o), c)); vals.append(v[o])
    rows, cols, vals = (np.concatenate(a) if a else np.zeros(0) for a in (rows, cols, vals))
    out = sp.csr_matrix((vals.astype(np.float32), (rows.astype(np.int64), cols.astype(np.int64))), shape=W.shape,
                        dtype=np.float32)
    out.sort_indices()
    return out


def weights(R, alpha, beta, k, normalize):
    """W (float32 CSR) and the similarity lists before normalisation."""
    Pui, Piu, degree = prepare(R, alpha, beta)
    n = len(degree)
    lists = similarity_lists(Pui, Piu, degree, k)
    S = lists_to_csr(lists, n)
    if normalize:
        S = sp.csr_matrix((l1_rows(S.indptr, S.data), S.indices, S.indptr), shape=S.shape)
    return prune_cols(S, k), lists


def preds(R, W, rows=None):
    """float32 R . W in SciPy's order (R's stored entry order), dense [len(rows)][n_items]."""
    R = sp.csr_matrix(R, dtype=np.float32) if not sp.issparse(R) else R
    users = range(R.shape[0]) if rows is None else rows
    return np.stack([ordered_row(R, u, W, W.shape[1]) for u in users]) if len(users) else np.zeros((0, W.shape[1]), np.float32)


# ---------------------------------------------------------------- comparisons with the reference's record
def reference_lists(s_row, s_col, s_val, n):
    """The reference's similarity lists (rp3beta.py:143's COO triples) as {i: (columns ascending, fp32 values)}."""
    out = {}
    for i in range(n):
        sel = np.flatnonzero(s_row == i)
        o = np.argsort(s_col[sel], kind="stable")
        out[i] = (s_col[sel][o].astype(np.int64), s_val[sel][o].astype(np.float32))
    return out


def row_lists_equal(mine, ref, k):
    """Kept values bit-equal as a multiset per row, and (column, value) pairs equal except at a full row's k-th value.
    Returns the number of entries that differ at such ties."""
    ties = 0
    for i, (rc, rv) in ref.items():
        mc, mv = mine[i]
        assert np.array_equal(np.sort(mv).view(np.int32), np.sort(rv).view(np.int32)), f"row {i}: kept values differ"
        a, b = dict(zip(mc.tolist(), mv.tolist())), dict(zip(rc.tolist(), rv.tolist()))
        for c in set(a) ^ set(b):
            v = a.get(c, b.get(c))
            assert len(rv) == k and v == rv.min(), f"row {i} column {c}: differs away from a tie at the k-th value"
            ties += 1
        for c in set(a) & set(b):
            assert np.float32(a[c]).view(np.int32) == np.float32(b[c]).view(np.int32), f"row {i} column {c}"
    return ties


def w_equal_but_ties(W, W_ref, lists, ref_lists, k):
    """W (CSR) equal to the reference's entry for entry and bit for bit, except entries at a tie: at a full similarity
    row's k-th value (in either's lists), at either W's smallest kept value of a full column, or anywhere in a column
    whose candidates differ through such a row tie.  Returns the number of differing entries."""
    A, B = sp.csc_matrix(W), sp.csc_matrix(W_ref)
    row_min = {i: (v.min() if len(v) == k else None) for i, (_, v) in ref_lists.items()}
    cand = lambda L, r: dict(zip(L[r][0].tolist(), L[r][1].tolist()))
    tied_cols = {c for r in ref_lists for c in set(cand(lists, r)) ^ set(cand(ref_lists, r))}
    ties = 0
    for c in range(A.shape[1]):
        sa, sb = slice(A.indptr[c], A.indptr[c + 1]), slice(B.indptr[c], B.indptr[c + 1])
        a, b = dict(zip(A.indices[sa].tolist(), A.data[sa].tolist())), dict(zip(B.indices[sb].tolist(), B.data[sb].tolist()))
        mins = [min(d.values()) for d in (a, b) if len(d) == k]
        for r in set(a) & set(b):
            assert np.float32(a[r]).view(np.int32) == np.float32(b[r]).view(np.int32), f"W[{r}, {c}]"
        for r in set(a) ^ set(b):
            v = a.get(r, b.get(r))
            ok = c in tied_cols or any(v == m for m in mins)
            assert ok, f"W[{r}, {c}] = {v}: differs away from a tie"
            ties += 1
    return ties


def preds_digest(P):
    """SHA-256 of a float32 preds matrix (dense, row-major): how tests/golden/rp3beta_cases.npz records the reference's
    preds, which are bit-identical to preds() of R and the recorded W."""
    return hashlib.sha256(np.ascontiguousarray(P, dtype=np.float32).tobytes()).hexdigest()


def check_case(g, name):
    """The oracle against one case of tests/golden/rp3beta_cases.npz (a dict of its arrays); asserts and returns counts."""
    from oracle.knn import isolated, topk
    R = g[f"{name}_R"].astype(np.float64)
    alpha, beta = float(g[f"{name}_alpha"]), float(g[f"{name}_beta"])
    norm, nbh = bool(g[f"{name}_normalize"]), int(g[f"{name}_neighborhood"])
    n, k, K = R.shape[1], (R.shape[1] if int(g[f"{name}_neighborhood"]) == -1 else nbh), int(g["topk"])
    Rs = sp.csr_matrix(R.astype(np.float32))
    W, lists = weights(Rs, alpha, beta, k, norm)
    ref_lists = reference_lists(g[f"{name}_s_row"], g[f"{name}_s_col"], g[f"{name}_s_val"], n)
    row_ties = row_lists_equal(lists, ref_lists, min(k, n))
    W_ref = sp.csc_matrix((g[f"{name}_w_data"], g[f"{name}_w_rows"], g[f"{name}_w_ptr"]), shape=(n, n)).tocsr()
    w_ties = w_equal_but_ties(W, W_ref, lists, ref_lists, k)
    P_ref = preds(Rs, W_ref)
    assert preds_digest(P_ref) == str(g[f"{name}_preds_sha256"]), "preds from the reference's W"
    if w_ties == 0:
        assert np.array_equal(preds(Rs, W).view(np.int32), P_ref.view(np.int32)), "preds from the oracle's W"
    _, ov = topk(P_ref.astype(np.float64), R != 0, K + 1)
    oi, _ = topk(P_ref.astype(np.float64), R != 0, K)
    iso = isolated(ov[:, :K], ov[:, K], rel=0.0)
    ri = g[f"{name}_topk_idx"]
    assert np.array_equal(oi[iso], ri[iso]), "top-k at isolated ranks"
    return {"row_ties": row_ties, "w_ties": w_ties, "w_nnz": W_ref.nnz, "isolated": float(iso.mean())}
