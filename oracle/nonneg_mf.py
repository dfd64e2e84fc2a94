"""fp64 restatement of the reference's NonNegMF (latent_factor_models/NonNegMF/non_negative_matrix_factorization_model.py),
bit-exact by construction, with its accumulators and biases starting from zero (the reference allocates them with
np.empty; see oracle/gen_golden_nonneg_mf.py):

  init     RandomState(seed): P = normal(size=(U, F)), then Q = normal(size=(I, F));
  epoch    over the ratings k of the dict-order CSR (users ascending, each user's items in dict order), with P, Q the
           tables at the start of the epoch:
             dot_k = (((0 + Q[i,0] P[u,0]) + Q[i,1] P[u,1]) + ...), every product and sum rounded on its own;
             est_k = ((mu + bu[u]) + bi[i]) + dot_k, err = r_k - est_k,
             bu[u] += lr (err - reg bu[u]), then bi[i] += lr (err - reg bi[i])   (a sequential chain over k);
           user_num[u] = sum_k Q[i] r_k, user_den[u] = sum_k Q[i] est_k in dict order, item_num[i] / item_den[i] the
           same with P[u] in ascending user order;
           den += (n reg) S, S *= num / den for both sides (n = the row's rating count), from the old P and Q;
  scores   P[u].Q[i] + bi[i] + bu[u] + mu (BLAS here, so only to a tolerance).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import numpy as np


def init_tables(seed, n_users, n_items, factors):
    """(P, Q) as the reference draws them."""
    rs = np.random.RandomState(seed)
    P = rs.normal(size=(n_users, factors))
    Q = rs.normal(size=(n_items, factors))
    return P, Q


def row_of(indptr):
    """The user of every rating of a CSR."""
    return np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))


def dots(P, Q, indptr, items):
    """dot_k for every rating k: vectorised over k, summed over f in order from +0.0."""
    users = row_of(indptr)
    d = np.zeros(len(items))
    for f in range(P.shape[1]):
        d = d + Q[items, f] * P[users, f]
    return d


def bias_chain(bu, bi, mu, indptr, items, ratings, d, lr, reg):
    """est_k for every rating, updating bu and bi in place: one Python step per rating, in order."""
    mu, lr, reg = float(mu), float(lr), float(reg)
    est = np.empty(len(items))
    for u in range(len(indptr) - 1):
        b = float(bu[u])
        for k in range(int(indptr[u]), int(indptr[u + 1])):
            i = int(items[k])
            e = ((mu + b) + float(bi[i])) + float(d[k])
            err = float(ratings[k]) - e
            b = b + lr * (err - reg * b)
            bi[i] = bi[i] + lr * (err - reg * bi[i])
            est[k] = e
        bu[u] = b
    return est


def row_update(S, T, rows, cols, n_rows, ratings, est, reg):
    """S * (num / den) with num = sum T[col] r, den = sum T[col] est + (n reg) S, each sum taken in the order of
    (rows, cols, ratings, est) by np.add.at."""
    num = np.zeros_like(S)
    den = np.zeros_like(S)
    for f in range(S.shape[1]):
        t = T[cols, f]
        np.add.at(num[:, f], rows, t * ratings)
        np.add.at(den[:, f], rows, t * est)
    den += (n_rows.astype(np.float64) * reg)[:, None] * S
    with np.errstate(divide="ignore", invalid="ignore"):
        return S * (num / den)


def epoch(P, Q, bu, bi, mu, indptr, items, ratings, lr, reg):
    """One train_step: returns (P, Q, dots, est); bu and bi are updated in place."""
    d = dots(P, Q, indptr, items)
    est = bias_chain(bu, bi, mu, indptr, items, ratings, d, lr, reg)
    users = row_of(indptr)
    # every item's sums run in k order, which is ascending user order
    P1 = row_update(P, Q, users, items, np.diff(indptr), ratings, est, reg)
    Q1 = row_update(Q, P, items, users, np.bincount(items, minlength=Q.shape[0]), ratings, est, reg)
    return P1, Q1, d, est


def scores(P, Q, bu, bi, mu):
    """predict() for every (user, item) pair, summed as the reference does after its BLAS dot."""
    return ((P @ Q.T + bi[None, :]) + bu[:, None]) + float(mu)
