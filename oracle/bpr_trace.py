"""Triple-by-triple audit of one fp32 BPR step from the tables before and after it.  TEST INFRASTRUCTURE ONLY.

For one triple (u, i, j) the update of ``elliot_b200/csrc/bpr_update.cuh`` is

    x  = a.(v_i - v_j) + b_i - b_j          a = the user row the triple saw
    z  = 1 / (1 + e^x)
    un = a + lr ((v_i - v_j) z - reg_u a)   (du = un - a)
    v_i += lr (un z - reg_pos v_i)          v_j += lr (-un z - reg_neg v_j)
    b_i += lr (z - reg_b b_i)               b_j += lr (-z - reg_b b_j)

A triple is *clean* when its items i and j are touched by no other triple of the call: their rows and biases then move
because of this triple alone, and the update can be inverted in fp64 (``reconstruct``): z twice (from b_i and from b_j),
un twice (from v_i and from v_j), then a, du and x.  That is the exact user-row state the kernel read and the exact update
it produced, whatever order the kernel applied the triples in, so the user rows can be audited against a model of the
schedule (``check_user``): within a segment (a stretch of one user's triples applied by one lane group that keeps the row
in registers) every triple reads the row the previous one left; between segments the row goes through memory.

Every tolerance is derived from the fp32 rounding of the quantities involved (half an ulp per rounding, a few roundings
per formula, times a safety factor), never from a fixed constant; ``check_user`` also reports the margin, i.e. how far a
single lost or doubled update lies outside the tolerance.
"""
import itertools

import numpy as np

U32 = 2.0 ** -24          # unit roundoff of fp32
SAFETY = 4.0              # every bound below is a few roundings; 4x covers the ones the bounds leave out


def hulp(x):
    """Half an fp32 ulp of |x| (fp64), elementwise: the rounding error of storing x in fp32."""
    return 0.5 * np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


def hyper32(hp):
    """The hyper-parameters as the kernels see them (fp32), as fp64 numbers."""
    return tuple(float(np.float32(v)) for v in hp)


def _z_from_rows(lr, reg_u, w, dv, z_min):
    """z of a triple without biases (x = a.dv): the root in (z_min, 1) of f(z) = z - 1 / (1 + e^x(z)), where
    a(z) = (w / z - lr z dv) / (1 - lr reg_u) follows from the item-row deltas (w = un z).  When x > 0, f is also positive
    near z = 0 and has a second, spurious root where f falls (z ln(1/z) ~ x z, so z < 1/e); the true root is the one where
    f rises.  NaN unless exactly one rising root lies in (z_min, 1)."""
    c = 1.0 - lr * reg_u
    wd, dd = float(w @ dv), float(dv @ dv)
    f = lambda z: z - 1.0 / (1.0 + np.exp((wd / z - lr * z * dd) / c))
    grid = np.linspace(z_min, 1.0 - 1e-9, 257)
    fg = np.array([f(z) for z in grid])
    sign = np.nonzero((fg[:-1] < 0) & (fg[1:] >= 0))[0]
    if len(sign) != 1:
        return np.nan, np.nan
    lo, hi = grid[sign[0]], grid[sign[0] + 1]
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        if np.sign(f(mid)) == np.sign(f(lo)): lo = mid
        else: hi = mid
    z = 0.5 * (lo + hi)
    eps = 1e-7
    return z, (f(z + eps) - f(z - eps)) / (2 * eps)


def reconstruct(hp, U0, V0, b0, U1, V1, b1, tu, ti, tj, z_min=0.05):
    """Invert the update of every clean triple.  U*, V*: the first d columns of the fp32 tables before (0) and after (1)
    the step; b0, b1: the item biases, or None for a kernel without biases (z is then solved from the item rows).

    Returns a dict of per-triple arrays (NaN where not ``ok``):
      clean     items i and j appear in no other triple (and i != j)
      skipped   clean, but z < z_min: the inversion divides by z and is not trusted there
      ok        clean and not skipped: a, un, du, z, x are set
      z, x      the triple's sigmoid argument and weight; a, un, du: [n, d]
      tol_z, tol_a, tol_un, tol_du, tol_x: the matching error bounds
      res_z     |z from b_i - z from b_j| / bound           (each must be <= 1)
      res_un    max_e |un from v_i - un from v_j| / bound
      res_zx    |z - 1 / (1 + e^x)| / bound: the reconstructed a reproduces the z the kernel used
    """
    lr, reg_u, reg_b, reg_pos, reg_neg = hyper32(hp)
    f = lambda t: np.asarray(t, np.float64)
    U0, V0, U1, V1 = f(U0), f(V0), f(U1), f(V1)
    tu, ti, tj = (np.asarray(t, np.int64) for t in (tu, ti, tj))
    n, d = len(tu), V0.shape[1]
    cnt = np.bincount(np.concatenate([ti, tj]), minlength=V0.shape[0])
    clean = (cnt[ti] == 1) & (cnt[tj] == 1) & (ti != tj)

    vi0, vj0 = V0[ti], V0[tj]
    dvi, dvj = V1[ti] - vi0, V1[tj] - vj0                     # exact: differences of fp32 values in fp64
    # w = un z, from each item row (half an ulp for storing v1, three roundings inside lr (un z - reg v))
    wi = dvi / lr + reg_pos * vi0
    wj = -(dvj / lr + reg_neg * vj0)
    tol_wi = SAFETY * (hulp(V1[ti]) / lr + U32 * (3 * np.abs(wi) + 3 * reg_pos * np.abs(vi0)))
    tol_wj = SAFETY * (hulp(V1[tj]) / lr + U32 * (3 * np.abs(wj) + 3 * reg_neg * np.abs(vj0)))
    dv = vi0 - vj0

    z = np.full(n, np.nan); tol_z = np.full(n, np.nan); res_z = np.zeros(n)
    if b0 is not None:
        b0, b1 = f(b0), f(b1)
        zi = (b1[ti] - b0[ti]) / lr + reg_b * b0[ti]
        zj = -((b1[tj] - b0[tj]) / lr + reg_b * b0[tj])
        tzi = SAFETY * (hulp(b1[ti]) / lr + U32 * (2 * np.abs(zi) + 3 * reg_b * np.abs(b0[ti])))
        tzj = SAFETY * (hulp(b1[tj]) / lr + U32 * (2 * np.abs(zj) + 3 * reg_b * np.abs(b0[tj])))
        z = 0.5 * (zi + zj)
        tol_z = 0.5 * (tzi + tzj)
        res_z = np.abs(zi - zj) / (tzi + tzj)
        bdiff = b0[ti] - b0[tj]
        tol_bdiff = SAFETY * U32 * (np.abs(b0[ti]) + np.abs(b0[tj]))
    else:
        bdiff = np.zeros(n); tol_bdiff = np.zeros(n)
        for k in np.nonzero(clean)[0]:
            w = 0.5 * (wi[k] + wj[k])
            zk, fp = _z_from_rows(lr, reg_u, w, dv[k], z_min)
            if not np.isfinite(zk):
                continue
            # how far z moves when w moves within its bound: dz = z (1 - z) dx / |f'(z)|, dx = |dv|.dw / (z (1 - lr reg_u))
            tw = 0.5 * (tol_wi[k] + tol_wj[k])
            dx = float(np.abs(dv[k]) @ tw) / (zk * (1 - lr * reg_u))
            z[k] = zk
            tol_z[k] = SAFETY * (zk * (1 - zk) * dx / max(abs(fp), 1e-3) + U32 * zk)

    skipped = clean & ~(z >= z_min)
    ok = clean & ~skipped
    zc = np.where(ok, z, np.nan)[:, None]
    tzc = np.where(ok, tol_z, np.nan)[:, None]
    uni, unj = wi / zc, wj / zc
    tui = tol_wi / zc + np.abs(uni) * tzc / zc
    tuj = tol_wj / zc + np.abs(unj) * tzc / zc
    un = 0.5 * (uni + unj)
    tol_un = 0.5 * (tui + tuj)
    res_un = np.nanmax(np.abs(uni - unj) / (tui + tuj), axis=1, initial=0.0)

    # un = fl(a + du), du = fl(lr fl(fl(fl(v_i - v_j) z) - fl(reg_u a)))  =>  a (1 - lr reg_u) = un - lr z dv + rounding
    c = 1.0 - lr * reg_u
    e_du = lr * U32 * (4 * np.abs(dv * zc) + 3 * reg_u * np.abs(un))
    a = (un - lr * zc * dv) / c
    tol_a = (tol_un + lr * np.abs(dv) * tzc + SAFETY * (e_du + hulp(un))) / c
    du = lr * (dv * zc - reg_u * a)
    tol_du = lr * np.abs(dv) * tzc + lr * reg_u * tol_a + SAFETY * e_du

    x = np.einsum("ij,ij->i", a, dv) + bdiff
    ad = np.einsum("ij,ij->i", np.abs(a), np.abs(dv))
    tol_x = np.einsum("ij,ij->i", tol_a, np.abs(dv)) + SAFETY * ((d + 8) * U32 * ad + U32 * np.abs(x)) + tol_bdiff
    zx = 1.0 / (1.0 + np.exp(x))
    tol_zx = tol_z + zx * (1 - zx) * tol_x + SAFETY * 4 * U32 * (1 + np.abs(x)) * zx    # __expf / __fdividef
    res_zx = np.where(ok, np.abs(zx - z) / tol_zx, 0.0) if b0 is not None else np.zeros(n)

    nan = lambda t: np.where(ok if t.ndim == 1 else ok[:, None], t, np.nan)
    return dict(clean=clean, skipped=skipped, ok=ok, z=nan(z), x=nan(x), a=nan(a), un=nan(un), du=nan(du),
                tol_z=nan(tol_z), tol_a=nan(tol_a), tol_un=nan(tol_un), tol_du=nan(tol_du), tol_x=nan(tol_x),
                res_z=np.where(ok, res_z, 0.0), res_un=np.where(ok, res_un, 0.0), res_zx=res_zx)


def softplus_neg(x):
    """softplus(-x) = -log sigmoid(x): the BPR loss of a triple with score difference x."""
    x = np.asarray(x, np.float64)
    return np.maximum(-x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def grouped_segments(tu_sorted, ld):
    """Segment id of every sorted position of the grouped sampled step (``bpr_grouped_kernel`` in bpr_train.cu).

    The kernel walks the triples sorted by user in windows of 32 positions, one per warp; the window's lane groups of
    G = min(ld / 4, 32) lanes each take a contiguous slice of G positions, so the slice of sorted position p is p // G.
    A group keeps the row of the user it is on in registers and writes it back when the user changes and at the end of
    its slice: a segment is a maximal run of one user inside one slice.  This mirrors the kernel's slicing and must
    change if the slicing does."""
    tu_sorted = np.asarray(tu_sorted)
    G = min(ld // 4, 32)
    p = np.arange(len(tu_sorted))
    new = np.ones(len(tu_sorted), bool)
    new[1:] = (tu_sorted[1:] != tu_sorted[:-1]) | (p[1:] // G != p[:-1] // G)
    return np.cumsum(new) - 1


def _chunks(d, width):
    return [np.arange(c, min(c + width, d)) for c in range(0, d, width)]


def check_user(rec, idx, seg, U0u, U1u, atomic=True, chunk=4, max_bits=10):
    """Audit one user's row against the schedule model.  rec: ``reconstruct`` output; idx: the user's triples in the
    order the kernel applies them (every one ``ok``); seg: their segment ids (equal ids are one segment, in order);
    U0u, U1u: the user's row (first d columns) before and after.  Per-triple kernels: every triple is its own segment.

    Within a segment each triple's a equals the previous triple's un.  Between segments the row goes through memory,
    checked per ``chunk`` columns (one float4 load or store):
      atomic (the segment adds its summed update):  every segment starts from U0 plus the updates of some subset of the
        user's other segments (enumerated when there are at most max_bits others, else that start is not checked), and
        U1 - U0 is the sum of every triple's du: each update lands exactly once;
      racy (the segment stores its row):  every segment starts from U0 or from another segment's end state, and U1
        equals one segment's end state.

    Returns (failures, stats): failures is a list of messages, empty when the row is explained; stats counts the
    checks made and gives ``margin``, the smallest |du| of the user's triples over the largest tolerance used (L2 norms):
    how far outside every bound one lost or doubled update lies."""
    idx = np.asarray(idx); seg = np.asarray(seg)
    assert rec["ok"][idx].all(), "check_user needs reconstructed triples"
    U0u = np.asarray(U0u, np.float64); U1u = np.asarray(U1u, np.float64)
    d = len(U0u)
    a, un, du = rec["a"][idx], rec["un"][idx], rec["du"][idx]
    ta, tun, tdu = rec["tol_a"][idx], rec["tol_un"][idx], rec["tol_du"][idx]
    M = np.max(np.abs(np.vstack([U0u, U1u, a, un])), axis=0)
    hU = SAFETY * hulp(M)                                        # one fp32 add into a row of this size
    segs = [np.nonzero(seg == s)[0] for s in dict.fromkeys(seg.tolist())]
    fails, tols = [], [np.zeros(d)]
    stats = dict(triples=len(idx), segments=len(segs), chained=0, starts_checked=0, starts_unchecked=0)

    for s, ks in enumerate(segs):
        for k0, k1 in zip(ks[:-1], ks[1:]):
            t = ta[k1] + tun[k0]; tols.append(t)
            stats["chained"] += 1
            if np.any(np.abs(a[k1] - un[k0]) > t):
                fails.append(f"segment {s}: triple {idx[k1]} did not read the row triple {idx[k0]} left "
                             f"(max |a - un_prev| / tol = {np.max(np.abs(a[k1] - un[k0]) / t):.3g})")

    first = np.array([ks[0] for ks in segs]); last = np.array([ks[-1] for ks in segs])
    if atomic:
        # a segment's summed update: its updates, each within its bound, plus one fp32 rounding per partial sum
        acc = np.array([du[ks].sum(0) for ks in segs])
        tacc = np.array([tdu[ks].sum(0) + SAFETY * hulp(np.cumsum(du[ks], axis=0)).sum(0) for ks in segs])
        for s in range(len(segs)):
            others = [q for q in range(len(segs)) if q != s]
            if len(others) > max_bits:
                stats["starts_unchecked"] += 1
                continue
            stats["starts_checked"] += 1
            B = np.array(list(itertools.product((0.0, 1.0), repeat=len(others))), np.float64).reshape(2 ** len(others), len(others))
            cand = U0u + B @ acc[others]
            tol = ta[first[s]] + B @ tacc[others] + (B.sum(1, keepdims=True) + 1) * hU
            bad = np.abs(a[first[s]] - cand) > tol
            for cols in _chunks(d, chunk):
                if not np.any(~bad[:, cols].any(1)):
                    fails.append(f"segment {s}: the row it started from (columns {cols[0]}..{cols[-1]}) is not U0 plus "
                                 f"the updates of any subset of the other {len(others)} segments")
                    break
            tols.append(np.min(tol, axis=0))
        t = tacc.sum(0) + (len(segs) + 1) * hU; tols.append(t)
        r = np.abs((U1u - U0u) - acc.sum(0))
        if np.any(r > t):
            fails.append(f"U1 - U0 is not the sum of the {len(idx)} updates (max |residual| / tol = {np.max(r / t):.3g})")
    else:
        ends, tend = un[last], tun[last]
        for s in range(len(segs)):
            stats["starts_checked"] += 1
            others = [q for q in range(len(segs)) if q != s]
            cand = np.vstack([U0u[None, :], ends[others]])
            tol = ta[first[s]] + np.vstack([np.zeros((1, d)), tend[others]])
            bad = np.abs(a[first[s]] - cand) > tol
            for cols in _chunks(d, chunk):
                if not np.any(~bad[:, cols].any(1)):
                    fails.append(f"segment {s}: the row it started from (columns {cols[0]}..{cols[-1]}) is neither U0 "
                                 f"nor another segment's end state")
                    break
            tols.append(np.max(tol, axis=0))
        bad = np.abs(U1u - ends) > tend
        for cols in _chunks(d, chunk):
            if not np.any(~bad[:, cols].any(1)):
                fails.append(f"U1 (columns {cols[0]}..{cols[-1]}) is no segment's end state")
                break
        tols.append(np.max(tend, axis=0))
    stats["margin"] = float(np.min(np.linalg.norm(du, axis=1)) / max(max(float(np.linalg.norm(t)) for t in tols), 1e-300))
    return fails, stats
