"""oracle/bpr_trace.py on emulated fp32 schedules (no GPU): the BPR update of bpr_update.cuh restated in float32 numpy, applied
to a user's triples in segments (stretches applied with the row kept in registers) that meet through memory in the ways
a free-running step allows.  The reconstruction must recover every triple's z, a and du from the tables alone, the
schedule audit must accept each legal schedule and reject one lost, doubled or misapplied update."""
import numpy as np
import pytest

from oracle import bpr_trace as bt

HP = (0.05, 0.0025, 0.01, 0.0025, 0.00025)
F = np.float32


def _update32(hp, a, vi, vj, bi, bj):
    """One triple's update in fp32, operation by operation as bpr_update.cuh does it (exact exp instead of __expf)."""
    lr, reg_u, reg_b, reg_pos, reg_neg = (F(v) for v in hp)
    dv = vi - vj
    x = F(np.dot(a, dv)) + (bi - bj)
    z = F(1) / (F(1) + np.exp(x))
    du = lr * (dv * z - reg_u * a)
    un = a + du
    di = lr * (un * z - reg_pos * vi)
    dj = lr * (-un * z - reg_neg * vj)
    return x, z, du, un, di, dj, lr * (z - reg_b * bi), lr * (-z - reg_b * bj)


# schedules of user 1's three segments of three triples (user 0 runs one segment of three first):
#   atomic: the segments whose summed update had landed when the segment read the row
#   racy:   the segment whose stored end state it read (None: U0), and the segment that wrote last
SCHEDULES = {
    "sequential": dict(n_seg=1, atomic=[[]], racy=[None], last=0),
    "two from U0": dict(n_seg=2, atomic=[[], []], racy=[None, None], last=1),
    "stale read": dict(n_seg=3, atomic=[[], [0], [1]], racy=[None, 0, None], last=2),
    "last writer wins": dict(n_seg=3, atomic=[[], [0], [0, 1]], racy=[None, 0, 1], last=1),
}
FAULTS = ["dropped update", "doubled update", "update on the wrong row state", "acc carried across users"]
PER_SEG = 3


def _problem(d, n_seg, seed):
    rs = np.random.RandomState(seed)
    n = PER_SEG * (1 + n_seg)
    U0 = (rs.normal(0, 0.1, (2, d))).astype(F)
    V0 = (rs.normal(0, 0.1, (2 * n + 7, d))).astype(F)
    b0 = (rs.normal(0, 0.05, 2 * n + 7)).astype(F)
    items = rs.permutation(2 * n + 7)[:2 * n]                      # every item in one triple: all triples clean
    tu = np.array([0] * PER_SEG + [1] * (PER_SEG * n_seg))
    return U0, V0, b0, tu, items[:n], items[n:]


def _run(hp, U0, V0, b0, tu, ti, tj, sched, atomic, fault=None, bias=True):
    """Apply the triples segment by segment (segment 0: user 0; 1..: user 1 as `sched` says); returns U1, V1, b1 and
    the true per-triple (a, du, z)."""
    segs = [list(range(s * PER_SEG, (s + 1) * PER_SEG)) for s in range(1 + sched["n_seg"])]
    starts = [[] if atomic else None] + [([q + 1 for q in st] if atomic else (None if st is None else st + 1))
                                        for st in sched["atomic" if atomic else "racy"]]
    V, b = V0.copy(), b0.copy()
    acc, end = {}, {}
    truth = {"a": np.zeros((len(tu), U0.shape[1])), "du": np.zeros((len(tu), U0.shape[1])), "z": np.zeros(len(tu))}
    for s, ks in enumerate(segs):
        u = tu[ks[0]]
        if atomic:
            cur = U0[u].copy()
            for q in starts[s]:
                cur = cur + acc[q]
        else:
            cur = U0[u].copy() if starts[s] is None else end[starts[s]].copy()
        sacc = np.zeros_like(cur)
        if fault == "acc carried across users" and s == 1:
            if atomic: sacc = acc[0].copy()
            else: cur = end[0].copy()
        for k in ks:
            i, j = ti[k], tj[k]
            x, z, du, un, di, dj, dbi, dbj = _update32(hp, cur, V[i], V[j], b[i] if bias else F(0), b[j] if bias else F(0))
            truth["a"][k], truth["du"][k], truth["z"][k] = cur, du, z
            V[i] = V[i] + di; V[j] = V[j] + dj
            if bias:
                b[i] = b[i] + dbi; b[j] = b[j] + dbj
            mid = s == len(segs) - 1 and k == ks[1]                # the fault hits user 1's last segment, middle triple
            if mid and fault == "dropped update":
                continue
            if mid and fault == "doubled update":
                cur = cur + du + du; sacc = sacc + du + du
            elif mid and fault == "update on the wrong row state":
                cur = U0[u] + du; sacc = sacc + du
            else:
                cur = un; sacc = sacc + du
        acc[s], end[s] = sacc, cur
    U1 = U0.copy()
    if atomic:
        for s, ks in enumerate(segs):
            U1[tu[ks[0]]] = U1[tu[ks[0]]] + acc[s]
    else:
        U1[0] = end[0]
        U1[1] = end[sched["last"] + 1]
    return U1, V, b, truth, segs


def _audit(rec, tu, segs, U0, U1, atomic):
    out = []
    for u in (0, 1):
        idx = [k for ks in segs for k in ks if tu[k] == u]
        seg = [s for s, ks in enumerate(segs) for k in ks if tu[k] == u]
        out.append(bt.check_user(rec, idx, seg, U0[u], U1[u], atomic=atomic))
    return out


@pytest.mark.parametrize("d", [5, 64])
@pytest.mark.parametrize("atomic", [True, False], ids=["atomic", "racy"])
@pytest.mark.parametrize("name", list(SCHEDULES))
def test_reconstruction_recovers_each_triple_and_the_audit_accepts_the_schedule(name, atomic, d):
    sched = SCHEDULES[name]
    U0, V0, b0, tu, ti, tj = _problem(d, sched["n_seg"], d + sched["n_seg"])
    U1, V1, b1, truth, segs = _run(HP, U0, V0, b0, tu, ti, tj, sched, atomic)
    rec = bt.reconstruct(HP, U0, V0, b0, U1, V1, b1, tu, ti, tj)
    assert rec["ok"].all()
    assert (rec["res_z"] <= 1).all() and (rec["res_un"] <= 1).all() and (rec["res_zx"] <= 1).all()
    assert (np.abs(rec["z"] - truth["z"]) <= rec["tol_z"]).all()
    assert (np.abs(rec["a"] - truth["a"]) <= rec["tol_a"]).all()
    assert (np.abs(rec["du"] - truth["du"]) <= rec["tol_du"]).all()
    # the bounds are not vacuous: about 1e-6 on rows of scale 0.1, where one update moves an entry by ~1e-3
    assert np.max(rec["tol_a"]) < 5e-6 and np.max(rec["tol_z"]) < 1e-6
    for fails, stats in _audit(rec, tu, segs, U0, U1, atomic):
        assert fails == [], fails
        assert stats["starts_unchecked"] == 0 and stats["margin"] >= 100, stats


@pytest.mark.parametrize("atomic", [True, False], ids=["atomic", "racy"])
@pytest.mark.parametrize("name", list(SCHEDULES))
@pytest.mark.parametrize("fault", FAULTS)
def test_the_audit_rejects_a_lost_doubled_or_misapplied_update(fault, name, atomic):
    sched = SCHEDULES[name]
    d = 16
    U0, V0, b0, tu, ti, tj = _problem(d, sched["n_seg"], 7)
    U1, V1, b1, _, segs = _run(HP, U0, V0, b0, tu, ti, tj, sched, atomic, fault=fault)
    rec = bt.reconstruct(HP, U0, V0, b0, U1, V1, b1, tu, ti, tj)
    assert rec["ok"].all()
    (f0, _), (f1, _) = _audit(rec, tu, segs, U0, U1, atomic)
    assert f0 == []
    assert f1, f"{fault} under '{name}' was accepted"


def test_reconstruction_without_biases_solves_z_from_the_item_rows():
    """Kernels whose item rows carry no bias (x = a.(v_i - v_j)): z is the unique root of the update's own equation."""
    sched = SCHEDULES["two from U0"]
    U0, V0, b0, tu, ti, tj = _problem(60, sched["n_seg"], 3)
    U1, V1, _, truth, segs = _run(HP, U0, V0, b0, tu, ti, tj, sched, True, bias=False)
    rec = bt.reconstruct(HP, U0, V0, None, U1, V1, None, tu, ti, tj)
    assert rec["ok"].all()
    assert (np.abs(rec["z"] - truth["z"]) <= rec["tol_z"]).all()
    assert (np.abs(rec["a"] - truth["a"]) <= rec["tol_a"]).all()
    for fails, stats in _audit(rec, tu, segs, U0, U1, True):
        assert fails == [] and stats["margin"] >= 100, (fails, stats)


def test_unclean_and_small_z_triples_are_left_out_and_counted():
    U0, V0, b0, tu, ti, tj = _problem(8, 2, 1)
    tj = tj.copy(); tj[4] = ti[0]                                  # item shared by triples 0 and 4
    b0 = b0.copy()
    b0[ti[2]], b0[tj[2]] = -40.0, 0.0                              # x ~ -40: z ~ 1, inverted as usual
    b0[ti[3]], b0[tj[3]] = 40.0, 0.0                               # x ~ 40: z ~ 0, not trusted
    U1, V1, b1, _, _ = _run(HP, U0, V0, b0, tu, ti, tj, SCHEDULES["two from U0"], True)
    rec = bt.reconstruct(HP, U0, V0, b0, U1, V1, b1, tu, ti, tj)
    assert not rec["clean"][0] and not rec["clean"][4]
    assert rec["ok"][2] and rec["skipped"][3]
    assert rec["ok"].sum() == len(tu) - 3 and np.isnan(rec["a"][3]).all()


def test_grouped_segments_follow_the_lane_group_slices():
    # ld 8 -> G = 2: positions 0-1, 2-3, ... are slices; ld 256 -> G = 32: one slice per window
    tu = np.array([0, 0, 0, 1, 1, 1, 1, 2])
    assert bt.grouped_segments(tu, 8).tolist() == [0, 0, 1, 2, 3, 3, 4, 5]
    assert bt.grouped_segments(tu, 16).tolist() == [0, 0, 0, 1, 2, 2, 2, 3]
    assert bt.grouped_segments(tu, 256).tolist() == [0, 0, 0, 1, 1, 1, 1, 2]
    tu = np.zeros(70, int)
    assert bt.grouped_segments(tu, 256).tolist() == [0] * 32 + [1] * 32 + [2] * 6
    assert bt.grouped_segments(tu, 512).tolist() == bt.grouped_segments(tu, 128).tolist()
