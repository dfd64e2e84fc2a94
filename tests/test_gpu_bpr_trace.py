"""Every BPR kernel audited triple by triple where users repeat (oracle/bpr_trace.py).  A triple whose items no other triple
touches is inverted in fp64 from the tables before and after the step: the user-row state it read and the update it
produced.  The user rows must then be explained by the kernel's schedule: inside a run kept in registers each triple reads
the row the previous one left, every segment starts from a state the memory model allows, and every update lands exactly
once (atomic) or the row ends as one segment left it (racy).  The data are few users with many items each over a large
catalogue, so that nearly every user's triples are all clean; the tests assert how much was actually checked."""
import numpy as np
import pytest
import torch

from elliot_b200 import ops
from oracle import bpr_trace as bt

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HP = (0.05, 0.0025, 0.01, 0.0025, 0.00025)
NI = 1 << 22                                   # item catalogue of the sampled cases: items drawn twice are rare
FIRST = 11


def _np(t):
    return t.detach().cpu().numpy()


def _user_tables(nu, d, ld, gen):
    U = torch.zeros((nu, ld), device=DEV); U[:, :d] = torch.randn(nu, d, device=DEV, generator=gen) * 0.1
    return U


def _item_tables(ni, d, ld, rows, gen):
    """Item rows are random where a triple touches them and on both neighbours of such a row, zero elsewhere (a table of
    millions of rows need not be filled); biases are random everywhere."""
    V = torch.zeros((ni, ld), device=DEV)
    nb = np.setdiff1d(np.clip(np.concatenate([rows - 1, rows + 1]), 0, ni - 1), rows)
    for r in (rows, nb):
        r = torch.from_numpy(r).to(DEV)
        V[r, :d] = torch.randn(len(r), d, device=DEV, generator=gen) * 0.1
    b = torch.randn(ni, device=DEV, generator=gen) * 0.05
    return V, b, nb


def _check_items_untouched(V, b0, b, rows, nb, V_nb, d):
    """Rows no triple touched are bit-identical to before; padding columns d..ld of the touched rows stay zero."""
    r = torch.from_numpy(rows).to(DEV)
    assert not V[r, d:].any(), "padding columns of item rows written"
    assert torch.equal(V[torch.from_numpy(nb).to(DEV)], V_nb), "an untouched item row next to a touched one changed"
    V[r] = 0
    V[torch.from_numpy(nb).to(DEV)] = 0
    assert not V.any(), "an untouched item row changed"
    keep = torch.ones(len(b), dtype=torch.bool, device=DEV); keep[r] = False
    assert torch.equal(b[keep], b0[keep]), "an untouched item bias changed"


def _audit(U0, U1, V0r, V1r, b0r, b1r, rows, tu, ti, tj, seg, d, atomic, min_clean=0.9, bias=True):
    """Reconstruct every clean triple (items compacted to `rows`) and audit every user whose triples are all
    reconstructed.  seg: the segment of each triple (the kernel walks a segment in ascending triple order)."""
    ci, cj = np.searchsorted(rows, ti), np.searchsorted(rows, tj)
    rec = bt.reconstruct(HP, U0[:, :d], V0r[:, :d], b0r if bias else None, U1[:, :d], V1r[:, :d], b1r if bias else None,
                         tu, ci, cj)
    ok = rec["ok"]
    for key in ("res_z", "res_un", "res_zx"):
        assert rec[key].max(initial=0) <= 1, (key, rec[key].max(), np.argmax(rec[key]))
    walk = np.lexsort((np.arange(len(tu)), seg))
    users = np.unique(tu)
    fails, stats = [], dict(users=len(users), clean_users=0, skipped=int(rec["skipped"].sum()), starts_checked=0,
                            starts_unchecked=0, chained=0, margin=np.inf)
    for u in users:
        idx = walk[tu[walk] == u]
        if not ok[idx].all():
            continue
        stats["clean_users"] += 1
        f, st = bt.check_user(rec, idx, seg[idx], U0[u, :d], U1[u, :d], atomic=atomic)
        fails += [f"user {u}: {m}" for m in f]
        for k in ("starts_checked", "starts_unchecked", "chained"):
            stats[k] += st[k]
        stats["margin"] = min(stats["margin"], st["margin"])
    assert not fails, fails[:10]
    assert stats["clean_users"] >= min_clean * len(users), stats
    assert stats["margin"] >= 100, stats
    return rec, stats


def _check_loss(rec, loss):
    if rec["ok"].all():
        want = bt.softplus_neg(rec["x"]).sum()
        assert abs(loss - want) <= 1e-5 * want, (loss, want)


# ---------------------------------------------------------------- the grouped sampled step
def _owner_csr(nu):
    """User u owns items [u P, (u + 1) P): half the catalogue in disjoint blocks, so positives collide only within a user
    (rarely: P is large) and negatives are drawn from a catalogue of millions."""
    P = NI // (2 * nu)
    indptr = torch.arange(nu + 1, dtype=torch.int64, device=DEV) * P
    idx = torch.arange(nu * P, dtype=torch.int32, device=DEV)
    return indptr, idx


def _clean_users(tu, ti, tj):
    cnt = np.bincount(np.concatenate([ti, tj]), minlength=NI)
    clean = (cnt[ti] == 1) & (cnt[tj] == 1)
    users = np.unique(tu)
    return np.mean([clean[tu == u].all() for u in users])


REGIMES = {                                    # mean run length per user and call, and users
    "short": lambda G: (max(1, G // 2), 64),   # runs shorter than a lane group's slice
    "2G": lambda G: (2 * G, max(4, 1024 // (2 * G))),
    "3 windows": lambda G: (96, 10),
    "n < 32": lambda G: (7, 3),
}


def _pick_seed(nu, ni, indptr, idx, n):
    """The first seed whose batch leaves at least 90% of the users with only clean triples."""
    for seed in range(1, 60):
        out = [_np(x) for x in ops.bpr_sample_philox(nu, ni, indptr, idx, n, seed, FIRST)]
        if _clean_users(*out) >= 0.9:
            return seed, out
    pytest.fail("no seed gives a mostly clean batch")


@pytest.mark.parametrize("d", [5, 16, 30, 64, 100, 256])
@pytest.mark.parametrize("regime", list(REGIMES))
def test_grouped_sampled_step_explained_triple_by_triple(regime, d):
    ld = ops.padded_dim(d)
    G = min(ld // 4, 32)
    L, nu = REGIMES[regime](G)
    n = nu * L + 7 if regime != "n < 32" else 20
    assert n % 32 != 0
    indptr, idx = _owner_csr(nu)
    seed, (tu, ti, tj) = _pick_seed(nu, NI, indptr, idx, n)
    order = np.argsort(tu, kind="stable")
    seg = np.empty(n, np.int64)
    seg[order] = bt.grouped_segments(tu[order], ld)
    # structural coverage: runs that leave a lane group's slice, and runs that leave a 32-entry window
    p = np.empty(n, np.int64); p[order] = np.arange(n)
    span = {u: (p[tu == u].min(), p[tu == u].max()) for u in np.unique(tu)}
    cross_slice = sum(lo // G != hi // G for lo, hi in span.values())
    cross_window = sum(lo // 32 != hi // 32 for lo, hi in span.values())
    if regime != "n < 32":
        assert cross_slice > 0 and cross_window > 0, (cross_slice, cross_window)
    rows = np.unique(np.concatenate([ti, tj]))

    for atomic in (True, False):
        gen = torch.Generator(device=DEV); gen.manual_seed(1000 * d + n)
        U = _user_tables(nu, d, ld, gen)
        V, b, nb = _item_tables(NI, d, ld, rows, gen)
        U0, b0 = U.clone(), b.clone()
        r = torch.from_numpy(rows).to(DEV)
        V0r, V_nb = _np(V[r]), V[torch.from_numpy(nb).to(DEV)].clone()
        out = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        ops.bpr_step_sampled_f32(U, V, b, d, nu, NI, indptr, idx, n, seed, FIRST, *HP, loss=loss, out=out, racy=not atomic)
        torch.cuda.synchronize()
        for a, c in zip(out, (tu, ti, tj)):
            assert np.array_equal(_np(a), c), "emitted triples differ from the sampler's"
        assert not U[:, d:].any(), "padding columns of user rows written"
        seen = np.zeros(nu, bool); seen[tu] = True
        assert torch.equal(U[torch.from_numpy(~seen).to(DEV)], U0[torch.from_numpy(~seen).to(DEV)])
        V1r, b0r, b1r = _np(V[r]), _np(b0[r]), _np(b[r])
        _check_items_untouched(V, b0, b, rows, nb, V_nb, d)
        rec, st = _audit(_np(U0), _np(U), V0r, V1r, b0r, b1r, rows, tu, ti, tj, seg, d, atomic)
        # at G <= 4 a 96-triple run spans more than 11 slices: no segment start fits the subset model's 2^10 cap there
        # (the chains and the sum of the updates still pin every row)
        assert st["starts_checked"] > 0 or (regime == "3 windows" and G <= 4), st
        assert L < 2 or st["chained"] > 0, st
        _check_loss(rec, loss.item())


# ---------------------------------------------------------------- per-triple kernels on materialised triples
def _materialised(nu, d, seed, max_run=10):
    """nu users with 1..max_run triples each, interleaved at random; every item in exactly one triple."""
    rs = np.random.RandomState(seed)
    runs = rs.randint(1, max_run + 1, nu)
    tu = rs.permutation(np.repeat(np.arange(nu), runs)).astype(np.int32)
    n = len(tu)
    items = rs.permutation(4 * n)[:2 * n].astype(np.int32)
    return tu, items[:n], items[n:], 4 * n


def _per_triple_case(d, step, nu=150, seed=0):
    ld = ops.padded_dim(d)
    tu, ti, tj, ni = _materialised(nu, d, seed + d)
    rows = np.unique(np.concatenate([ti, tj]))
    gen = torch.Generator(device=DEV); gen.manual_seed(d + seed)
    U = _user_tables(nu, d, ld, gen)
    V, b, nb = _item_tables(ni, d, ld, rows, gen)
    U0, b0, V0 = U.clone(), b.clone(), V.clone()
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    V, b = step(U, V, b, d, *(torch.from_numpy(x).to(DEV) for x in (tu, ti, tj)), loss)
    torch.cuda.synchronize()
    assert not U[:, d:].any()
    r = torch.from_numpy(rows).to(DEV)
    V_nb = V0[torch.from_numpy(nb).to(DEV)]
    V0r, V1r, b0r, b1r = _np(V0[r]), _np(V[r]), _np(b0[r]), _np(b[r])
    _check_items_untouched(V, b0, b, rows, nb, V_nb, d)
    rec, st = _audit(_np(U0), _np(U), V0r, V1r, b0r, b1r, rows, tu, ti, tj, np.arange(len(tu)), d, True, min_clean=1.0)
    assert st["starts_unchecked"] == 0 and st["starts_checked"] == len(tu), st
    _check_loss(rec, loss.item())


@pytest.mark.parametrize("d", [5, 64, 100, 256])
@pytest.mark.parametrize("deterministic", [False, True], ids=["hogwild", "rounds"])
def test_per_triple_step_explained_triple_by_triple(deterministic, d):
    """bpr_hogwild_kernel on materialised triples, free-running or in deterministic rounds: every triple is its own
    segment, reads U0 plus some subset of its user's other updates, and adds its update exactly once."""
    def step(U, V, b, d, tu, ti, tj, loss):
        ops.bpr_step_f32(U, V, b, d, tu, ti, tj, *HP, loss=loss, deterministic=deterministic)
        return V, b
    _per_triple_case(d, step)


def _split(full, n_shards):
    sr = -(-full.shape[0] // n_shards)
    shards = []
    for s in range(n_shards):
        t = torch.zeros((sr,) + tuple(full.shape[1:]), device=full.device, dtype=full.dtype)
        blk = full[s * sr:(s + 1) * sr]
        t[:blk.shape[0]] = blk
        shards.append(t)
    return shards, sr


@pytest.mark.parametrize("d", [30, 100])
@pytest.mark.parametrize("n_shards", [1, 3])
@pytest.mark.parametrize("variant", [0, 16], ids=["staged", "register"])
def test_peer_step_explained_triple_by_triple(variant, n_shards, d):
    """The peer-addressed kernels (item table split over shard allocations) on materialised triples."""
    def step(U, V, b, d, tu, ti, tj, loss):
        ni = V.shape[0]
        Vs, sr = _split(V, n_shards); bs, _ = _split(b, n_shards)
        ops.bpr_step_peer_f32(U, Vs, bs, sr, d, ni, tu, ti, tj, *HP, loss=loss, _variant=variant)
        return torch.cat(Vs)[:ni], torch.cat(bs)[:ni]
    _per_triple_case(d, step, seed=n_shards + variant)


@pytest.mark.parametrize("d", [30, 100])
@pytest.mark.parametrize("n_shards", [1, 3])
@pytest.mark.parametrize("variant", [0, 16], ids=["staged", "register"])
def test_sampled_peer_step_explained_triple_by_triple(variant, n_shards, d):
    ld = ops.padded_dim(d)
    nu, ni = 64, 1 << 20
    n = nu * 4 + 7
    P = ni // (2 * nu)
    indptr = torch.arange(nu + 1, dtype=torch.int64, device=DEV) * P
    idx = torch.arange(nu * P, dtype=torch.int32, device=DEV)
    for seed in range(1, 60):
        tu, ti, tj = (_np(x) for x in ops.bpr_sample_philox(nu, ni, indptr, idx, n, seed, FIRST))
        cnt = np.bincount(np.concatenate([ti, tj]), minlength=ni)
        if np.mean([((cnt[ti] == 1) & (cnt[tj] == 1))[tu == u].all() for u in np.unique(tu)]) >= 0.9:
            break
    rows = np.unique(np.concatenate([ti, tj]))
    gen = torch.Generator(device=DEV); gen.manual_seed(d + n_shards)
    U = _user_tables(nu, d, ld, gen)
    V, b, nb = _item_tables(ni, d, ld, rows, gen)
    U0, V0, b0 = U.clone(), V.clone(), b.clone()
    Vs, sr = _split(V, n_shards); bs, _ = _split(b, n_shards)
    out = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_step_sampled_peer_f32(U, Vs, bs, sr, d, nu, ni, indptr, idx, n, seed, FIRST, *HP, loss=loss, out=out,
                                  _variant=variant)
    torch.cuda.synchronize()
    for a, c in zip(out, (tu, ti, tj)):
        assert np.array_equal(_np(a), c), "emitted triples differ from the sampler's"
    V, b = torch.cat(Vs)[:ni], torch.cat(bs)[:ni]
    assert not U[:, d:].any()
    r = torch.from_numpy(rows).to(DEV)
    V1r, b1r = _np(V[r]), _np(b[r])
    _check_items_untouched(V, b0, b, rows, nb, V0[torch.from_numpy(nb).to(DEV)], d)
    rec, st = _audit(_np(U0), _np(U), _np(V0[r]), V1r, _np(b0[r]), b1r, rows, tu, ti, tj, np.arange(n), d, True)
    assert st["starts_checked"] > 0.9 * n, st
    _check_loss(rec, loss.item())


@pytest.mark.parametrize("d,bias_col", [(60, 60), (60, -1), (256, -1)])
def test_fetched_rows_step_explained_triple_by_triple(d, bias_col):
    """eb_bpr_step_rows_f32: item rows come from fetched buffers (the bias, if any, in column bias_col of the padded row)
    and every triple's item deltas are written out, so each triple is reconstructed without any cleanliness condition."""
    ld = ops.padded_dim(d)
    nu = 120
    tu, _, _, _ = _materialised(nu, d, d + bias_col)
    n = len(tu)
    gen = torch.Generator(device=DEV); gen.manual_seed(d)
    U = _user_tables(nu, d, ld, gen)
    R = torch.zeros((2 * n, ld), device=DEV); R[:, :d] = torch.randn(2 * n, d, device=DEV, generator=gen) * 0.1
    if bias_col >= 0:
        R[:, bias_col] = torch.randn(2 * n, device=DEV, generator=gen) * 0.05
    Ri, Rj = R[:n].contiguous(), R[n:].contiguous()
    U0 = U.clone()
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    dRi, dRj = ops.bpr_step_rows_f32(U, torch.from_numpy(tu).to(DEV), Ri, Rj, bias_col, *HP, loss=loss)
    torch.cuda.synchronize()
    assert not U[:, d:].any(), "padding (or bias) columns of user rows written"
    dR = torch.cat([dRi, dRj])
    pad = [c for c in range(d, ld) if c != bias_col]
    assert not dR[:, pad].any(), "deltas in padding columns"
    R1 = R + dR                                                   # the owner's fp32 scatter-add
    R0n, R1n = _np(R), _np(R1)
    rows = np.arange(2 * n)
    b0r = R0n[:, bias_col] if bias_col >= 0 else None
    b1r = R1n[:, bias_col] if bias_col >= 0 else None
    rec, st = _audit(_np(U0), _np(U), R0n, R1n, b0r, b1r, rows, tu, rows[:n], rows[n:], np.arange(n), d, True,
                     min_clean=1.0, bias=bias_col >= 0)
    assert st["starts_checked"] == n, st
    _check_loss(rec, loss.item())
