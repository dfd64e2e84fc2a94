"""GPU parity tests for the BPR training path, through the C ABI (elliot_b200.ops -> ctypes).

Checker: oracle/ (CPU restatement pinned to the reference) and tests/golden/*.npz (minted from
the reference's own code).  Tolerances are stated per test.
"""
import numpy as np
import pytest
import torch

import oracle
from elliot_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _csr_dev(g):
    indptr = torch.from_numpy(g["ui_indptr"].astype(np.int64)).to(DEV)
    set_idx = torch.from_numpy(g["ui_indices"].astype(np.int32)).to(DEV)
    srt = g["ui_indices"].astype(np.int32).copy()
    ip = g["ui_indptr"]
    for u in range(len(ip) - 1):
        srt[ip[u]:ip[u + 1]].sort()
    return indptr, set_idx, torch.from_numpy(srt).to(DEV)


def _pad(a, ld, dtype):
    out = np.zeros((a.shape[0], ld), dtype=dtype)
    out[:, :a.shape[1]] = a
    return torch.from_numpy(out).to(DEV)


def test_device_is_hopper():
    sm, cc = ops.device_info()
    assert cc == 90 and sm >= 100


def test_mt19937_raw_bit_exact(golden_tiny):
    indptr, set_idx, srt = _csr_dev(golden_tiny)
    s = ops.MtSampler(len(golden_tiny["users"]), len(golden_tiny["items"]), indptr, set_idx, srt, seed=42)
    a = s.raw(1000).cpu().numpy().view(np.uint32)
    b = s.raw(3001).cpu().numpy().view(np.uint32)   # crosses several 624-word regenerations
    want = oracle.Rng(42).raw(4001)
    assert np.array_equal(np.concatenate([a, b]), want)


def test_mt_sampler_replays_reference_stream(golden):
    """Bit-exact (u,i,j) for two consecutive epochs and the stream position after them."""
    g = golden
    indptr, set_idx, srt = _csr_dev(g)
    s = ops.MtSampler(len(g["users"]), len(g["items"]), indptr, set_idx, srt, seed=42)
    T, E = int(g["transactions"]), int(g["epochs"])
    us, is_, js = [], [], []
    for _ in range(E):
        u, i, j = s.step(T)
        us.append(u.cpu().numpy()); is_.append(i.cpu().numpy()); js.append(j.cpu().numpy())
    assert np.array_equal(np.concatenate(us), g["tu"])
    assert np.array_equal(np.concatenate(is_), g["ti"])
    assert np.array_equal(np.concatenate(js), g["tj"])
    tail = s.raw(4).cpu().numpy().view(np.uint32) & ((1 << 20) - 1)   # randint(1<<20) consumes exactly one draw
    assert list(tail) == list(g["tail"])


def test_mt_sampler_odd_event_counts(golden_small):
    """Ragged chunking: the same stream cut into uneven calls gives the same triples."""
    g = golden_small
    indptr, set_idx, srt = _csr_dev(g)
    s = ops.MtSampler(len(g["users"]), len(g["items"]), indptr, set_idx, srt, seed=42)
    got = []
    for n in [1, 2, 31, 513, 1000, 4099]:
        u, i, j = s.step(n)
        got.append(np.stack([u.cpu().numpy(), i.cpu().numpy(), j.cpu().numpy()]))
    got = np.concatenate(got, axis=1)
    n = got.shape[1]
    assert np.array_equal(got[0], g["tu"][:n]) and np.array_equal(got[1], g["ti"][:n]) and np.array_equal(got[2], g["tj"][:n])


def test_exact_f64_matches_sequential_reference(golden):
    """Exact mode == the reference's strictly sequential fp64 SGD.  Tolerance 1e-12 abs on every
    table entry (differences: reduction order of the two 1xd dots and 1-ulp exp)."""
    g = golden
    d = int(g["d"])
    U = torch.from_numpy(g["U0"].copy()).to(DEV); V = torch.from_numpy(g["V0"].copy()).to(DEV)
    b = torch.zeros(len(g["items"]), dtype=torch.float64, device=DEV)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    T = int(g["transactions"])
    tu = torch.from_numpy(g["tu"]).to(DEV); ti = torch.from_numpy(g["ti"]).to(DEV); tj = torch.from_numpy(g["tj"]).to(DEV)
    hp = [float(x) for x in g["hp"]]
    ops.bpr_exact_f64(U, V, b, d, tu[:T].contiguous(), ti[:T].contiguous(), tj[:T].contiguous(), *hp, loss=loss)
    torch.cuda.synchronize()
    assert np.abs(U.cpu().numpy() - g["U_ep1"]).max() < 1e-12
    assert np.abs(V.cpu().numpy() - g["V_ep1"]).max() < 1e-12
    assert np.abs(b.cpu().numpy() - g["b_ep1"]).max() < 1e-12
    ops.bpr_exact_f64(U, V, b, d, tu[T:].contiguous(), ti[T:].contiguous(), tj[T:].contiguous(), *hp, loss=loss)
    torch.cuda.synchronize()
    assert np.abs(U.cpu().numpy() - g["U"]).max() < 1e-12
    assert np.abs(V.cpu().numpy() - g["V"]).max() < 1e-12
    assert np.abs(b.cpu().numpy() - g["b"]).max() < 1e-12
    assert np.isfinite(loss.item()) and loss.item() > 0


def test_exact_f64_heavy_conflicts():
    """Every triple hits the same user and two hot items: the schedule degenerates to a chain."""
    rs = np.random.RandomState(0)
    nu, ni, d, n = 4, 6, 33, 3000
    U0 = rs.normal(0, 0.1, (nu, d)); V0 = rs.normal(0, 0.1, (ni, d))
    tu = rs.randint(0, 2, n).astype(np.int32); ti = rs.randint(0, 3, n).astype(np.int32)
    tj = (3 + rs.randint(0, 3, n)).astype(np.int32)
    U, V, b = U0.copy(), V0.copy(), np.zeros(ni)
    oracle.bpr_update_seq(U, V, b, tu, ti, tj, 0.05, 0.0025, 0.01, 0.0025, 0.00025)
    Ud = torch.from_numpy(U0.copy()).to(DEV); Vd = torch.from_numpy(V0.copy()).to(DEV)
    bd = torch.zeros(ni, dtype=torch.float64, device=DEV)
    ops.bpr_exact_f64(Ud, Vd, bd, d, torch.from_numpy(tu).to(DEV), torch.from_numpy(ti).to(DEV),
                      torch.from_numpy(tj).to(DEV), 0.05, 0.0025, 0.01, 0.0025, 0.00025)
    torch.cuda.synchronize()
    assert np.abs(Ud.cpu().numpy() - U).max() < 1e-11 and np.abs(Vd.cpu().numpy() - V).max() < 1e-11
    assert np.abs(bd.cpu().numpy() - b).max() < 1e-11


def _conflict_free(tu, ti, tj):
    seen_u, seen_i, keep = set(), set(), []
    for t in range(len(tu)):
        if tu[t] in seen_u or ti[t] in seen_i or tj[t] in seen_i:
            continue
        seen_u.add(tu[t]); seen_i.add(ti[t]); seen_i.add(tj[t]); keep.append(t)
    return np.array(keep)


@pytest.mark.parametrize("racy", [False, True])
def test_hogwild_f32_conflict_free_batch_equals_sequential(golden, racy):
    """Without row conflicts Hogwild == sequential.  fp32 vs the fp64 oracle: 2e-6 abs."""
    g = golden
    d = int(g["d"]); ld = ops.padded_dim(d)
    keep = _conflict_free(g["tu"], g["ti"], g["tj"])
    tu, ti, tj = g["tu"][keep], g["ti"][keep], g["tj"][keep]
    assert len(keep) >= 8
    U, V, b = g["U0"].copy(), g["V0"].copy(), np.zeros(len(g["items"]))
    hp = [float(x) for x in g["hp"]]
    hp[2] = 0.01  # exercise the bias regulariser too
    l0 = oracle.bpr_loss(U, V, b, tu, ti, tj)
    oracle.bpr_update_seq(U, V, b, tu, ti, tj, *hp)
    Ud, Vd = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32)
    bd = torch.zeros(len(g["items"]), dtype=torch.float32, device=DEV)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_step_f32(Ud, Vd, bd, d, torch.from_numpy(tu).to(DEV), torch.from_numpy(ti).to(DEV),
                     torch.from_numpy(tj).to(DEV), *hp, loss=loss, racy=racy)
    torch.cuda.synchronize()
    Uh, Vh = Ud.cpu().numpy(), Vd.cpu().numpy()
    assert np.abs(Uh[:, :d] - U).max() < 2e-6 and np.abs(Vh[:, :d] - V).max() < 2e-6
    assert np.abs(bd.cpu().numpy() - b).max() < 2e-6
    assert not Uh[:, d:].any() and not Vh[:, d:].any()          # padding columns stay zero
    assert abs(loss.item() - l0) < 1e-3 * max(1.0, l0)


@pytest.mark.parametrize("d", [5, 16, 30, 64, 100, 256])
def test_hogwild_variants_agree_bitwise_on_conflict_free_batch(golden_small, d):
    """Without row conflicts every triple's update is formed from the initial rows, so the kernel variants must leave
    bit-identical tables: register + atomics (default), deterministic rounds, packed host triples, and on the strides the
    sharded item table supports the peer step (shared-memory-staged on 1 and 3 shards, register on 3).  Racy stores differ
    from the atomic result in the last bit.  The loss is summed per lane group in a kernel-dependent order: 1e-6 relative."""
    from elliot_b200.parallel import ceil_shard
    g = golden_small
    rs = np.random.RandomState(d)
    nu, ni = len(g["users"]), len(g["items"])
    ld = ops.padded_dim(d)
    hp = (0.05, 0.0025, 0.01, 0.0025, 0.00025)
    keep = _conflict_free(g["tu"], g["ti"], g["tj"])
    tu, ti, tj = (torch.from_numpy(g[k][keep].astype(np.int32)) for k in ("tu", "ti", "tj"))
    U0 = _pad(rs.normal(0, 0.1, (nu, d)), ld, np.float32); V0 = _pad(rs.normal(0, 0.1, (ni, d)), ld, np.float32)
    b0 = torch.from_numpy(rs.normal(0, 0.05, ni).astype(np.float32)).to(DEV)
    dev_t = [x.to(DEV) for x in (tu, ti, tj)]

    def local(**kw):
        U, V, b = U0.clone(), V0.clone(), b0.clone()
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        ops.bpr_step_f32(U, V, b, d, *dev_t, *hp, loss=loss, **kw)
        return U, V, b, loss.item()

    def packed():
        U, V, b = U0.clone(), V0.clone(), b0.clone()
        host = ops.pack_triples(tu, ti, tj, nu, ni).pin_memory()
        staging = torch.empty(host.numel(), dtype=torch.int64, device=DEV)
        ld_, lh = torch.zeros(1, dtype=torch.float64, device=DEV), torch.zeros(1, dtype=torch.float64).pin_memory()
        ops.bpr_step_host_packed_f32(U, V, b, d, host, nu, ni, *hp, staging, ld_, lh)
        return U, V, b, lh.item()

    def peer(n_shards, variant=0):
        sr = ceil_shard(ni, n_shards)
        Vs = [torch.zeros((sr, ld), device=DEV) for _ in range(n_shards)]
        bs = [torch.zeros(sr, device=DEV) for _ in range(n_shards)]
        for s in range(n_shards):
            blk = slice(s * sr, min((s + 1) * sr, ni))
            Vs[s][:blk.stop - blk.start] = V0[blk]; bs[s][:blk.stop - blk.start] = b0[blk]
        U = U0.clone()
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        ops.bpr_step_peer_f32(U, Vs, bs, sr, d, ni, *dev_t, *hp, loss=loss, _variant=variant)
        return U, torch.cat(Vs)[:ni], torch.cat(bs)[:ni], loss.item()

    runs = {"racy": local(racy=True), "deterministic": local(deterministic=True), "packed": packed()}
    if ld in (32, 64, 128):
        runs.update({"peer1": peer(1), "peer3": peer(3), "peer3_register": peer(3, 16)})
    ref = local()
    torch.cuda.synchronize()
    assert not torch.equal(ref[0], U0) and ref[3] > 0
    for name, got in runs.items():
        for k, (a, c) in enumerate(zip(got[:3], ref[:3])):
            if name == "racy":
                # a plain store rounds once (row + lr * g contracts to one FMA), an atomic add rounds the delta and then the
                # sum: the last bit of the larger entries differs, 2^-25 at most on these inputs
                ok = (a - c).abs().max().item() <= 2.0 ** -25
            else:
                ok = torch.equal(a, c)
            assert ok, (name, "UVb"[k], (a - c).abs().max().item())
        assert abs(got[3] - ref[3]) <= 1e-6 * ref[3], (name, got[3], ref[3])


def test_hogwild_f32_epoch_tracks_sequential(golden_small):
    """A full epoch in one Hogwild launch (heavy staleness) stays close to sequential SGD:
    loss on the epoch's triples drops and the tables correlate > 0.98 with the oracle's."""
    g = golden_small
    d = int(g["d"]); ld = ops.padded_dim(d)
    T = int(g["transactions"])
    tu, ti, tj = g["tu"][:T], g["ti"][:T], g["tj"][:T]
    hp = [float(x) for x in g["hp"]]
    Ud, Vd = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32)
    bd = torch.zeros(len(g["items"]), dtype=torch.float32, device=DEV)
    dt = [torch.from_numpy(x).to(DEV) for x in (tu, ti, tj)]
    # four quarter-epoch launches
    q = T // 4
    for s in range(4):
        sl = slice(s * q, T if s == 3 else (s + 1) * q)
        ops.bpr_step_f32(Ud, Vd, bd, d, dt[0][sl].contiguous(), dt[1][sl].contiguous(), dt[2][sl].contiguous(), *hp)
    torch.cuda.synchronize()
    U, V, b = g["U0"].copy(), g["V0"].copy(), np.zeros(len(g["items"]))
    l0 = oracle.bpr_loss(U, V, b, tu, ti, tj)
    Uh = Ud.cpu().numpy()[:, :d].astype(np.float64); Vh = Vd.cpu().numpy()[:, :d].astype(np.float64)
    l1 = oracle.bpr_loss(Uh, Vh, bd.cpu().numpy().astype(np.float64), tu, ti, tj)
    assert l1 < l0
    cu = np.corrcoef(Uh.ravel(), g["U_ep1"].ravel())[0, 1]; cv = np.corrcoef(Vh.ravel(), g["V_ep1"].ravel())[0, 1]
    assert cu > 0.98 and cv > 0.98, (cu, cv)


def test_philox_sampler_invariants(golden_small):
    g = golden_small
    nu, ni = len(g["users"]), len(g["items"])
    indptr, _, srt = _csr_dev(g)
    n = 200000
    u, i, j = ops.bpr_sample_philox(nu, ni, indptr, srt, n, seed=1234)
    u2, i2, j2 = ops.bpr_sample_philox(nu, ni, indptr, srt, n, seed=1234)
    assert torch.equal(u, u2) and torch.equal(i, i2) and torch.equal(j, j2)      # deterministic
    u3, _, _ = ops.bpr_sample_philox(nu, ni, indptr, srt, n, seed=1235)
    assert not torch.equal(u, u3)
    u, i, j = u.cpu().numpy(), i.cpu().numpy(), j.cpu().numpy()
    assert u.min() >= 0 and u.max() < nu and j.min() >= 0 and j.max() < ni
    rows = [set(g["ui_indices"][g["ui_indptr"][x]:g["ui_indptr"][x + 1]].tolist()) for x in range(nu)]
    for t in range(0, n, 37):
        assert i[t] in rows[u[t]] and j[t] not in rows[u[t]]
    # u uniform over users (custom_sampler.py:32): chi-square, dof = nu-1, 6-sigma bound
    cnt = np.bincount(u, minlength=nu); chi = ((cnt - n / nu) ** 2 / (n / nu)).sum()
    assert abs(chi - (nu - 1)) < 6 * np.sqrt(2 * (nu - 1))
    # i uniform over the user's items (custom_sampler.py:37): heavy user 2
    sel = i[u == 2]; r2 = sorted(rows[2])
    c2 = np.array([(sel == x).sum() for x in r2]); e2 = len(sel) / len(r2)
    chi2 = ((c2 - e2) ** 2 / e2).sum()
    assert abs(chi2 - (len(r2) - 1)) < 6 * np.sqrt(2 * (len(r2) - 1))


@pytest.mark.parametrize("words", [1, 8, 32])
def test_membership_signatures_do_not_change_the_samples(golden_small, words):
    """The Bloom signatures only prove misses: with them the sampler emits exactly the unfiltered sampler's triples."""
    g = golden_small
    nu, ni = len(g["users"]), len(g["items"])
    indptr, _, srt = _csr_dev(g)
    filt = ops.bloom_build(indptr, srt, nu, words)
    # every train item sets both of its bits (host recomputation of the two hash positions)
    f = filt.cpu().numpy().view(np.uint32)
    lb = 5 + int(np.log2(words))
    for u in (0, 2, nu - 1):
        for x in g["ui_indices"][g["ui_indptr"][u]:g["ui_indptr"][u + 1]].astype(np.uint32):
            a = (int(x) * 0x9E3779B1 & 0xFFFFFFFF) >> (32 - lb)
            bb = ((int(x) ^ 0x5bd1e995) * 0x85EBCA6B & 0xFFFFFFFF) >> (32 - lb)
            assert (f[u, a >> 5] >> (a & 31)) & 1 and (f[u, bb >> 5] >> (bb & 31)) & 1
    n = 100000
    a = ops.bpr_sample_philox(nu, ni, indptr, srt, n, seed=77, first=5)
    b = ops.bpr_sample_philox(nu, ni, indptr, srt, n, seed=77, first=5, filter=filt)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    d = int(g["d"]); ld = ops.padded_dim(d)
    hp = [float(x) for x in g["hp"]]
    out = [torch.empty(4096, dtype=torch.int32, device=DEV) for _ in range(3)]
    Ud, Vd = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32)
    ops.bpr_step_sampled_f32(Ud, Vd, torch.zeros(ni, device=DEV), d, nu, ni, indptr, srt, 4096, 77, 5, *hp, out=out, filter=filt)
    for x, y in zip(out, a):
        assert torch.equal(x, y[:4096])


def test_sampler_near_dense_and_full_users():
    """A user owning all but 3 items still gets a uniform negative from exactly those 3 (rank draw after the rejection
    cap, ADVICE r1); a user owning EVERY item is never sampled (the reference would loop forever on it)."""
    ni = 64
    rows = [list(range(ni)), [x for x in range(ni) if x not in (5, 17, 40)], [1, 2, 3]]
    indptr = torch.tensor(np.cumsum([0] + [len(r) for r in rows]), dtype=torch.int64, device=DEV)
    idx = torch.tensor([x for r in rows for x in r], dtype=torch.int32, device=DEV)
    u, i, j = (t.cpu().numpy() for t in ops.bpr_sample_philox(3, ni, indptr, idx, 60000, seed=3))
    assert set(np.unique(u)) == {1, 2}
    ju = j[u == 1]
    assert set(np.unique(ju)) == {5, 17, 40}
    cnt = np.array([(ju == x).sum() for x in (5, 17, 40)])
    assert np.all(np.abs(cnt - len(ju) / 3) < 6 * np.sqrt(len(ju) * 2 / 9))
    assert not np.isin(j[u == 2], [1, 2, 3]).any()


def test_fused_sampled_step_equals_sample_then_step(golden_small):
    """The fused kernel's emitted triples equal the stand-alone sampler's, and applying them
    through the materialised-triple kernel on a conflict-free subset gives the same tables."""
    g = golden_small
    d = int(g["d"]); ld = ops.padded_dim(d)
    nu, ni = len(g["users"]), len(g["items"])
    indptr, _, srt = _csr_dev(g)
    n = 5000
    hp = [float(x) for x in g["hp"]]
    Ud, Vd = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32)
    bd = torch.zeros(ni, dtype=torch.float32, device=DEV)
    out = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_step_sampled_f32(Ud, Vd, bd, d, nu, ni, indptr, srt, n, 99, 7, *hp, loss=loss, out=out)
    u, i, j = ops.bpr_sample_philox(nu, ni, indptr, srt, n, seed=99, first=7)
    assert torch.equal(out[0], u) and torch.equal(out[1], i) and torch.equal(out[2], j)
    assert loss.item() > 0
    # tables moved and stayed finite
    assert torch.isfinite(Ud).all() and torch.isfinite(Vd).all()
    assert (Ud.cpu().numpy()[:, :d] != g["U0"].astype(np.float32)).any()


def test_exact_mode_rejects_triples_it_cannot_order():
    """i == j would make the ordered kernel wait on one row counter twice (ADVICE r1): it must be refused, not spin."""
    from elliot_b200._lib import EbError
    U = torch.zeros((4, 8), dtype=torch.float64, device=DEV); V = torch.zeros((5, 8), dtype=torch.float64, device=DEV)
    b = torch.zeros(5, dtype=torch.float64, device=DEV)
    t = lambda *a: torch.tensor(a, dtype=torch.int32, device=DEV)
    with pytest.raises(EbError, match="i == j"):
        ops.bpr_exact_f64(U, V, b, 8, t(0, 1), t(2, 3), t(4, 3), 0.05, 0, 0, 0, 0)
    with pytest.raises(EbError, match="out of range"):
        ops.bpr_exact_f64(U, V, b, 8, t(0, 9), t(2, 3), t(4, 1), 0.05, 0, 0, 0, 0)
    ops.bpr_exact_f64(U, V, b, 8, t(0, 1), t(2, 3), t(4, 1), 0.05, 0, 0, 0, 0)        # a valid batch still runs
    torch.cuda.synchronize()


def test_packed_host_triples_equal_the_three_array_path(golden_small):
    g = golden_small
    d = int(g["d"]); ld = ops.padded_dim(d)
    nu, ni = len(g["users"]), len(g["items"])
    hp = [float(x) for x in g["hp"]]
    seen_u, seen_i, keep = set(), set(), []
    for t in range(len(g["tu"])):                                  # conflict-free subset: the result is order independent
        u, i, j = g["tu"][t], g["ti"][t], g["tj"][t]
        if u in seen_u or i in seen_i or j in seen_i: continue
        seen_u.add(u); seen_i.add(i); seen_i.add(j); keep.append(t)
    keep = np.array(keep)
    tu, ti, tj = (torch.from_numpy(g[k][keep].astype(np.int32)) for k in ("tu", "ti", "tj"))
    packed = ops.pack_triples(tu, ti, tj, nu, ni).pin_memory()
    bu, bi = ops.pack_bits(nu, ni)
    assert int(packed[5]) == int(tu[5]) | (int(ti[5]) << bu) | (int(tj[5]) << (bu + bi))
    Ua, Va = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32); ba = torch.zeros(ni, device=DEV)
    Ub, Vb = Ua.clone(), Va.clone(); bb = torch.zeros(ni, device=DEV)
    la = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_step_f32(Ua, Va, ba, d, tu.to(DEV), ti.to(DEV), tj.to(DEV), *hp, loss=la)
    staging = torch.empty(packed.numel(), dtype=torch.int64, device=DEV)
    lb = torch.zeros(1, dtype=torch.float64, device=DEV); lh = torch.zeros(1, dtype=torch.float64).pin_memory()
    ops.bpr_step_host_packed_f32(Ub, Vb, bb, d, packed, nu, ni, *hp, staging, lb, lh)
    assert torch.equal(Ua, Ub) and torch.equal(Va, Vb) and torch.equal(ba, bb)
    assert abs(lh.item() - la.item()) < 1e-9 * abs(la.item())


def test_bad_arguments_raise():
    from elliot_b200._lib import EbError
    U = torch.zeros((4, 12), dtype=torch.float32, device=DEV)   # stride 12 is not a supported row stride
    b = torch.zeros(4, dtype=torch.float32, device=DEV)
    t = torch.zeros(4, dtype=torch.int32, device=DEV)
    with pytest.raises(EbError):
        ops.bpr_step_f32(U, U, b, 10, t, t, t, 0.05, 0, 0, 0, 0)
    with pytest.raises(RuntimeError):
        ops.bpr_step_f32(U.cpu(), U.cpu(), b.cpu(), 10, t.cpu(), t.cpu(), t.cpu(), 0.05, 0, 0, 0, 0)


def test_deterministic_rounds_repeat_and_match_sequential_without_conflicts(golden_small):
    """deterministic=True (rounds of reads, grid barrier, atomic adds, grid barrier): (1) a conflict-free batch still equals
    sequential SGD (fp32 vs the fp64 oracle: 2e-6 abs); (2) a conflict-heavy launch (a whole epoch over a 400 x 300 matrix)
    gives the same tables on a second run up to fp32 summation order (1e-5 relative to the largest entry),
    and its loss falls as sequential SGD's does."""
    g = golden_small
    d = int(g["d"]); ld = ops.padded_dim(d)
    hp = [float(x) for x in g["hp"]]
    keep = _conflict_free(g["tu"], g["ti"], g["tj"])
    tu, ti, tj = g["tu"][keep], g["ti"][keep], g["tj"][keep]
    U, V, b = g["U0"].copy(), g["V0"].copy(), np.zeros(len(g["items"]))
    oracle.bpr_update_seq(U, V, b, tu, ti, tj, *hp)
    Ud, Vd = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32)
    bd = torch.zeros(len(g["items"]), dtype=torch.float32, device=DEV)
    ops.bpr_step_f32(Ud, Vd, bd, d, torch.from_numpy(tu).to(DEV), torch.from_numpy(ti).to(DEV), torch.from_numpy(tj).to(DEV),
                     *hp, deterministic=True)
    torch.cuda.synchronize()
    assert np.abs(Ud.cpu().numpy()[:, :d] - U).max() < 2e-6 and np.abs(Vd.cpu().numpy()[:, :d] - V).max() < 2e-6
    assert np.abs(bd.cpu().numpy() - b).max() < 2e-6

    indptr, _, srt = _csr_dev(g)
    nu, ni, n = len(g["users"]), len(g["items"]), 200_000
    runs = []
    for _ in range(2):
        Ud, Vd = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32)
        bd = torch.zeros(ni, dtype=torch.float32, device=DEV)
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        ops.bpr_step_sampled_f32(Ud, Vd, bd, d, nu, ni, indptr, srt, n, 3, 0, *hp, loss=loss, deterministic=True)
        torch.cuda.synchronize()
        runs.append((Ud.cpu().numpy(), Vd.cpu().numpy(), bd.cpu().numpy(), loss.item()))
    for a, c in zip(runs[0][:3], runs[1][:3]):
        assert np.isfinite(a).all() and np.abs(a - c).max() < 1e-5 * max(1.0, np.abs(a).max())
    tu2, ti2, tj2 = ops.bpr_sample_philox(nu, ni, indptr, srt, n, 3, 0)
    tu2, ti2, tj2 = (x.cpu().numpy() for x in (tu2, ti2, tj2))
    l0 = oracle.bpr_loss(g["U0"], g["V0"], np.zeros(ni), tu2, ti2, tj2)
    l1 = oracle.bpr_loss(runs[0][0][:, :d].astype(np.float64), runs[0][1][:, :d].astype(np.float64), runs[0][2].astype(np.float64),
                         tu2, ti2, tj2)
    assert l1 < l0


def test_deterministic_rounds_are_refused_where_they_do_not_exist(golden_tiny):
    g = golden_tiny
    d = int(g["d"]); ld = ops.padded_dim(d)
    Ud, Vd = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32)
    bd = torch.zeros(len(g["items"]), dtype=torch.float32, device=DEV)
    t = torch.zeros(4, dtype=torch.int32, device=DEV)
    from elliot_b200._lib import EbError
    with pytest.raises(EbError):
        ops.bpr_step_f32(Ud, Vd, bd, d, t, t, t, 0.05, 0, 0, 0, 0, racy=True, deterministic=True)


def test_shared_memory_staged_kernel_is_refused_on_one_table(golden_tiny):
    """The shared-memory-staged kernel (_variant=32) exists for sharded item tables only."""
    from elliot_b200._lib import EbError
    g = golden_tiny
    d = int(g["d"]); ld = ops.padded_dim(d)
    nu, ni = len(g["users"]), len(g["items"])
    indptr, _, srt = _csr_dev(g)
    Ud, Vd = _pad(g["U0"], ld, np.float32), _pad(g["V0"], ld, np.float32)
    bd = torch.zeros(ni, dtype=torch.float32, device=DEV)
    with pytest.raises(EbError, match="sharded item tables only"):
        ops.bpr_step_sampled_f32(Ud, Vd, bd, d, nu, ni, indptr, srt, 64, 1, 0, 0.05, 0, 0, 0, 0, _variant=32)
    ops.bpr_step_sampled_f32(Ud, Vd, bd, d, nu, ni, indptr, srt, 64, 1, 0, 0.05, 0, 0, 0, 0, _variant=16)
    torch.cuda.synchronize()
