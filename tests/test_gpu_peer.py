"""Peer-addressed tables (csrc/peer.cu, PEER mode of csrc/bpr_train.cu; SURVEY.md §8e) on ONE GPU: the kernels only see
an array of shard base addresses, so several shards (or several replicas) allocated on the same device exercise
exactly the code that runs over NVLink when the shards sit on different GPUs.  The multi-process mapping itself
(CUDA IPC handles) is covered by tools/peer_check.py under torchrun."""
import numpy as np
import pytest
import torch

import oracle
from elliot_b200 import ops
from elliot_b200.parallel import PeerShardedTable, PeerTableSync, ceil_shard
from elliot_b200.peer import PeerBuffer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HP = (0.05, 0.0025, 0.01, 0.0025, 0.00025)


def _split(full, n_shards):
    """ceil-partition rows into separately allocated shard tensors (the last padded to shard_rows)."""
    sr = ceil_shard(full.shape[0], n_shards)
    out = []
    for s in range(n_shards):
        t = torch.zeros((sr,) + tuple(full.shape[1:]), device=full.device, dtype=full.dtype)
        blk = full[s * sr:(s + 1) * sr]
        t[:blk.shape[0]] = blk
        out.append(t)
    return out, sr


def _join(shards, n_rows):
    return torch.cat(shards)[:n_rows]


def test_peer_buffer_single_process():
    buf = PeerBuffer(1024, device=DEV)
    assert buf.kind == "single" and buf.ptrs[0] == buf.local.data_ptr() and buf.local.numel() == 1024
    assert not buf.local.any()                                    # eb_peer_alloc zero-fills
    buf.local.add_(1.0)
    assert float(buf.local.sum()) == 1024.0
    buf.close()


@pytest.mark.parametrize("n_shards,d", [(1, 64), (3, 64), (4, 32), (8, 128), (5, 60)])
def test_bpr_peer_step_equals_oracle_on_conflict_free_batch(golden_small, n_shards, d):
    g = golden_small
    rs = np.random.RandomState(d + n_shards)
    nu, ni = len(g["users"]), len(g["items"])
    ld = ops.padded_dim(d)
    U0 = rs.normal(0, 0.1, (nu, d)); V0 = rs.normal(0, 0.1, (ni, d)); b0 = rs.normal(0, 0.05, ni)
    seen_u, seen_i, keep = set(), set(), []
    for t in range(len(g["tu"])):
        u, i, j = g["tu"][t], g["ti"][t], g["tj"][t]
        if u in seen_u or i in seen_i or j in seen_i: continue
        seen_u.add(u); seen_i.add(i); seen_i.add(j); keep.append(t)
    keep = np.array(keep); tu, ti, tj = g["tu"][keep], g["ti"][keep], g["tj"][keep]
    U, V, b = U0.copy(), V0.copy(), b0.copy()
    oracle.bpr_update_seq(U, V, b, tu, ti, tj, *HP)
    Ud = torch.zeros((nu, ld), device=DEV); Ud[:, :d] = torch.from_numpy(U0).float().to(DEV)
    Vd = torch.zeros((ni, ld), device=DEV); Vd[:, :d] = torch.from_numpy(V0).float().to(DEV)
    bd = torch.from_numpy(b0).float().to(DEV)
    Vs, sr = _split(Vd, n_shards); bs, _ = _split(bd, n_shards)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_step_peer_f32(Ud, Vs, bs, sr, d, ni, torch.from_numpy(tu).to(DEV), torch.from_numpy(ti).to(DEV),
                          torch.from_numpy(tj).to(DEV), *HP, loss=loss)
    torch.cuda.synchronize()
    assert np.abs(Ud.cpu().numpy()[:, :d] - U).max() < 2e-6
    assert np.abs(_join(Vs, ni).cpu().numpy()[:, :d] - V).max() < 2e-6
    assert np.abs(_join(bs, ni).cpu().numpy() - b).max() < 2e-6
    assert loss.item() > 0


def test_bpr_sampled_peer_draws_the_same_triples_as_the_single_table_kernel(golden_small):
    g = golden_small
    nu, ni, d = len(g["users"]), len(g["items"]), 64
    indptr = torch.from_numpy(g["ui_indptr"].astype(np.int64)).to(DEV)
    srt = g["ui_indices"].astype(np.int32).copy()
    for u in range(nu):
        srt[g["ui_indptr"][u]:g["ui_indptr"][u + 1]].sort()
    srt = torch.from_numpy(srt).to(DEV)
    gen = torch.Generator(device=DEV); gen.manual_seed(3)
    U0 = torch.randn(nu, d, device=DEV, generator=gen) * 0.1; V0 = torch.randn(ni, d, device=DEV, generator=gen) * 0.1
    n = 512                                                       # few triples on a 400x300 matrix: conflicts are rare, order effects tiny
    out1 = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
    out2 = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
    U1, V1, b1 = U0.clone(), V0.clone(), torch.zeros(ni, device=DEV)
    ops.bpr_step_sampled_f32(U1, V1, b1, d, nu, ni, indptr, srt, n, 9, 77, *HP, out=out1)
    U2 = U0.clone(); Vs, sr = _split(V0, 3); bs, _ = _split(torch.zeros(ni, device=DEV), 3)
    l2 = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_step_sampled_peer_f32(U2, Vs, bs, sr, d, nu, ni, indptr, srt, n, 9, 77, *HP, loss=l2, out=out2)
    torch.cuda.synchronize()
    for a, c in zip(out1, out2):
        assert torch.equal(a, c)
    # same triples, same arithmetic; rows hit by several triples see them in a different (Hogwild) order: compare in norm
    rel = lambda a, c: ((a - c).norm() / c.norm().clamp_min(1e-12)).item()
    assert rel(U1, U2) < 1e-2 and rel(V1, _join(Vs, ni)) < 1e-2 and l2.item() > 0
    assert (b1 - _join(bs, ni)).abs().max().item() < 0.05


@pytest.mark.parametrize("n_rep,reduce", [(1, "mean"), (2, "mean"), (3, "mean"), (4, "sum"), (8, "mean")])
def test_reconcile_peer_kernel_agrees_on_mean_of_steps(n_rep, reduce):
    """n_rep replicas of one table on one device; "rank" r reconciles slice r of all of them."""
    gen = torch.Generator(device=DEV); gen.manual_seed(11)
    n = 4 * 5000 + 4 * 3                                          # float4 count not divisible by the replica count
    base = torch.randn(n, device=DEV, generator=gen)
    reps = [base.clone() for _ in range(n_rep)]
    n4 = n // 4
    cuts = [4 * (r * (n4 // n_rep) + min(r, n4 % n_rep)) for r in range(n_rep + 1)]
    prevs = [base[cuts[r]:cuts[r + 1]].clone() for r in range(n_rep)]
    scale = 1.0 / n_rep if reduce == "mean" else 1.0
    total = torch.zeros_like(base)
    for rnd in range(3):
        steps = []
        for r in range(n_rep):                                    # sparse local "training" on every replica
            st = torch.randn(n, device=DEV, generator=gen) * (torch.rand(n, device=DEV, generator=gen) < 0.3)
            reps[r] += st; steps.append(st)
        for r in range(n_rep):
            ptrs = [t.data_ptr() + 4 * cuts[r] for t in reps]
            ops.table_reconcile_peer_f32(ptrs, prevs[r], scale)
        total += scale * sum(steps)
        torch.cuda.synchronize()
        want = base + total
        for t in reps:
            assert (t - want).abs().max().item() < 1e-5
        assert (torch.cat(prevs) - want).abs().max().item() < 1e-5


def test_reconcile_keeps_updates_that_arrive_after_the_snapshot():
    """What a replica adds between two reconciliations is never lost nor counted twice: after k rounds with fresh
    local steps in between, every replica = base + mean of ALL steps except its own still-unshared last one."""
    gen = torch.Generator(device=DEV); gen.manual_seed(5)
    n, R = 4096, 3
    base = torch.randn(n, device=DEV, generator=gen)
    reps = [base.clone() for _ in range(R)]
    prev = base.clone()
    shared = torch.zeros_like(base)
    ptrs = [t.data_ptr() for t in reps]
    for rnd in range(4):
        steps = [torch.randn(n, device=DEV, generator=gen) * 0.1 for _ in range(R)]
        for t, s in zip(reps, steps):
            t += s
        ops.table_reconcile_peer_f32(ptrs, prev, 1.0 / R)
        late = [torch.randn(n, device=DEV, generator=gen) * 0.1 for _ in range(R)]      # arrives "during" the next step
        for t, s in zip(reps, late):
            t += s
        shared += sum(steps) / R
        torch.cuda.synchronize()
        for t, s in zip(reps, late):
            assert (t - (base + shared + s)).abs().max().item() < 1e-5
        # the late parts are the next round's local deltas
        ops.table_reconcile_peer_f32(ptrs, prev, 1.0 / R)
        shared += sum(late) / R
        torch.cuda.synchronize()
        for t in reps:
            assert (t - (base + shared)).abs().max().item() < 1e-5


def test_peer_table_sync_single_rank_is_a_no_op():
    buf = PeerBuffer(4096, device=DEV)
    buf.local.normal_()
    sync = PeerTableSync(buf)
    before = buf.local.clone()
    buf.local[:100] += 1.0
    sync.sync(); sync.flush()
    torch.cuda.synchronize()
    assert torch.allclose(buf.local[:100], before[:100] + 1.0) and torch.equal(buf.local[100:], before[100:])
    buf.close()


@pytest.mark.parametrize("n_shards", [1, 3, 4])
def test_neumf_peer_gather_scatter_equal_the_single_table_kernels(n_shards):
    gen = torch.Generator(device=DEV); gen.manual_seed(2)
    nu, ni, f, B = 300, 157, 16, 2000
    Umf = torch.randn(nu, f, device=DEV, generator=gen); Umlp = torch.randn(nu, f, device=DEV, generator=gen)
    Imf = torch.randn(ni, f, device=DEV, generator=gen); Imlp = torch.randn(ni, f, device=DEV, generator=gen)
    u = torch.randint(0, nu, (B,), device=DEV, generator=gen, dtype=torch.int32)
    it = torch.randint(0, ni, (B,), device=DEV, generator=gen, dtype=torch.int32)
    x0 = torch.empty(B, 2 * f, device=DEV); pm = torch.empty(B, f, device=DEV)
    ops.neumf_gather(Umf, Imf, Umlp, Imlp, f, u, it, x0, pm)
    I = torch.cat([Imf, Imlp], dim=1).contiguous()
    Is, sr = _split(I, n_shards)
    x0p = torch.empty_like(x0); pmp = torch.empty_like(pm)
    ops.neumf_gather_peer(Umf, Umlp, Is, sr, 2 * f, f, u, it, x0p, pmp)
    assert torch.equal(x0, x0p) and torch.equal(pm, pmp)
    dpm = torch.randn(B, f, device=DEV, generator=gen); dx0 = torch.randn(B, 2 * f, device=DEV, generator=gen)
    dUmf, dImf, dUmlp, dImlp = (torch.zeros_like(t) for t in (Umf, Imf, Umlp, Imlp))
    ops.neumf_scatter(Umf, Imf, f, u, it, dpm, dx0, dUmf, dImf, dUmlp, dImlp)
    dUmf2, dUmlp2 = torch.zeros_like(Umf), torch.zeros_like(Umlp)
    GIs = [torch.zeros_like(t) for t in Is]
    ops.neumf_scatter_peer(Umf, Is, GIs, sr, 2 * f, f, u, it, dpm, dx0, dUmf2, dUmlp2)
    GI = _join(GIs, ni)
    tol = dict(rtol=1e-4, atol=1e-4)                              # atomic accumulation order differs
    assert torch.allclose(dUmf, dUmf2, **tol) and torch.allclose(dUmlp, dUmlp2, **tol)
    assert torch.allclose(GI[:, :f], dImf, **tol) and torch.allclose(GI[:, f:], dImlp, **tol)
    rows = ops.gather_rows_peer_f32(Is, sr, 2 * f, it, 2 * f)
    assert torch.equal(rows, I[it.long()])


def test_sharded_neumf_single_rank_tracks_the_ordinary_model():
    from elliot_b200.recommender.neumf import NeuralMatrixFactorizationModel
    from elliot_b200.recommender.neumf_sharded import ShardedNeuMFModel
    nu, ni, f, B = 500, 300, 16, 1024
    ref = NeuralMatrixFactorizationModel(nu, ni, f, 1e-3, 42, DEV)
    sh = ShardedNeuMFModel(nu, ni, f, 1e-3, 42, DEV)
    assert torch.equal(sh.P["U_mf"], ref.P["U_mf"]) and torch.equal(sh.P["I"][:ni, :f], ref.P["I_mf"])
    assert torch.equal(sh.P["I"][:ni, f:], ref.P["I_mlp"]) and torch.equal(sh.P["W1"], ref.P["W1"])
    gen = torch.Generator(device=DEV); gen.manual_seed(8)
    for _ in range(3):
        u = torch.randint(0, nu, (B,), device=DEV, generator=gen, dtype=torch.int32)
        it = torch.randint(0, ni, (B,), device=DEV, generator=gen, dtype=torch.int32)
        y = (torch.rand(B, device=DEV, generator=gen) < 0.3).float()
        l1 = ref.train_step((u, it, y)).item(); l2 = sh.train_step((u, it, y)).item()
        assert abs(l1 - l2) < 1e-6 * max(1.0, abs(l1))
    rel = lambda a, b: float((a - b).norm() / b.norm().clamp_min(1e-12))
    assert rel(sh.P["U_mf"], ref.P["U_mf"]) < 1e-5 and rel(sh.P["I"][:ni, :f], ref.P["I_mf"]) < 1e-5
    assert rel(sh.P["I"][:ni, f:], ref.P["I_mlp"]) < 1e-5 and rel(sh.P["W2"], ref.P["W2"]) < 1e-5
    # scoring over the sharded item table = the ordinary model's scoring
    indptr = torch.zeros(nu + 1, dtype=torch.int64, device=DEV); indices = torch.zeros(1, dtype=torch.int32, device=DEV)
    i1, v1 = ref.get_recs_topk(0, 64, 5, indptr, indices); i2, v2 = sh.get_recs_topk(0, 64, 5, indptr, indices)
    assert (i1 == i2).float().mean().item() > 0.98 and torch.allclose(v1, v2, atol=1e-4)
    sh.close()


@pytest.mark.parametrize("two_ids", [False, True])
def test_group_by_owner_is_a_permutation_ordered_by_rotated_owner(two_ids):
    """eb_group_by_owner_i32: the three arrays travel together, the elements come out bucketed by
    ((owner(i) - rank) mod W [, (owner(j) - rank) mod W]) in ascending order, nothing is lost or duplicated."""
    dev = DEV
    g = torch.Generator(device=dev); g.manual_seed(5)
    n, world, rank, shard_rows = 300_001, 8, 3, 12_345
    n_items = shard_rows * world - 7                                   # the last shard is short
    u = torch.randint(0, 1_000_000, (n,), device=dev, generator=g, dtype=torch.int32)
    i = torch.randint(0, n_items, (n,), device=dev, generator=g, dtype=torch.int32)
    j = torch.randint(0, n_items, (n,), device=dev, generator=g, dtype=torch.int32)
    y = torch.rand(n, device=dev, generator=g)
    if two_ids:
        ou, oi, oj = ops.group_by_owner([u, i, j], 1, 2, shard_rows, rank, world)
        key = ((oi // shard_rows - rank) % world) * world + (oj // shard_rows - rank) % world
        before = torch.stack([u, i, j], 1); after = torch.stack([ou, oi, oj], 1)
    else:
        ou, oi, oy = ops.group_by_owner([u, i, y], 1, -1, shard_rows, rank, world)
        assert oy.dtype == torch.float32
        key = (oi // shard_rows - rank) % world
        before = torch.stack([u, i, y.view(torch.int32)], 1); after = torch.stack([ou, oi, oy.view(torch.int32)], 1)
    assert (key[1:] >= key[:-1]).all()
    # exact multiset equality through a full lexicographic sort
    def lex(t):
        t = t.cpu().long()
        for c in (2, 1, 0):
            t = t[torch.argsort(t[:, c], stable=True)]
        return t
    assert torch.equal(lex(before), lex(after))
