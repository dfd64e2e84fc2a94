"""Row-sharded item tables (SURVEY.md §8e): kernels + the fetch/update/push protocol at world size 1 against the
replicated-table kernel and the oracle; the multi-rank exchange itself is covered by tests/test_parallel_cpu.py
(gloo) and tools/sharded_check.py (torchrun on 2+ GPUs)."""
import numpy as np
import pytest
import torch

import oracle
from elliot_b200 import ops
from elliot_b200.parallel import ShardedTable, sharded_bpr_step

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_gather_scatter_rows():
    g = torch.Generator(device=DEV); g.manual_seed(0)
    T = torch.randn(50, 16, device=DEV, generator=g)
    ids = torch.tensor([3, 3, 49, 0, 17], dtype=torch.int32, device=DEV)
    rows = ops.gather_rows_f32(T, ids)
    assert torch.equal(rows, T[ids.long()])
    T2 = T.clone()
    ops.scatter_add_rows_f32(T2, ids, torch.ones_like(rows))
    want = T.clone(); want.index_add_(0, ids.long(), torch.ones_like(rows))
    assert torch.allclose(T2, want)


@pytest.mark.parametrize("d,with_bias", [(60, True), (64, False), (10, True)])
def test_sharded_step_equals_sequential_on_conflict_free_batch(golden_small, d, with_bias):
    g = golden_small
    rs = np.random.RandomState(d)
    nu, ni = len(g["users"]), len(g["items"])
    ld = ops.padded_dim(d + (1 if with_bias else 0))
    U0 = rs.normal(0, 0.1, (nu, d)); V0 = rs.normal(0, 0.1, (ni, d)); b0 = rs.normal(0, 0.05, ni) if with_bias else np.zeros(ni)
    seen_u, seen_i, keep = set(), set(), []
    for t in range(len(g["tu"])):
        u, i, j = g["tu"][t], g["ti"][t], g["tj"][t]
        if u in seen_u or i in seen_i or j in seen_i: continue
        seen_u.add(u); seen_i.add(i); seen_i.add(j); keep.append(t)
    keep = np.array(keep); tu, ti, tj = g["tu"][keep], g["ti"][keep], g["tj"][keep]
    hp = (0.05, 0.0025, 0.01 if with_bias else 0.0, 0.0025, 0.00025)
    U, V, b = U0.copy(), V0.copy(), b0.copy()
    oracle.bpr_update_seq(U, V, b, tu, ti, tj, *hp)
    Ud = torch.zeros((nu, ld), device=DEV); Ud[:, :d] = torch.from_numpy(U0).float().to(DEV)
    Vd = torch.zeros((ni, ld), device=DEV); Vd[:, :d] = torch.from_numpy(V0).float().to(DEV)
    if with_bias: Vd[:, d] = torch.from_numpy(b0).float().to(DEV)
    items = ShardedTable(ni, Vd)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    sharded_bpr_step(Ud, items, torch.from_numpy(tu).to(DEV), torch.from_numpy(ti).to(DEV), torch.from_numpy(tj).to(DEV), hp,
                     bias_col=d if with_bias else -1, loss=loss)
    torch.cuda.synchronize()
    assert np.abs(Ud.cpu().numpy()[:, :d] - U).max() < 2e-6
    assert np.abs(Vd.cpu().numpy()[:, :d] - V).max() < 2e-6
    if with_bias:
        assert np.abs(Vd.cpu().numpy()[:, d] - b).max() < 2e-6
        assert not Ud[:, d:].any()                                # the bias column never leaks into the user rows
    assert loss.item() > 0


def test_table_delta_apply_and_late_kernels():
    """Replicated-table reconciliation kernels: delta = cur - prev; apply: cur = prev = prev + scale*sum;
    late: cur += scale*sum - local, prev += scale*sum (atomic on cur)."""
    g = torch.Generator(device=DEV); g.manual_seed(3)
    n = 4 * 1031
    prev = torch.randn(n, device=DEV, generator=g); cur = prev + torch.randn(n, device=DEV, generator=g) * 0.1
    d = torch.empty_like(cur)
    ops.table_delta_f32(cur, prev, d)
    assert torch.equal(d, cur - prev)
    other = torch.randn(n, device=DEV, generator=g) * 0.1          # stands in for the other ranks' deltas
    s = d + other
    c1, p1 = cur.clone(), prev.clone()
    ops.table_apply_delta_f32(c1, p1, s, 0.5)
    want = prev + 0.5 * s
    assert torch.allclose(c1, want, atol=1e-6) and torch.equal(c1, p1)
    c2, p2 = cur.clone(), prev.clone()
    newer = torch.randn(n, device=DEV, generator=g) * 0.01          # local updates made while the all-reduce ran
    c2 += newer
    ops.table_apply_delta_late_f32(c2, p2, s, d, 0.5)
    assert torch.allclose(p2, want, atol=1e-6)
    assert torch.allclose(c2, want + newer, atol=1e-6)


def test_reserved_sms_grid_gives_same_statistics(golden_small):
    """flags bits 8..15 only shrink the persistent grid: the sampled triples (a pure function of the counter) are
    identical and the update is the same Hogwild step."""
    g = golden_small
    nu, ni = len(g["users"]), len(g["items"])
    ip = g["ui_indptr"].astype(np.int64); srt = g["ui_indices"].astype(np.int32).copy()
    for x in range(nu):
        srt[ip[x]:ip[x + 1]].sort()
    indptr = torch.from_numpy(ip).to(DEV); indices = torch.from_numpy(srt).to(DEV)
    n = 4096
    outs = []
    for reserve in (0, 100):
        gen = torch.Generator(device=DEV); gen.manual_seed(1)
        U = torch.randn(nu, 16, device=DEV, generator=gen) * 0.1; V = torch.randn(ni, 16, device=DEV, generator=gen) * 0.1
        b = torch.zeros(ni, device=DEV)
        out = tuple(torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3))
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        ops.bpr_step_sampled_f32(U, V, b, 16, nu, ni, indptr, indices, n, 5, 0, 0.05, 0.0025, 0.0, 0.0025, 0.00025,
                                 loss=loss, out=out, reserve_sms=reserve)
        outs.append((out, loss.item(), U.clone(), V.clone()))
    for a, c in zip(outs[0][0], outs[1][0]):
        assert torch.equal(a, c)
    # Hogwild: conflicting rows race differently from launch to launch, so only statistics are compared
    assert abs(outs[0][1] - outs[1][1]) < 2e-2 * abs(outs[0][1])
    assert (outs[0][2] - outs[1][2]).abs().mean() < 2e-3 and (outs[0][3] - outs[1][3]).abs().mean() < 2e-3


def test_partition_stream_runs_kernels_inside_green_context():
    """eb_partition_streams_create: streams bound to an SM partition; a step launched there gives the same result
    as on the default stream (conflict-free batch -> deterministic)."""
    streams, granted = ops.partition_streams(torch.device(DEV), 16, 2)
    total = ops.device_info()[0]
    assert len(streams) == 2 and 8 <= granted <= total - 16
    g = torch.Generator(device=DEV); g.manual_seed(5)
    n = 2000
    U = torch.randn(n, 64, device=DEV, generator=g) * 0.1; V = torch.randn(2 * n, 64, device=DEV, generator=g) * 0.1
    b = torch.zeros(2 * n, device=DEV)
    tu = torch.arange(n, dtype=torch.int32, device=DEV); ti = tu.clone(); tj = tu + n
    hp = (0.05, 0.0025, 0.0, 0.0025, 0.00025)
    U1, V1, b1 = U.clone(), V.clone(), b.clone()
    ops.bpr_step_f32(U1, V1, b1, 64, tu, ti, tj, *hp)
    U2, V2, b2 = U.clone(), V.clone(), b.clone()
    torch.cuda.synchronize()
    with torch.cuda.stream(streams[0]):
        ops.bpr_step_f32(U2, V2, b2, 64, tu, ti, tj, *hp)
    streams[0].synchronize()
    assert torch.equal(U1, U2) and torch.equal(V1, V2) and torch.equal(b1, b2)
