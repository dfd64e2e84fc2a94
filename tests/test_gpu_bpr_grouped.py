"""The free-running sampled BPR step applies its triples grouped by user (key pass, stable sort by user, grouped update):
same samples as the stand-alone sampler, the per-triple kernel's arithmetic wherever runs have one triple, and the update's
invariants where users repeat many times per launch."""
import numpy as np
import pytest
import torch

import oracle
from elliot_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HP = (0.05, 0.0025, 0.01, 0.0025, 0.00025)


def _csr(rows):
    indptr = torch.tensor(np.cumsum([0] + [len(r) for r in rows]), dtype=torch.int64, device=DEV)
    idx = torch.tensor([x for r in rows for x in sorted(r)], dtype=torch.int32, device=DEV)
    return indptr, idx


def _tables(nu, ni, d, seed):
    ld = ops.padded_dim(d)
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    U = torch.zeros((nu, ld), device=DEV); U[:, :d] = torch.randn(nu, d, device=DEV, generator=g) * 0.1
    V = torch.zeros((ni, ld), device=DEV); V[:, :d] = torch.randn(ni, d, device=DEV, generator=g) * 0.1
    b = torch.randn(ni, device=DEV, generator=g) * 0.05
    return U, V, b


def _fused(U, V, b, d, nu, ni, indptr, idx, n, seed, hp, **kw):
    out = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_step_sampled_f32(U, V, b, d, nu, ni, indptr, idx, n, seed, 11, *hp, loss=loss, out=out, **kw)
    torch.cuda.synchronize()
    return out, loss.item()


@pytest.mark.parametrize("d", [5, 16, 30, 64, 100, 256])
def test_grouped_step_is_bitwise_the_per_triple_step_without_conflicts(d):
    """Many users with one item each over a huge item range: one sampled batch repeats no u, i or j, so every user run has
    one triple and the grouped step must leave exactly the tables the per-triple kernel leaves on the emitted triples (atomic
    and racy alike).  The loss is summed in a different lane order: 1e-6 relative."""
    nu = ni = 1 << 22
    n = 256
    indptr = torch.arange(nu + 1, dtype=torch.int64, device=DEV)
    idx = torch.arange(nu, dtype=torch.int32, device=DEV)
    for seed in range(1, 20):                                   # the first seed whose batch has no repeated row
        u, i, j = (x.cpu().numpy() for x in ops.bpr_sample_philox(nu, ni, indptr, idx, n, seed, 11))
        if len(np.unique(u)) == n and len(np.unique(np.concatenate([i, j]))) == 2 * n:
            break
    else:
        pytest.fail("no conflict-free seed")
    U0, V0, b0 = _tables(nu, ni, d, d)
    for racy in (False, True):
        Ua, Va, ba = U0.clone(), V0.clone(), b0.clone()
        out, la = _fused(Ua, Va, ba, d, nu, ni, indptr, idx, n, seed, HP, racy=racy)
        assert np.array_equal(out[0].cpu().numpy(), u) and np.array_equal(out[1].cpu().numpy(), i)
        assert np.array_equal(out[2].cpu().numpy(), j)
        Ub, Vb, bb = U0.clone(), V0.clone(), b0.clone()
        lb = torch.zeros(1, dtype=torch.float64, device=DEV)
        ops.bpr_step_f32(Ub, Vb, bb, d, *out, *HP, loss=lb, racy=racy)
        torch.cuda.synchronize()
        assert not torch.equal(Ua, U0)
        for name, a, c in (("U", Ua, Ub), ("V", Va, Vb), ("b", ba, bb)):
            assert torch.equal(a, c), (racy, name, (a - c).abs().max().item())
        assert abs(la - lb.item()) <= 1e-6 * lb.item(), (racy, la, lb.item())
        del Ua, Va, ba, Ub, Vb, bb


def _heavy():
    nu, ni, d = 50, 2000, 64
    rs = np.random.RandomState(5)
    rows = [rs.choice(ni, rs.randint(1, 80), replace=False) for _ in range(nu)]
    return nu, ni, d, rows


def test_grouped_step_with_heavy_user_repetition():
    """50 users and 200K triples per call: user runs straddle lane-group and window boundaries and many warps add partial
    updates to the same user row.  Emitted triples equal the sampler's; with zero regularisation the column sums of V and the
    sum of b are invariant (every triple adds +lr z u' to V_i and -lr z u' to V_j); the batch loss drops and the user rows
    move as sequential SGD on the emitted triples moves them (relative Frobenius error of U1 - U0, which a lost or doubled
    flush of a run would blow up); lr = 0 leaves the tables bit-identical."""
    nu, ni, d, rows = _heavy()
    indptr, idx = _csr(rows)
    n = 200_000
    U0, V0, b0 = _tables(nu, ni, d, 3)

    U, V, b = U0.clone(), V0.clone(), b0.clone()
    out, _ = _fused(U, V, b, d, nu, ni, indptr, idx, n, 9, (0.002, 0.0, 0.0, 0.0, 0.0))
    want = ops.bpr_sample_philox(nu, ni, indptr, idx, n, 9, 11)
    assert all(torch.equal(a, c) for a, c in zip(out, want))
    assert torch.isfinite(U).all() and torch.isfinite(V).all()
    assert not torch.equal(U, U0)
    col0, col1 = V0.double().sum(0), V.double().sum(0)
    assert (col1 - col0).abs().max().item() < 5e-3 * V0.double().abs().sum(0).max().item() / 1e3
    assert abs(b.double().sum().item() - b0.double().sum().item()) < 1e-3

    hp = (0.002, 0.0025, 0.01, 0.0025, 0.00025)
    U, V, b = U0.clone(), V0.clone(), b0.clone()
    out, _ = _fused(U, V, b, d, nu, ni, indptr, idx, n, 10, hp)
    tu, ti, tj = (x.cpu().numpy() for x in out)
    Us, Vs, bs = (x.double().cpu().numpy() for x in (U0[:, :d], V0[:, :d], b0))
    l0 = oracle.bpr_loss(Us, Vs, bs, tu, ti, tj)
    oracle.bpr_update_seq(Us, Vs, bs, tu, ti, tj, *hp)
    Uh, Vh = U[:, :d].double().cpu().numpy(), V[:, :d].double().cpu().numpy()
    l1 = oracle.bpr_loss(Uh, Vh, b.double().cpu().numpy(), tu, ti, tj)
    assert l1 < l0
    # Hogwild staleness alone: 0.134-0.136 over 5 runs on an H100 80GB HBM3 (700 W); bound with 1.5x margin
    U0h = U0[:, :d].double().cpu().numpy()
    eu = np.linalg.norm((Uh - U0h) - (Us - U0h)) / np.linalg.norm(Us - U0h)
    assert eu < 0.2, eu
    cv = np.corrcoef(Vh.ravel(), Vs.ravel())[0, 1]
    assert cv > 0.98, cv

    U, V, b = U0.clone(), V0.clone(), b0.clone()
    _fused(U, V, b, d, nu, ni, indptr, idx, n, 10, (0.0,) + HP[1:])
    assert torch.equal(U, U0) and torch.equal(V, V0) and torch.equal(b, b0)


@pytest.mark.parametrize("n", [1, 20, 33, 1000])
def test_grouped_step_edge_shapes_emit_the_sampler_triples(n):
    """Fewer triples than one window, one triple, a single user, users without items and users owning every item or all but
    a few (the redraw and the rank paths of the sampler): the emitted triples are the stand-alone sampler's."""
    ni, d = 64, 16
    cases = {
        "one user": [[3, 9, 20]],
        "redraw and rank": [list(range(ni)), [x for x in range(ni) if x not in (5, 17, 40)], [], [1, 2, 3]],
    }
    for name, rows in cases.items():
        nu = len(rows)
        indptr, idx = _csr(rows)
        U, V, b = _tables(nu, ni, d, n)
        out, loss = _fused(U, V, b, d, nu, ni, indptr, idx, n, 4, HP)
        want = ops.bpr_sample_philox(nu, ni, indptr, idx, n, 4, 11)
        assert all(torch.equal(a, c) for a, c in zip(out, want)), name
        assert loss > 0 and torch.isfinite(U).all() and torch.isfinite(V).all(), name


def test_grouped_step_refuses_a_short_workspace():
    from elliot_b200._lib import EbError, check, lib
    nu, ni, d, rows = _heavy()
    indptr, idx = _csr(rows)
    U, V, b = _tables(nu, ni, d, 1)
    n = 5000
    need = lib().eb_bpr_step_sampled_workspace_bytes(n, nu)
    assert need >= 16 * n
    ws = torch.empty(need - 256, dtype=torch.uint8, device=DEV)
    with pytest.raises(EbError, match="workspace"):
        check(lib().eb_bpr_step_sampled_f32(U.data_ptr(), V.data_ptr(), b.data_ptr(), d, U.stride(0), nu, ni, indptr.data_ptr(),
                                            idx.data_ptr(), n, 1, 0, *HP, None, None, None, None, ws.data_ptr(), ws.numel(), 0,
                                            torch.cuda.current_stream().cuda_stream))
    with pytest.raises(EbError, match="sharded item tables only"):
        ops.bpr_step_sampled_f32(U, V, b, d, nu, ni, indptr, idx, n, 1, 0, *HP, _variant=32)
    ops.bpr_step_sampled_f32(U, V, b, d, nu, ni, indptr, idx, n, 1, 0, *HP)
    torch.cuda.synchronize()
    assert torch.isfinite(U).all()
