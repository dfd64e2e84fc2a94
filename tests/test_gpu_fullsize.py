"""Parity at BASELINE.json's sizes through size-independent properties (and, where the oracle still finishes in
seconds, directly against it)."""
import numpy as np
import pytest
import torch

import oracle
from elliot_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _synth_csr(nu, ni, per, seed):
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    cand = (torch.rand(nu, per, device=DEV, generator=g) ** 2 * ni).to(torch.int32).clamp_(max=ni - 1)
    cand, _ = torch.sort(cand, dim=1)
    keep = torch.ones_like(cand, dtype=torch.bool); keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    indptr = torch.zeros(nu + 1, dtype=torch.int64, device=DEV); indptr[1:] = torch.cumsum(keep.sum(1), 0)
    return indptr, cand[keep].contiguous()


@pytest.fixture(scope="module")
def c2():
    nu, ni, d = 1_000_000, 100_000, 64
    g = torch.Generator(device=DEV); g.manual_seed(0)
    U = torch.randn(nu, d, device=DEV, generator=g) * 0.1; V = torch.randn(ni, d, device=DEV, generator=g) * 0.1
    b = torch.randn(ni, device=DEV, generator=g) * 0.01
    indptr, indices = _synth_csr(nu, ni, 100, 1)
    return nu, ni, d, U, V, b, indptr, indices


def test_c2_fused_step_invariants(c2):
    """C2 (1M x 100K, d=64, 4M triples/launch): sampled triples are valid; with zero regularisation every triple adds
    +lr z u' to V_i and -lr z u' to V_j, so the column sums of V and the sum of the biases are invariant (a checksum
    over all 4M scatter-adds); lr = 0 leaves the tables bit-identical (idempotence)."""
    nu, ni, d, U, V, b, indptr, indices = c2
    n = 1 << 22
    U1, V1, b1 = U.clone(), V.clone(), b.clone()
    out = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_step_sampled_f32(U1, V1, b1, d, nu, ni, indptr, indices, n, 7, 0, 0.05, 0.0, 0.0, 0.0, 0.0, loss=loss, out=out)
    torch.cuda.synchronize()
    tu, ti, tj = [x.long() for x in out]
    assert tu.min() >= 0 and tu.max() < nu and tj.min() >= 0 and tj.max() < ni
    # membership through the CSR: i in row(u), j not in row(u), on a 200K sample
    sel = torch.randint(0, n, (200_000,), device=DEV)
    for t_items, want in ((ti[sel], True), (tj[sel], False)):
        beg, end = indptr[tu[sel]], indptr[tu[sel] + 1]
        lo = beg.clone(); hi = end.clone()
        for _ in range(8):                                                         # vectorised binary search inside each row
            mid = (lo + hi) // 2
            go = (indices[mid.clamp(max=indices.numel() - 1)].long() < t_items) & (lo < hi)
            lo = torch.where(go, mid + 1, lo); hi = torch.where(go, hi, torch.minimum(hi, mid))
        found = (lo < end) & (indices[lo.clamp(max=indices.numel() - 1)].long() == t_items)
        assert bool((found == want).all())
    assert torch.isfinite(U1).all() and torch.isfinite(V1).all()
    col0, col1 = V.double().sum(0), V1.double().sum(0)
    assert (col1 - col0).abs().max().item() < 5e-3 * V.double().abs().sum(0).max().item() / 1e3     # ~fp32 atomic rounding of 8M adds
    assert abs(b1.double().sum().item() - b.double().sum().item()) < 1e-2
    assert (U1 != U).any()
    # idempotence with lr = 0
    U2, V2, b2 = U.clone(), V.clone(), b.clone()
    ops.bpr_step_sampled_f32(U2, V2, b2, d, nu, ni, indptr, indices, n, 7, 0, 0.0, 0.0025, 0.0, 0.0025, 0.00025)
    assert torch.equal(U2, U) and torch.equal(V2, V) and torch.equal(b2, b)
    # determinism of the sampler stream: same seed/offset -> same triples
    out2 = ops.bpr_sample_philox(nu, ni, indptr, indices, n, 7, 0)
    assert all(torch.equal(a, c) for a, c in zip(out, out2))


def test_c2_scoring_properties_and_spot_parity(c2):
    """C2 scoring (100K items, bias + mask) on 33 792 users (two 128-user blocks per H100 SM): descending scores, no train item, idempotent, and
    identical to the exact kernel on 1 024 of the users."""
    nu, ni, d, U, V, b, indptr, indices = c2
    ns = 132 * 128 * 2
    idx, val, st = ops.score_topk_tc(U, V, b, d, 10, indptr, indices, user_begin=0, n_sel=ns)
    idx2, val2, _ = ops.score_topk_tc(U, V, b, d, 10, indptr, indices, user_begin=0, n_sel=ns)
    assert torch.equal(idx, idx2) and torch.equal(val, val2)
    assert bool((val[:, :-1] >= val[:, 1:]).all()) and bool((idx >= 0).all())
    rows = torch.arange(ns, device=DEV).repeat_interleave(10)
    flat = idx.reshape(-1).long()
    lo, hi = indptr[rows].clone(), indptr[rows + 1].clone(); end = hi.clone()
    for _ in range(8):
        mid = (lo + hi) // 2
        go = (indices[mid.clamp(max=indices.numel() - 1)].long() < flat) & (lo < hi)
        lo = torch.where(go, mid + 1, lo); hi = torch.where(go, hi, torch.minimum(hi, mid))
    hit = (lo < end) & (indices[lo.clamp(max=indices.numel() - 1)].long() == flat)
    assert not bool(hit.any())                                   # no masked (train) item is ever recommended
    i0, v0 = ops.score_topk(U, V, b, d, 10, indptr, indices, user_begin=0, n_sel=1024)
    assert torch.equal(i0, idx[:1024]) and torch.equal(v0, val[:1024])


def test_c1_exact_epoch_equals_oracle():
    """C1 scale (6 040 x 3 706, one 800 K-triple epoch, d=64): device MT19937 replay and the sequentially consistent
    fp64 update against the C oracle end to end (the oracle needs ~1 s)."""
    rs = np.random.RandomState(0)
    nu, ni, d, T = 6040, 3706, 64, 800_000
    rows = [np.unique((rs.rand(rs.randint(20, 260)) ** 2 * ni).astype(np.int32)) for _ in range(nu)]
    setrows = [np.array(list(set(r.tolist())), np.int32) for r in rows]      # the reference's list(set(..)) order
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in setrows])
    set_idx = np.concatenate(setrows); srt_idx = np.concatenate([np.sort(r) for r in setrows])
    rng = oracle.Rng(42)
    ou, oi, oj, _ = oracle.sampler_step(rng, nu, ni, indptr, set_idx, T)
    U0 = rs.normal(0, 0.1, (nu, d)); V0 = rs.normal(0, 0.1, (ni, d))
    U, V, b = U0.copy(), V0.copy(), np.zeros(ni)
    hp = (0.05, 0.0025, 0.0, 0.0025, 0.00025)
    oracle.bpr_update_seq(U, V, b, ou, oi, oj, *hp)
    s = ops.MtSampler(nu, ni, torch.from_numpy(indptr).to(DEV), torch.from_numpy(set_idx).to(DEV), torch.from_numpy(srt_idx).to(DEV), 42)
    tu, ti, tj = s.step(T)
    assert np.array_equal(tu.cpu().numpy(), ou) and np.array_equal(ti.cpu().numpy(), oi) and np.array_equal(tj.cpu().numpy(), oj)
    Ud, Vd = torch.from_numpy(U0.copy()).to(DEV), torch.from_numpy(V0.copy()).to(DEV)
    bd = torch.zeros(ni, dtype=torch.float64, device=DEV)
    ops.bpr_exact_f64(Ud, Vd, bd, d, tu, ti, tj, *hp)
    torch.cuda.synchronize()
    assert np.abs(Ud.cpu().numpy() - U).max() < 1e-10 and np.abs(Vd.cpu().numpy() - V).max() < 1e-10
    assert np.abs(bd.cpu().numpy() - b).max() < 1e-10
    # and the rankings: identical top-10 lists for all users (fp64 scores)
    idx, val = ops.score_topk(Ud, Vd, bd, d, 10, torch.from_numpy(indptr).to(DEV), torch.from_numpy(set_idx).to(DEV))
    oi10, ov10 = oracle.user_topk(U, V, b, indptr, set_idx, np.arange(0, nu, 7), 10)
    assert np.array_equal(idx.cpu().numpy()[::7], oi10)


def test_empty_and_degenerate_inputs():
    U = torch.zeros((8, 64), device=DEV); V = torch.zeros((8, 64), device=DEV); b = torch.zeros(8, device=DEV)
    e = torch.zeros(0, dtype=torch.int32, device=DEV)
    ops.bpr_step_f32(U, V, b, 64, e, e, e, 0.05, 0, 0, 0, 0)                          # n = 0 is a no-op
    Ud = U.double(); Vd = V.double(); bd = b.double()
    ops.bpr_exact_f64(Ud, Vd, bd, 64, e, e, e, 0.05, 0, 0, 0, 0)
    # single user, catalogue smaller than one MMA tile, k = 1
    g = torch.Generator(device=DEV); g.manual_seed(1)
    U1 = torch.randn(1, 64, device=DEV, generator=g); V1 = torch.randn(5, 64, device=DEV, generator=g)
    i0, v0 = ops.score_topk(U1, V1, None, 64, 1)
    i1, v1, _ = ops.score_topk_tc(U1, V1, None, 64, 1)
    assert torch.equal(i0, i1) and torch.equal(v0, v1)
