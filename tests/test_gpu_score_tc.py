"""wgmma scoring kernel: (1) raw accumulators equal a bf16-rounded matmul, (2) final lists and
scores are IDENTICAL to the exact CUDA-core kernel (the certification + re-check make the
tensor-core path exact), incl. masks, biases, ragged sizes and adversarial near-ties."""
import numpy as np
import pytest
import torch

from elliot_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True, params=[("2", "0", "0"), ("1", "0", "0"), ("2", "1", "0"), ("2", "0", "1")],
                ids=["two_epilogue_groups", "one_epilogue_group", "cta_pairs", "users_in_tmem"])
def _kernel_variant(request, monkeypatch):
    """every test runs against the four kernels: two consumer warpgroups, one (EB_TC_NG=1), CTA pairs sharing each item
    tile through TMA multicast (EB_TC_PAIR=1), and the user block held in registers as the wgmma A operand (EB_TC_ATM=1;
    the id keeps its historical name)"""
    monkeypatch.setenv("EB_TC_NG", request.param[0])
    monkeypatch.setenv("EB_TC_PAIR", request.param[1])
    monkeypatch.setenv("EB_TC_ATM", request.param[2])


def _tables(nu, ni, d, seed, scale=0.1, bias=True):
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    ld = ops.padded_dim(d)
    U = torch.zeros((nu, ld), device=DEV); V = torch.zeros((ni, ld), device=DEV)
    U[:, :d] = torch.randn(nu, d, device=DEV, generator=g) * scale
    V[:, :d] = torch.randn(ni, d, device=DEV, generator=g) * scale
    b = (torch.randn(ni, device=DEV, generator=g) * 0.05) if bias else None
    return U, V, b


def _mask(nu, ni, per, seed):
    rs = np.random.RandomState(seed)
    rows = [np.sort(rs.choice(ni, size=min(ni - 1, rs.randint(0, 2 * per + 1)), replace=False)).astype(np.int32) for _ in range(nu)]
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    return torch.from_numpy(indptr).to(DEV), torch.from_numpy(np.concatenate(rows) if indptr[-1] else np.zeros(0, np.int32)).to(DEV)


@pytest.mark.parametrize("d,nu,ni", [(64, 300, 1000), (128, 130, 700), (10, 257, 513), (200, 128, 300), (256, 64, 129)])
def test_accumulators_equal_bf16_matmul(d, nu, ni):
    U, V, _ = _tables(nu, ni, d, seed=d)
    _, _, st = ops.score_topk_tc(U, V, None, d, 10, dump=True)
    ref = (U[:, :d].bfloat16().double() @ V[:, :d].bfloat16().double().T)
    got = st["dump"].double()
    assert torch.isfinite(got).all()
    # bf16 products are exact in fp32; only the fp32 accumulation order differs
    assert (got - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item()) + 1e-6


@pytest.mark.parametrize("d,nu,ni,k", [(64, 1000, 5000, 10), (128, 300, 3000, 10), (10, 500, 777, 5), (96, 129, 2049, 16),
                                      (256, 200, 1500, 10)])
def test_tc_lists_identical_to_exact_kernel(d, nu, ni, k):
    U, V, b = _tables(nu, ni, d, seed=7 * d + 1)
    mp, mi = _mask(nu, ni, 40, seed=d)
    i0, v0 = ops.score_topk(U, V, b, d, k, mp, mi)
    i1, v1, st = ops.score_topk_tc(U, V, b, d, k, mp, mi)
    torch.cuda.synchronize()
    assert torch.equal(i0, i1), (st, (i0 != i1).sum().item())
    assert torch.equal(v0, v1)                       # same fp32 summation order -> bit-identical scores
    assert st["rechecked"] < nu * 0.2, st            # the bound certifies the bulk on random data


def test_tc_user_range_no_mask_no_bias():
    U, V, _ = _tables(700, 4000, 64, seed=3, bias=False)
    i0, v0 = ops.score_topk(U, V, None, 64, 10, user_begin=100, n_sel=333)
    i1, v1, st = ops.score_topk_tc(U, V, None, 64, 10, user_begin=100, n_sel=333)
    assert torch.equal(i0, i1) and torch.equal(v0, v1)


def test_tc_adversarial_near_ties_fall_back_to_exact():
    """Items that differ by less than the bf16 bound around rank k: the kernel must refuse to
    certify those users and the re-check must still deliver the exact list."""
    nu, ni, d, k = 256, 2000, 64, 10
    U, V, _ = _tables(nu, ni, d, seed=11, bias=False)
    # 200 near-duplicates of item 0 (relative perturbation 1e-4 << 2^-8)
    g = torch.Generator(device=DEV); g.manual_seed(5)
    V[1:201, :d] = V[0, :d] * (1 + 1e-4 * torch.randn(200, d, device=DEV, generator=g))
    V[:201] *= 4.0                                    # make the cluster dominate every user's top ranks half of the time
    i0, v0 = ops.score_topk(U, V, None, d, k)
    i1, v1, st = ops.score_topk_tc(U, V, None, d, k)
    assert st["rechecked"] > 0
    assert torch.equal(i0, i1) and torch.equal(v0, v1)


@pytest.mark.parametrize("nu,ndup,why", [(6000, 200, "more flagged users than the re-check filter's row capacity"),
                                         (140, 1500, "more near-ties above the bound than one re-check list holds")])
def test_tc_recheck_overflow_paths_stay_exact(nu, ndup, why):
    """The re-check spreads the items over the grid and keeps short per-user lists; users it cannot hold (too many flagged
    users, too many items above the bound) must still come out exact through the row-per-CTA kernel."""
    ni, d, k = 4000, 64, 10
    U, V, b = _tables(nu, ni, d, seed=13)
    g = torch.Generator(device=DEV); g.manual_seed(6)
    V[1:ndup + 1, :d] = V[0, :d] * (1 + 1e-4 * torch.randn(ndup, d, device=DEV, generator=g))
    V[:ndup + 1] *= 4.0
    b[:ndup + 1] = 0.0
    mp, mi = _mask(nu, ni, 20, seed=3)
    i0, v0 = ops.score_topk(U, V, b, d, k, mp, mi)
    i1, v1, st = ops.score_topk_tc(U, V, b, d, k, mp, mi)
    assert st["rechecked"] > (1024 if ndup == 200 else 10), (why, st)
    assert torch.equal(i0, i1) and torch.equal(v0, v1), why


def test_tc_heavy_mask_and_short_lists():
    """Users who own almost everything: fewer than k candidates, -1/-inf padding as the exact kernel."""
    nu, ni, d, k = 130, 600, 64, 10
    U, V, b = _tables(nu, ni, d, seed=21)
    rows = []
    rs = np.random.RandomState(0)
    for u in range(nu):
        keep = rs.choice(ni, size=(3 if u % 3 == 0 else 50), replace=False)
        rows.append(np.setdiff1d(np.arange(ni), keep).astype(np.int32))
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    mp = torch.from_numpy(indptr).to(DEV); mi = torch.from_numpy(np.concatenate(rows)).to(DEV)
    i0, v0 = ops.score_topk(U, V, b, d, k, mp, mi)
    i1, v1, st = ops.score_topk_tc(U, V, b, d, k, mp, mi)
    assert torch.equal(i0, i1) and torch.equal(v0, v1)
    assert (i1[0, 3:] == -1).all() and torch.isinf(v1[0, 3:]).all()


def test_tc_rejects_long_lists():
    from elliot_b200._lib import EbError
    U, V, _ = _tables(10, 100, 64, seed=1, bias=False)
    with pytest.raises(EbError):
        ops.score_topk_tc(U, V, None, 64, 17)
