"""wgmma scoring kernel: (1) raw accumulators equal a bf16-rounded matmul, (2) final lists and
scores are IDENTICAL to the exact CUDA-core kernel (the certification + re-check make the
tensor-core path exact), incl. masks, biases, ragged sizes and adversarial near-ties, and lie
within the fp32 rounding bound of the fp64 oracle.  The d sweep reaches every padded-K build
of the kernel, with and without the item bias."""
import numpy as np
import pytest
import torch

from elliot_b200 import ops
from oracle.topk_bound import check_topk_fp64

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32_UNIT = 2.0 ** -24

# the padded K values that have CTA-pair and users-in-registers builds; elsewhere those switches run the default kernel
VARIANT_KP = (64, 80, 128, 144)


def _expected_kp(d, has_bias):
    """the padded K the kernel is built for (tc_layout): d, plus the bias as two bf16 columns when they fit, rounded up to
    the MMA's K = 16, and a 48-column tail rounded up to a full 64-column block"""
    fold = has_bias and d + 2 <= 256
    kp = (d + 2 * fold + 15) // 16 * 16
    return kp + 16 if kp % 64 == 48 else kp


# every padded K from 16 to 256 without bias and with it (folded into the MMA up to d = 254, added in the epilogue above)
SWEEP = ([(d, False) for d in (1, 17, 32, 33, 65, 90, 112, 129, 150, 176, 200, 224, 255)]
         + [(d, True) for d in (14, 30, 62, 64, 94, 100, 128, 158, 190, 206, 222, 254, 255, 256)])
SWEEP_IDS = [f"K{_expected_kp(d, b)}-d{d}-{'bias' if b else 'nobias'}" for d, b in SWEEP]


@pytest.fixture(autouse=True, params=[("2", "0", "0"), ("1", "0", "0"), ("2", "1", "0"), ("2", "0", "1")],
                ids=["two_epilogue_groups", "one_epilogue_group", "cta_pairs", "users_in_tmem"])
def _kernel_variant(request, monkeypatch):
    """every test runs against the four kernels: two consumer warpgroups, one (EB_TC_NG=1), CTA pairs sharing each item
    tile through TMA multicast (EB_TC_PAIR=1), and the user block held in registers as the wgmma A operand (EB_TC_ATM=1;
    the id keeps its historical name).  Tests parametrized over (d, bias) skip the last two where K has no such build (the
    fixed-shape tests keep all four ids, as before)."""
    p = request.node.callspec.params
    if request.param[1:] != ("0", "0") and "bias" in p and _expected_kp(p["d"], p["bias"]) not in VARIANT_KP:
        pytest.skip(f"no CTA-pair / users-in-registers build at K = {_expected_kp(p['d'], p['bias'])}")
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


def _check_fp64(U, V, b, d, k, mp, mi, users, idx, val):
    """the fp32 lists against the fp64 oracle on the same tables (oracle/topk_bound.py); returns (qualified, filled) ranks"""
    cpu = lambda t: None if t is None else t.cpu().numpy()
    return check_topk_fp64(cpu(U), cpu(V), cpu(b), d, k, cpu(mp), cpu(mi), users, cpu(idx), cpu(val), F32_UNIT)


def _accumulators_equal_bf16_matmul(d, bias, nu, ni):
    """the instrumented build's dense dump: bf16(u) . bf16(v), plus the two folded bias columns hi = bf16(b) and
    lo = bf16(b - hi) when the bias travels through the MMA (without folding the epilogue adds it after the dump)"""
    U, V, b = _tables(nu, ni, d, seed=d, bias=bias)
    _, _, st = ops.score_topk_tc(U, V, b, d, 10, dump=True)
    assert st["kp"] == _expected_kp(d, bias)
    ref = U[:, :d].bfloat16().double() @ V[:, :d].bfloat16().double().T
    if bias and d + 2 <= 256:
        hi = b.bfloat16()
        lo = (b - hi.float()).bfloat16()               # b - hi is exact in fp32
        ref += (hi.double() + lo.double())[None, :]
    got = st["dump"].double()
    assert torch.isfinite(got).all()
    # bf16 products are exact in fp32; only the fp32 accumulation order differs
    assert (got - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item()) + 1e-6


@pytest.mark.parametrize("d,nu,ni", [(64, 300, 1000), (128, 130, 700), (10, 257, 513), (200, 128, 300), (256, 64, 129)])
def test_accumulators_equal_bf16_matmul(d, nu, ni):
    _accumulators_equal_bf16_matmul(d, False, nu, ni)


@pytest.mark.parametrize("d,bias", SWEEP, ids=SWEEP_IDS)
def test_accumulators_equal_bf16_matmul_every_k(d, bias):
    _accumulators_equal_bf16_matmul(d, bias, 300, 700 + d)


def _tc_lists_identical_to_exact_kernel(d, bias, nu, ni, k):
    U, V, b = _tables(nu, ni, d, seed=7 * d + 1, bias=bias)
    mp, mi = _mask(nu, ni, 40, seed=d)
    i0, v0 = ops.score_topk(U, V, b, d, k, mp, mi)
    i1, v1, st = ops.score_topk_tc(U, V, b, d, k, mp, mi)
    torch.cuda.synchronize()
    assert st["kp"] == _expected_kp(d, bias)
    assert torch.equal(i0, i1), (st, (i0 != i1).sum().item())
    assert torch.equal(v0, v1)                       # same fp32 summation order -> bit-identical scores
    assert st["rechecked"] < nu * 0.2, st            # the bound certifies the bulk on random data
    q, n = _check_fp64(U, V, b, d, k, mp, mi, np.arange(nu), i1, v1)
    assert q >= 0.9 * n, (q, n)


@pytest.mark.parametrize("d,nu,ni,k", [(64, 1000, 5000, 10), (128, 300, 3000, 10), (10, 500, 777, 5), (96, 129, 2049, 16),
                                      (256, 200, 1500, 10)])
def test_tc_lists_identical_to_exact_kernel(d, nu, ni, k):
    _tc_lists_identical_to_exact_kernel(d, True, nu, ni, k)


@pytest.mark.parametrize("d,bias", SWEEP, ids=SWEEP_IDS)
def test_tc_lists_identical_to_exact_kernel_every_k(d, bias):
    _tc_lists_identical_to_exact_kernel(d, bias, 300, 1500 + 3 * d, 16 if bias else 10)


# K = 32 (a 32-column tail and no full block), 80 (a 16-column tail; all four kernels) and 160 (32-item tiles)
EDGE = [(30, True), (64, True), (150, False)]


@pytest.mark.parametrize("ni_of", ["1", "BN-1", "BN", "BN+1", "9BN+1"])
@pytest.mark.parametrize("d,bias", EDGE, ids=[f"K{_expected_kp(d, b)}" for d, b in EDGE])
def test_tc_tile_and_block_edges(d, bias, ni_of):
    """Catalogues of one item, one tile +- 1 and nine tiles + 1 (the four-stage ring wraps with two consumer groups), user
    ranges of 1 (the CTA pair's second block is empty), 127, 128 and 129 starting past user 0 with a train mask (the mask
    cache is addressed from the first selected user), k = 1 and 16.  Half the users rank copies of one
    item row first, so exact ties cross rank k and the lower index must win; one user keeps 3 candidates and one none."""
    kp = _expected_kp(d, bias)
    bn = 64 if kp <= 128 else 32
    ni = {"1": 1, "BN-1": bn - 1, "BN": bn, "BN+1": bn + 1, "9BN+1": 9 * bn + 1}[ni_of]
    ub, nsel_max = 37, 129
    nu = ub + nsel_max
    U, V, b = _tables(nu, ni, d, seed=kp + ni, bias=bias)
    U[::2, 0] = 1.0
    dup = torch.arange(2, max(2, ni), max(1, ni // 20), device=DEV)[:20]   # spread over the tiles and both consumer groups
    if len(dup):
        V[dup, :d] = V[dup[0], :d].clone()
        V[dup, 0] = 0.5
        if bias:
            b[dup] = b[dup[0]].item()
    rs = np.random.RandomState(ni)
    rows = []
    for u in range(nu):
        q = u - ub
        if q == 126:                                   # 3 candidates
            keep = rs.choice(ni, size=min(3, ni), replace=False)
            rows.append(np.setdiff1d(np.arange(ni), keep))
        elif q == 128:                                 # everything masked
            rows.append(np.arange(ni))
        elif q == 5:                                   # no train items
            rows.append(np.zeros(0, np.int64))
        else:
            rows.append(np.sort(rs.choice(ni, size=rs.randint(0, ni // 4 + 1), replace=False)))
    indptr = np.zeros(nu + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    mp = torch.from_numpy(indptr).to(DEV)
    mi = torch.from_numpy(np.concatenate(rows).astype(np.int32)).to(DEV)
    qual = filled = 0
    for n_sel in (1, 127, 128, 129):
        for k in (1, 16):
            i0, v0 = ops.score_topk(U, V, b, d, k, mp, mi, user_begin=ub, n_sel=n_sel)
            i1, v1, st = ops.score_topk_tc(U, V, b, d, k, mp, mi, user_begin=ub, n_sel=n_sel)
            assert st["kp"] == kp
            assert torch.equal(i0, i1), (n_sel, k, st, (i0 != i1).sum().item())
            assert torch.equal(v0, v1), (n_sel, k)
            q, n = _check_fp64(U, V, b, d, k, mp, mi, ub + np.arange(n_sel), i1, v1)
            qual, filled = qual + q, filled + n
            if n_sel == 129:
                assert (i1[128] == -1).all() and torch.isneginf(v1[128]).all()
                assert (i1[126, min(3, ni):] == -1).all() and torch.isneginf(v1[126, min(3, ni):]).all()
    assert qual >= 0.9 * filled, (qual, filled)


@pytest.mark.parametrize("d,bias", EDGE, ids=[f"K{_expected_kp(d, b)}" for d, b in EDGE])
def test_tc_several_user_blocks_per_cta(d, bias):
    """More user blocks than CTAs (as at catalogue scale): every CTA loads a new user block, resets its candidate buffers
    and refills its mask cache three or four times."""
    sms, _ = ops.device_info()
    nu, ni, k = 3 * sms * 128 + 77, 700, 10
    U, V, b = _tables(nu, ni, d, seed=d + 5, bias=bias)
    mp, mi = _mask(nu, ni, 20, seed=d)
    i0, v0 = ops.score_topk(U, V, b, d, k, mp, mi)
    i1, v1, st = ops.score_topk_tc(U, V, b, d, k, mp, mi)
    assert st["kp"] == _expected_kp(d, bias)
    assert torch.equal(i0, i1), (st, (i0 != i1).sum().item())
    assert torch.equal(v0, v1)
    assert st["rechecked"] < nu * 0.2, st


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
