"""The fp32 training kernels that share the BPR step's shape (a row-stride or lane-group template, warp row gathers, a dot
product, vector-atomic scatters), each against an fp64 computation of the same operation at every compiled build:

  A. bpr_batch_grad_kernel<DP> (BPRMF_batch): the gradient tables and the loss read straight after the kernel;
  B. the dense Keras Adam (eb_adam_dense_f32 / eb_adam_dense_copy_f32) of BPRMF_batch, GMF, NeuMF, MultiVAE and SVD++,
     with a grid-stride loop that wraps, a late step number and the bf16 copy;
  C. mf_hogwild_kernel<DP> (MF2020 throughput mode): the sample stream bit for bit against oracle/mf2020_hogwild.py, and
     the arithmetic of launches whose rows do not repeat (then nothing is racy: every sample reads the pre-launch rows);
  D. the SVD++ / FunkSVD lane groups G = 1 and 8 (f = 4, 20, 32) of the implicit mean, the fused step and the pair pass.

Every check is deterministic.  Tolerances are derived beside each assert, as in test_gpu_dense_model_kernels.py: with
U = 2^-24 the fp32 unit roundoff and gamma(n) = nU/(1-nU), an n-term fp32 sum or dot product in any order is within
gamma(n) sum |term| of the exact one, and so is an atomic sum of n contributions; the intrinsics (CUDA C Programming
Guide, intrinsic functions) are within __expf(x): 2 + floor(1.173 |x|) ulp, __logf(x): 2^-21.41 absolute on [0.5, 2],
__fdividef(x, y): 2 ulp for |y| in [2^-126, 2^126]; and sigma' <= 1/4 carries an error of sigma's argument.
One ulp of a fp32 value v is at most 2U |v|.
"""
import math

import numpy as np
import pytest
import torch

from elliot_b200 import ops
from oracle import mf2020_hogwild as hw
from oracle import rating_mf as rmf
from oracle import tf_models as tfm

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
ULP = 2 * U
LOGF_ABS = 2.0 ** -21.41


def gamma(n):
    n = np.asarray(n, dtype=np.float64)
    return n * U / (1 - n * U)


def expf_rel(x):
    """relative error bound of __expf(x)"""
    return (2 + np.floor(1.173 * np.abs(x))) * ULP


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def host(t):
    return t.double().cpu().numpy()


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def table(a, ld):
    """fp32 device table of the rows of `a`, row stride ld, padding columns zero"""
    t = torch.zeros((a.shape[0], ld), device=DEV)
    t[:, :a.shape[1]] = dev(a.astype(np.float32))
    return t


def scatter(n_rows, idx, terms, errs):
    """(fp64 sum of `terms` into rows `idx`, bound of the fp32 atomic sum of their computed values): the computed terms
    are within errs of terms, and c atomic additions into a row add gamma(c) times the sum of their magnitudes."""
    shape = (n_rows,) + terms.shape[1:]
    S, A, E = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    np.add.at(S, idx, terms); np.add.at(A, idx, np.abs(terms) + errs); np.add.at(E, idx, errs)
    c = np.bincount(idx, minlength=n_rows).reshape((n_rows,) + (1,) * (terms.ndim - 1))
    return S, E + gamma(c) * A


# ======================================================================================== A. BPRMF_batch gradient
L_W, L_B = 0.125, 0.0625                      # exact in fp32: the kernel and the reference use the same values


def bpr_batch_reference(Gu, Gi, Bi, u, i, j, l_w, l_b):
    """fp64 (loss, dGu, dGi, dBi) of oracle.tf_models and their bounds for the fp32 kernel."""
    loss, dGu, dGi, dBi = tfm.bprmf_batch_loss_and_grads(Gu, Gi, Bi, u, i, j, l_w, l_b)
    d = Gu.shape[1]
    gu, gp, gn, bp, bn = Gu[u], Gi[i], Gi[j], Bi[i], Bi[j]
    raw = (bp + (gu * gp).sum(1)) - (bn + (gu * gn).sum(1))
    # two d-term dots, each plus a bias, then their difference: d + 2 roundings on every chain
    e_raw = gamma(d + 2) * (np.abs(bp) + np.abs(bn) + np.abs(gu * gp).sum(1) + np.abs(gu * gn).sum(1))
    diff = np.clip(raw, -80.0, 1e8)
    open_ = (raw > -80.0) & (raw < 1e8)
    sg = 1 / (1 + np.exp(diff))
    # sigmoid(-diff): sigma' <= 1/4 carries e_raw; __expf's relative error r moves sg by sg (1 - sg) r; 1 + E and the
    # division round once each
    e_g = np.where(open_, e_raw / 4 + sg * (1 - sg) * expf_rel(diff) + 2 * U * sg, 0.0)
    g = np.where(open_, -sg, 0.0)[:, None]
    e_g2 = e_g[:, None]
    # each table term: one difference, two products and one sum (4 roundings), plus e_g times its gradient factor
    tu = g * (gp - gn) + l_w * gu
    eu = e_g2 * np.abs(gp - gn) + gamma(4) * (np.abs(g * (gp - gn)) + l_w * np.abs(gu))
    ti, tj = g * gu + l_w * gp, -g * gu + l_w * gn
    ei = e_g2 * np.abs(gu) + gamma(3) * (np.abs(g * gu) + l_w * np.abs(gp))
    ej = e_g2 * np.abs(gu) + gamma(3) * (np.abs(g * gu) + l_w * np.abs(gn))
    _, bu_ = scatter(Gu.shape[0], u, tu, eu)
    _, bi_ = scatter(Gi.shape[0], np.r_[i, j], np.r_[ti, tj], np.r_[ei, ej])
    tb = np.r_[g[:, 0] + l_b * bp, -g[:, 0] + 0.1 * l_b * bn]
    # 0.1f differs from 0.1 by 1.5e-8 relative, below U
    eb = np.r_[e_g, e_g] + gamma(3) * (np.abs(np.r_[g[:, 0], g[:, 0]]) + l_b * np.abs(np.r_[bp, 0.1 * bn]))
    _, bb_ = scatter(Bi.shape[0], np.r_[i, j], tb, eb)
    # loss term: softplus(-diff) (Lipschitz 1 in diff; __expf(-|diff|) = E off by r E, which moves log(1 + E) by at most
    # r E / (1 + E); 1 + E rounds; __logf on [1, 2]) plus the three regularisers (sq: a 3d-term sum of squares)
    E = np.exp(-np.abs(diff))
    sq = (gu ** 2).sum(1) + (gp ** 2).sum(1) + (gn ** 2).sum(1)
    term = tfm.softplus(-diff) + 0.5 * l_w * sq + 0.5 * l_b * bp ** 2 + 0.05 * l_b * bn ** 2
    e_term = (e_raw + expf_rel(diff) * E / (1 + E) + U + LOGF_ABS + 0.5 * l_w * gamma(3 * d) * sq
              + gamma(6) * np.abs(term))
    # per-lane fp32 sums, a warp tree and fp64 atomics: at most B fp32 additions on any chain
    e_loss = e_term.sum() + gamma(len(u)) * (np.abs(term) + e_term).sum()
    return loss, dGu, dGi, dBi, bu_, bi_, bb_, e_loss


def _bpr_batch_tables(rs, nu, ni, d, ld):
    Gu, Gi = f32(rs.uniform(-0.4, 0.4, (nu, d))), f32(rs.uniform(-0.4, 0.4, (ni, d)))
    Bi = f32(rs.normal(0, 0.1, ni))
    nb = (ni + 3) // 4 * 4 + 4                               # dBi[ni:] is padding the kernel must not touch
    Bid = torch.zeros(nb, device=DEV); Bid[:ni] = dev(Bi.astype(np.float32))
    return Gu, Gi, Bi, table(Gu, ld), table(Gi, ld), Bid


def _bpr_batches(rs, nu, ni):
    """(name, u, i, j): tiny id ranges (every row dozens of times), all-distinct rows, partial tiles, an empty batch"""
    out = []
    k = min(nu, 7)
    u = rs.randint(0, k, 600); i = rs.randint(0, 9, 600); j = (i + 1 + rs.randint(0, 8, 600)) % 9
    out.append(("tiny_ids", u, i, j))
    B = min(nu, ni // 2, 1500)
    it = rs.permutation(ni)[:2 * B]
    out.append(("distinct", rs.permutation(nu)[:B], it[:B], it[B:]))
    for B in (1, 31, 33, 4097, 0):
        i = rs.randint(0, ni, B); out.append((f"B{B}", rs.randint(0, nu, B), i, (i + 1 + rs.randint(0, ni - 1, B)) % ni))
    return [(n, *(a.astype(np.int32) for a in t)) for n, *t in out]


@pytest.mark.parametrize("d, ld", [(5, 8), (16, 16), (30, 32), (64, 64), (100, 128), (256, 256), (5, 64)])
def test_bpr_batch_gradient_matches_fp64(d, ld):
    """Every row-stride build (VPL = 2 at ld 256, G = 2 at ld 8), d < ld and d = ld, and d = 5 at ld = 64 where most of
    the row is padding.  The gradient is read straight after the kernel: no Adam step hides its scale."""
    assert ops.padded_dim(d) <= ld
    rs = np.random.RandomState(d + ld)
    nu, ni = 3000, 4000
    Gu, Gi, Bi, Gud, Gid, Bid = _bpr_batch_tables(rs, nu, ni, d, ld)
    for name, u, i, j in _bpr_batches(rs, nu, ni):
        dGu, dGi, dBi = torch.zeros_like(Gud), torch.zeros_like(Gid), torch.zeros_like(Bid)
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        args = (Gud, Gid, Bid, dGu, dGi, dBi, d, dev(u), dev(i), dev(j), L_W, L_B)
        ops.bpr_batch_grad_f32(*args, loss=loss)
        first = [host(t) for t in (dGu, dGi, dBi)]
        if len(u) == 0:
            assert not dGu.any() and not dGi.any() and not dBi.any() and loss.item() == 0.0, name
            continue
        lref, rGu, rGi, rBi, bGu, bGi, bBi, e_loss = bpr_batch_reference(Gu, Gi, Bi, u, i, j, L_W, L_B)
        assert abs(loss.item() - lref) <= e_loss, (name, loss.item(), lref, e_loss)
        for got, want, bound, what in ((first[0][:, :d], rGu, bGu, "dGu"), (first[1][:, :d], rGi, bGi, "dGi"),
                                       (first[2][:len(Bi)], rBi, bBi, "dBi")):
            err = np.abs(got - want)
            assert (err <= bound).all(), (name, what, err.max(), bound[err > bound][:4])
        # structure, exactly: padding columns, rows no triple touches and dBi's tail stay 0
        assert not first[0][:, d:].any() and not first[1][:, d:].any() and not first[2][len(Bi):].any(), name
        assert not first[0][np.setdiff1d(np.arange(nu), u)].any(), name
        assert not first[1][np.setdiff1d(np.arange(ni), np.r_[i, j])].any(), name
        # a second call adds to the tables (the model relies on Adam to clear them): twice the first, bit for bit where
        # each row has one contribution, else within two atomic sums of the same terms
        ops.bpr_batch_grad_f32(*args)
        for t, f, bound in ((dGu, first[0], bGu), (dGi, first[1], bGi), (dBi, first[2], bBi)):
            got = host(t)
            if name == "distinct":
                assert np.array_equal(got, 2 * f), name
                continue
            w = bound.shape[0]
            live = (slice(0, w), slice(0, d)) if got.ndim == 2 else (slice(0, w),)
            assert (np.abs(got[live] - 2 * f[live]) <= 4 * bound).all(), name
            assert not (got[:, d:].any() if got.ndim == 2 else got[w:].any()), name


@pytest.mark.parametrize("d", [5, 64, 256])
def test_bpr_batch_clipped_triples(d):
    """raw < -80 and raw > 1e8 fall outside clip_by_value's open interval: zero gradient through the sigmoid, loss
    softplus(80) and 0.  (TF 2.x builds clip_by_value from minimum / maximum, whose gradients may pass at exact
    equality with the bound; the kernel and oracle/tf_models.py use the open interval.  That detail is not pinned against
    TensorFlow, which cannot run here; no triple below sits on a bound.)"""
    ld = ops.padded_dim(d)
    Gi = np.zeros((4, d)); Gi[0] = 0.5; Gi[1] = -0.5
    Gu = np.zeros((2, d)); Gu[0] = -200.0 / d; Gu[1] = 2e8 / d      # raw = -200 (user 0) and +2e8 (user 1) on (0, 1)
    Gu, Gi, Bi = f32(Gu), f32(Gi), np.zeros(4)
    u, i, j = (np.array(a, np.int32) for a in ([0, 1], [0, 0], [1, 1]))
    Gud, Gid = table(Gu, ld), table(Gi, ld)
    Bid = torch.zeros(8, device=DEV)
    dGu, dGi, dBi = torch.zeros_like(Gud), torch.zeros_like(Gid), torch.zeros_like(Bid)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.bpr_batch_grad_f32(Gud, Gid, Bid, dGu, dGi, dBi, d, dev(u), dev(i), dev(j), 0.0, 0.0, loss=loss)
    assert not dGu.any() and not dGi.any() and not dBi.any()
    # softplus(80) = 80 + log1p(e^-80): fmaxf exact, __logf(1 + __expf(-80)) within 2^-21.41 of 0, one fp32 sum
    want = 80.0 + math.log1p(math.exp(-80.0))
    assert abs(loss.item() - want) <= 2 * LOGF_ABS + 4 * U * want, loss.item()
    # with the regularisers on, the clipped triple's gradient is the regulariser's alone
    ops.bpr_batch_grad_f32(Gud, Gid, Bid, dGu, dGi, dBi, d, dev(u[:1]), dev(i[:1]), dev(j[:1]), L_W, L_B)
    _, rGu, rGi, rBi = tfm.bprmf_batch_loss_and_grads(Gu, Gi, Bi, u[:1], i[:1], j[:1], L_W, L_B)
    assert np.array_equal(host(dGu)[:, :d], f32(rGu)) and np.array_equal(host(dGi)[:, :d], f32(rGi))
    assert np.array_equal(host(dBi)[:4], rBi)


# ======================================================================================== B. Keras Adam
B1, B2, EPS, LR = (float(np.float32(x)) for x in (0.9, 0.999, 1e-7, 1e-3))   # the fp32 values the kernel receives


def adam_bounds(x0, m0, v0, g, step):
    """fp64 Keras Adam (oracle KerasAdam) of one step from the device's fp32 state, and its bounds for the kernel."""
    opt = tfm.KerasAdam(LR, B1, B2, EPS)
    opt.t = step - 1
    opt.begin_step()
    m, v, x = m0.copy(), v0.copy(), x0.copy()
    opt.state["x"] = (m, v)
    opt.apply("x", x, g)
    c1, c2 = 1 - B1, 1 - B2                               # exact in fp32 too (Sterbenz)
    em = gamma(2) * (B1 * np.abs(m0) + c1 * np.abs(g))    # b1 m + c1 g: two products, one sum
    ev = gamma(3) * (B2 * v0 + c2 * g * g)               # b2 v + (c1 g) g: three products, one sum
    lr_t = LR * math.sqrt(1 - B2 ** step) / (1 - B1 ** step)
    den = np.sqrt(v) + EPS
    q = lr_t * m / den
    dv_rel = np.where(v > 0, (np.sqrt(v + ev) - np.sqrt(v)) / den, np.sqrt(ev) / den)
    # lr_t rounded to fp32, the product, sqrtf, + eps and the division: 5 roundings; then the fp32 subtraction
    eq = lr_t * em / den + np.abs(q) * (dv_rel + gamma(6))
    ex = eq + U * np.abs(x)
    return x, m, v, ex, em, ev


def _adam_step(var, m, v, grad, step, copy):
    n = var.numel()
    if copy is None:
        ops.adam_dense_f32(var, m, v, grad, LR, step, B1, B2, EPS)
    else:
        ops._call("eb_adam_dense_copy_f32", var, ops._ptr(var), ops._ptr(m), ops._ptr(v), ops._ptr(grad), n, LR, B1, B2, EPS,
                  step, ops._ptr(copy))


@pytest.mark.parametrize("copy", [False, True], ids=["plain", "bf16_copy"])
@pytest.mark.parametrize("n", [4, 3 * 2 ** 20 + 4])
def test_keras_adam_matches_fp64(n, copy):
    """Five consecutive steps, then step 1000 (where the fp64 bias correction lr_t matters), each against fp64 Keras Adam
    from the kernel's own state.  At n = 3 2^20 + 4 the grid (sm_count 8 blocks of 256 float4 threads) wraps.  A third of
    the gradient is exactly 0: those entries still decay m and v and move, as TF's sparse apply does."""
    rs = np.random.RandomState(n % 97)
    var = dev(rs.normal(0, 0.1, n).astype(np.float32))
    m, v = torch.zeros_like(var), torch.zeros_like(var)
    cp = torch.full((n,), 3.0, dtype=torch.bfloat16, device=DEV) if copy else None
    moved_at_zero = 0
    for step in (1, 2, 3, 4, 5, 1000):
        g = f32(rs.normal(0, 1, n) * 10.0 ** rs.uniform(-6, 1, n))            # magnitudes 1e-6 .. 10: v near eps^2 too
        g[rs.rand(n) < 1 / 3] = 0.0
        g[:2] = 0.0
        x0, m0, v0 = host(var), host(m), host(v)
        grad = dev(g.astype(np.float32))
        _adam_step(var, m, v, grad, step, cp)
        x, mr, vr, ex, em, ev = adam_bounds(x0, m0, v0, g, step)
        for got, want, bound, what in ((host(m), mr, em, "m"), (host(v), vr, ev, "v"), (host(var), x, ex, "var")):
            err = np.abs(got - want)
            assert (err <= bound).all(), (step, what, err.max(), np.argmax(err - bound))
        assert not grad.any()                                                  # the gradient is cleared
        zero = (g == 0) & (m0 != 0)
        moved_at_zero += int((host(var)[zero] != x0[zero]).sum())
        if copy:
            # each bf16 is round-to-nearest-even of the fp32 weight just written, bit for bit
            assert torch.equal(cp.view(torch.int16), var.to(torch.bfloat16).view(torch.int16)), step
    assert moved_at_zero > 0


# ======================================================================================== C. MF2020 Hogwild launch
def _mf_call(T, d, pos_u, pos_i, m, n_items, seed, epoch, lr, reg, first, count, out=None, loss=None):
    ops.mf_pointwise_step_f32(T["U"], T["V"], T["ub"], T["ib"], T["gb"], d, pos_u, pos_i, m, n_items, seed, epoch, lr, reg,
                              loss=loss, out=out, first=first, count=count)


def _mf_tables(rs, n_users, n_items, d, ld, scale=0.3):
    T = {"U": table(rs.normal(0, scale, (n_users, d)), ld), "V": table(rs.normal(0, scale, (n_items, d)), ld),
         "ub": dev(rs.normal(0, 0.3, n_users).astype(np.float32)), "ib": dev(rs.normal(0, 0.3, n_items).astype(np.float32)),
         "gb": torch.full((1,), 0.2, device=DEV)}
    return T


@pytest.mark.parametrize("ld", ops.F32_STRIDES)
def test_mf_hogwild_stream_is_the_restatement(ld):
    """`out` holds the restated (user, item, label) of every position for two epochs, and a first / count window
    writes exactly its positions."""
    rs = np.random.RandomState(ld)
    n_users, n_items, m, seed = 300, 997, 3, 0x5EED + ld
    pos_u = np.sort(rs.randint(0, n_users, 5000)).astype(np.int32)
    pos_i = rs.randint(0, n_items, 5000).astype(np.int32)
    n = len(pos_u) * (1 + m)
    T = _mf_tables(rs, n_users, n_items, ld, ld)
    pu, pi = dev(pos_u), dev(pos_i)
    out = tuple(torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3))
    for epoch in (0, 1):
        _mf_call(T, ld, pu, pi, m, n_items, seed, epoch, 0.0, 0.0, 0, None, out=out)
        want = hw.sample_stream(pos_u, pos_i, m, n_items, seed, epoch)
        for got, w in zip(out, want):
            assert np.array_equal(got.cpu().numpy(), w), epoch
    first, count = 1234, 777
    for t in out:
        t.fill_(-7)
    _mf_call(T, ld, pu, pi, m, n_items, seed, 1, 0.0, 0.0, first, count, out=out)
    want = hw.sample_stream(pos_u, pos_i, m, n_items, seed, 1, first, count)
    for got, w in zip(out, want):
        got = got.cpu().numpy()
        assert np.array_equal(got[first:first + count], w)
        assert (got[:first] == -7).all() and (got[first + count:] == -7).all()


def mf_launch_bounds(R, a, b, bu, bi, gb0, r, lr, reg, d):
    """Bounds of the fp32 kernel's per-sample results for the fp64 launch R = hw.apply_launch(...) (a, b: the samples'
    pre-launch rows, bu, bi: their biases)."""
    pred, sig, grad, du, dv = R["pred"], R["sig"], R["grad"], R["du"], R["dv"]
    # ((gb0 + bu) + bi) + a d-term dot
    e_pred = gamma(d + 3) * (abs(gb0) + np.abs(bu) + np.abs(bi) + np.abs(a * b).sum(1))
    # sigma' <= 1/4 carries e_pred; __expf's relative error moves sig by sig (1 - sig) r; 1 + e rounds; __fdividef 2 ulp
    e_sig = e_pred / 4 + sig * (1 - sig) * expf_rel(pred) + (U + 2 * ULP) * sig
    e_grad = (e_sig + U * np.abs(grad))[:, None]
    g2 = grad[:, None]
    # du = lr (grad b - reg a): a product, a product and a difference, times lr
    e_du = lr * e_grad * np.abs(b) + gamma(4) * lr * (np.abs(g2 * b) + reg * np.abs(a))
    w = a + du                                                   # the updated user row, rounded once more
    e_w = e_du + U * np.abs(w)
    e_dv = lr * (e_grad * np.abs(w) + np.abs(g2) * e_w + e_grad * e_w) + gamma(4) * lr * (np.abs(g2 * w) + reg * np.abs(b))
    e_b = lambda x: lr * e_grad[:, 0] + gamma(3) * lr * (np.abs(grad) + reg * np.abs(x))
    E = np.exp(-np.abs(pred))
    term = np.maximum(pred, 0) - r * pred + np.log1p(E)
    # the loss term is Lipschitz 1 in pred; log(1 + e) moves by r e / (1 + e) for __expf, U for 1 + e, 2^-21.41 for __logf
    e_term = e_pred + expf_rel(pred) * E / (1 + E) + U + LOGF_ABS + gamma(3) * (np.abs(pred) + np.log1p(E))
    c = len(pred)
    e_loss = e_term.sum() + gamma(c) * (np.abs(term) + e_term).sum()
    h = sig * (1 - sig)
    e_h = e_sig * np.abs(1 - 2 * sig) + e_sig ** 2 + gamma(2) * h
    e_gsum = e_grad.sum() + gamma(c) * (np.abs(grad) + e_grad[:, 0]).sum()
    e_hsum = e_h.sum() + gamma(c) * (h + e_h).sum()
    # the finish is monotone in gsum (positive gain) and in k = hsum / c + reg (the gain decreases): its extremes over the
    # box of the two sums are at the corners; it runs in fp64 and rounds once to fp32
    corners = [hw.global_bias_finish(gb0, R["gsum"] + s1 * e_gsum, max(R["hsum"] + s2 * e_hsum, 0.0), c, lr, reg)
               for s1 in (-1, 1) for s2 in (-1, 1)]
    e_gb = max(abs(x - R["gb"]) for x in corners) + U * abs(R["gb"]) + 1e-12
    return e_du, e_dv, e_b(bu), e_b(bi), e_loss, e_gb


def _mf_distinct_windows(u, i, W, k):
    """first positions of k consecutive windows of W samples in which no user row and no item row repeats"""
    ok = [len(np.unique(u[s:s + W])) == W and len(np.unique(i[s:s + W])) == W for s in range(0, len(u) - W + 1, W)]
    for s in range(len(ok) - k + 1):
        if all(ok[s:s + k]):
            return [(s + q) * W for q in range(k)]
    raise AssertionError("no window without repeated rows")


def _mf_check_launch(T, snap, idx_u, idx_i, u, i, r, d, lr, reg, loss_got=None, checked_u=None, checked_i=None):
    """Compare the device tables after one launch with hw.apply_launch from the pre-launch state `snap` (fp64 host rows
    of the touched rows, by sample), for the samples `checked` (all when None)."""
    R = hw.apply_launch(snap["U"], snap["V"], snap["ub"], snap["ib"], snap["gb"], idx_u, idx_i, r.astype(np.float64), lr, reg)
    a, b = snap["U"][idx_u], snap["V"][idx_i]
    e_du, e_dv, e_bu, e_bi, e_loss, e_gb = mf_launch_bounds(R, a, b, snap["ub"][idx_u], snap["ib"][idx_i], snap["gb"], r,
                                                            lr, reg, d)
    sel = np.arange(len(u)) if checked_u is None else checked_u
    # one atomic addition onto the pre-launch value: the term's error plus one rounding of the sum
    Ug, Vg = host(T["U"][dev(u[sel].astype(np.int64))]), host(T["V"][dev(i[sel].astype(np.int64))])
    for got, want, e, what in ((Ug[:, :d], R["U"][idx_u[sel]], e_du[sel], "U"), (Vg[:, :d], R["V"][idx_i[sel]], e_dv[sel], "V"),
                               (host(T["ub"])[u[sel]], R["ub"][idx_u[sel]], e_bu[sel], "ub"),
                               (host(T["ib"])[i[sel]], R["ib"][idx_i[sel]], e_bi[sel], "ib")):
        err = np.abs(got - want)
        assert (err <= e + U * np.abs(want)).all(), (what, err.max())
    assert not Ug[:, d:].any() and not Vg[:, d:].any()
    if checked_u is None:
        assert abs(loss_got - R["loss"]) <= e_loss, (loss_got, R["loss"], e_loss)
        assert abs(T["gb"].item() - R["gb"]) <= e_gb, (T["gb"].item(), R["gb"], e_gb)
    return len(sel)


def _mf_snapshot(T, u, i, d):
    """fp64 host copies of the rows the samples touch (sample order) and the global bias"""
    return {"U": host(T["U"][dev(u.astype(np.int64))])[:, :d], "V": host(T["V"][dev(i.astype(np.int64))])[:, :d],
            "ub": host(T["ub"])[u], "ib": host(T["ib"])[i], "gb": T["gb"].item()}


@pytest.mark.parametrize("d, ld", [(6, 8), (16, 16), (29, 32), (64, 64), (100, 128), (200, 256)])
def test_mf_hogwild_launch_matches_fp64(d, ld):
    """Two consecutive windows of 256 samples without repeated rows: every row update, the biases, the loss and the
    closed-form global bias against fp64, each window against its own closed form (a global-bias accumulator that is not
    reset between launches fails the second); rows outside the launch stay bit-identical, padding columns 0."""
    rs = np.random.RandomState(d)
    n_pos, n_items, m, W, seed, lr, reg = 50000, 60000, 1, 256, 77 + d, 0.1, 0.05
    pos_u = np.arange(n_pos, dtype=np.int32)                   # one positive per user: a user repeats only via its slots
    pos_i = rs.permutation(n_items)[:n_pos].astype(np.int32)
    T = _mf_tables(rs, n_pos, n_items, d, ld)
    pu, pi = dev(pos_u), dev(pos_i)
    su, si, sr = hw.sample_stream(pos_u, pos_i, m, n_items, seed, 0)
    firsts = _mf_distinct_windows(su, si, W, 2)
    for first in firsts:
        u, i, r = su[first:first + W], si[first:first + W], sr[first:first + W]
        snap = _mf_snapshot(T, u, i, d)
        before = {k: t.clone() for k, t in T.items()}
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        _mf_call(T, d, pu, pi, m, n_items, seed, 0, lr, reg, first, W, loss=loss)
        _mf_check_launch(T, snap, np.arange(W), np.arange(W), u, i, r, d, lr, reg, loss_got=loss.item())
        for k, rows in (("U", u), ("V", i), ("ub", u), ("ib", i)):
            keep = torch.ones(T[k].shape[0], dtype=torch.bool, device=DEV); keep[dev(rows.astype(np.int64))] = False
            assert torch.equal(T[k][keep], before[k][keep]), k                 # untouched rows: bit-identical
        assert not T["U"][:, d:].any() and not T["V"][:, d:].any()


def test_mf_hogwild_launch_with_repeated_rows():
    """A window where rows repeat: the samples whose user row and item row the window touches once read no other
    sample's write, so their rows are checked against fp64; the rest (racy by design) only stay finite."""
    rs = np.random.RandomState(5)
    d, ld, n_users, n_items, m, seed, lr, reg = 40, 64, 400, 500, 2, 9, 0.1, 0.05
    pos_u = np.sort(rs.randint(0, n_users, 3000)).astype(np.int32)
    pos_i = rs.randint(0, n_items, 3000).astype(np.int32)
    T = _mf_tables(rs, n_users, n_items, d, ld)
    first, W = 1000, 600
    u, i, r = hw.sample_stream(pos_u, pos_i, m, n_items, seed, 3, first, W)
    assert len(np.unique(u)) < W and len(np.unique(i)) < W
    once = (np.bincount(u, minlength=n_users)[u] == 1) & (np.bincount(i, minlength=n_items)[i] == 1)
    snap = _mf_snapshot(T, u, i, d)
    _mf_call(T, d, dev(pos_u), dev(pos_i), m, n_items, seed, 3, lr, reg, first, W)
    sel = np.flatnonzero(once)
    checked = _mf_check_launch(T, snap, np.arange(W), np.arange(W), u, i, r, d, lr, reg, checked_u=sel)
    assert checked == len(sel) >= 20, checked                  # how much was actually checked
    assert bool(torch.isfinite(T["U"]).all()) and bool(torch.isfinite(T["V"]).all())


# ======================================================================================== D. SVD++ / FunkSVD lane groups
# G = f/4 rounded up to a power of two: f = 4 -> G = 1, f = 20 and 32 -> G = 8; ld = f = 20 runs without padding
LANES = [(4, 8), (20, 32), (32, 32), (20, 20)]


def _rating_csr(nu, ni, seed):
    """sorted train rows: row 0 holds one item, row 1 most of the catalogue, the others 1 .. 60 items"""
    rs = np.random.RandomState(seed)
    rows = [np.sort(rs.choice(ni, size=rs.randint(1, 60), replace=False)) for _ in range(nu)]
    rows[0] = np.array([5])
    rows[1] = np.sort(rs.choice(ni, size=ni - 3, replace=False))
    indptr = np.r_[0, np.cumsum([len(x) for x in rows])].astype(np.int64)
    return indptr, np.concatenate(rows).astype(np.int32)


def _rating_tables(rs, nu, ni, f, ld):
    H = {"P": f32(rs.normal(0, 0.3, (nu, f))), "Q": f32(rs.normal(0, 0.3, (ni, f))), "Y": f32(rs.normal(0, 0.3, (ni, f))),
         "bu": f32(rs.normal(0, 0.2, nu)), "bi": f32(rs.normal(0, 0.2, ni)), "g": float(np.float32(0.31))}
    D = {k: table(H[k], ld) for k in ("P", "Q", "Y")}
    D["bu"] = dev(np.r_[H["bu"], np.zeros(4)].astype(np.float32)); D["bi"] = dev(np.r_[H["bi"], np.zeros(4)].astype(np.float32))
    D["g"] = torch.tensor([H["g"], 0, 0, 0], dtype=torch.float32, device=DEV)
    return H, D


def implicit_mean_bound(H, users, indptr, indices):
    """|Z - fp64| bound per element: an L-term fp32 sum, times fp32(1/L) (two roundings), plus P (one rounding)"""
    Z = rmf.implicit_means(H["P"], H["Y"], users, indptr, indices)
    S = np.stack([np.abs(H["Y"][indices[indptr[x]:indptr[x + 1]]]).sum(0) for x in users])
    L = (indptr[users + 1] - indptr[users])[:, None]
    return Z, gamma(L + 2) * S / L + U * np.abs(Z)


@pytest.mark.parametrize("f, ld", LANES)
def test_implicit_mean_lane_groups(f, ld):
    nu, ni = 300, 700
    indptr, indices = _rating_csr(nu, ni, f + ld)
    H, D = _rating_tables(np.random.RandomState(f), nu, ni, f, ld)
    users = np.r_[np.arange(nu), [1, 1, 0, 7, 7]].astype(np.int32)       # every user, repeats, the 1-item and long rows
    Z = ops.implicit_mean_f32(D["P"], D["Y"], f, dev(indptr), dev(indices), users=dev(users))
    want, bound = implicit_mean_bound(H, users, indptr, indices)
    err = np.abs(host(Z)[:, :f] - want)
    assert (err <= bound).all(), err.max()
    assert not Z[:, f:].any()


@pytest.mark.parametrize("implicit", [True, False], ids=["svdpp", "funk_svd"])
@pytest.mark.parametrize("f, ld", LANES)
def test_rating_step_lane_groups(f, ld, implicit):
    """The fused step against the fp64 restatement (oracle/rating_mf.py): loss, dP, dQ, dY, the biases and dg, per
    element, on a full batch with repeated users (the long and the 1-item rows) and a short last batch."""
    nu, ni = 400, 900
    indptr, indices = _rating_csr(nu, ni, 11 + f)
    H, D = _rating_tables(np.random.RandomState(f + ld), nu, ni, f, ld)
    T = {k: H[k] for k in (("P", "Q", "Y", "bu", "bi", "g") if implicit else ("P", "Q", "bu", "bi"))}
    gen = np.random.RandomState(f)
    ip, ix = dev(indptr), dev(indices)
    for B in (2048, 333):
        u = gen.randint(0, nu, B).astype(np.int32); u[:64] = 1; u[64:80] = 0
        it = gen.randint(0, ni, B).astype(np.int32)
        y = gen.randint(1, 6, B).astype(np.float32)
        Gd = {k: torch.zeros_like(D[k]) for k in ("P", "Q", "Y", "bu", "bi", "g")}
        loss = torch.zeros(1, dtype=torch.float64, device=DEV)
        if implicit:
            Z = ops.implicit_mean_f32(D["P"], D["Y"], f, ip, ix, users=dev(u))
            loss_ref, G, out = rmf.svdpp_forward_backward(T, u.astype(np.int64), it, y.astype(np.float64), indptr, indices)
            z, ez = implicit_mean_bound(H, u, indptr, indices)
            ops.rating_mf_step_f32(D["P"], D["Q"], D["bu"], D["bi"], D["g"], f, dev(u), dev(it), dev(y), Gd["P"], Gd["Q"],
                                   Gd["bu"], Gd["bi"], Gd["g"], Z=Z, indptr=ip, indices=ix, dY=Gd["Y"], loss=loss)
        else:
            loss_ref, G, out = rmf.funk_svd_forward_backward(T, u.astype(np.int64), it, y.astype(np.float64))
            z, ez = H["P"][u], np.zeros((B, f))
            ops.rating_mf_step_f32(D["P"], D["Q"], D["bu"], D["bi"], None, f, dev(u), dev(it), dev(y), Gd["P"], Gd["Q"],
                                   Gd["bu"], Gd["bi"], None, loss=loss)
        q = H["Q"][it]
        dres = out - y
        e = 2 * dres / B
        # residual: an f-term dot of z (itself within ez) with q, plus b_u, b_i, g and - y (4 more roundings)
        e_d = gamma(f + 4) * (np.abs(z * q).sum(1) + np.abs(H["bu"][u]) + np.abs(H["bi"][it]) + abs(T.get("g", 0.0))
                              + np.abs(y)) + (ez * np.abs(q)).sum(1)
        e_e = 2 * e_d / B + gamma(2) * np.abs(e)                             # 2 d (1/B), 1/B rounded, one product
        e2, ee2 = e[:, None], e_e[:, None]
        bounds = {"Q": scatter(ni, it, e2 * z, np.abs(e2) * ez + ee2 * np.abs(z) + U * np.abs(e2 * z))[1],
                  "P": scatter(nu, u, e2 * q, ee2 * np.abs(q) + U * np.abs(e2 * q))[1],
                  "bu": scatter(nu, u, e, e_e)[1], "bi": scatter(ni, it, e, e_e)[1]}
        if implicit:
            L = indptr[u + 1] - indptr[u]
            rows = np.concatenate([indices[indptr[x]:indptr[x + 1]] for x in u])
            rep = np.repeat(np.arange(B), L)
            tY = (e / L)[rep, None] * q[rep]
            # q (e / L): e / L rounded, one product
            bounds["Y"] = scatter(ni, rows, tY, (e_e / L)[rep, None] * np.abs(q[rep]) + gamma(2) * np.abs(tY))[1]
        for k in bounds:
            got = host(Gd[k])
            got = got[:, :f] if got.ndim == 2 else got[:bounds[k].shape[0]]
            err = np.abs(got - G[k])
            assert (err <= bounds[k]).all(), (k, B, err.max())
        for k in ("P", "Q") + (("Y",) if implicit else ()):
            assert not Gd[k][:, f:].any(), k                                 # padding columns never receive gradient
        assert not Gd["bu"][nu:].any() and not Gd["bi"][ni:].any()
        if implicit:
            # one fp32 sum per warp of its samples' e, then an atomic per warp: at most B additions on a chain
            assert abs(Gd["g"][0].item() - G["g"]) <= e_e.sum() + gamma(B) * (np.abs(e) + e_e).sum()
            assert not Gd["g"][1:].any()
        # the loss: (double) d^2 of the fp32 residual, summed in fp64 and scaled by the fp32 1/B (one rounding)
        assert abs(loss.item() - loss_ref) <= (2 * np.abs(dres) * e_d + e_d ** 2).sum() / B + (U + 1e-12) * loss_ref


@pytest.mark.parametrize("f, ld", LANES)
def test_score_pairs_lane_groups(f, ld):
    """Every (user, relevant item) score against fp64 (U.V + b_i) + (user offset + global offset): -inf for an item of
    the user's mask row, NaN for an out-of-catalogue -1, nothing written for an empty row."""
    rs = np.random.RandomState(f * ld)
    nu, ni = 250, 600
    indptr, indices = _rating_csr(nu, ni, f)
    Uh, Vh = f32(rs.normal(0, 0.4, (nu, f))), f32(rs.normal(0, 0.4, (ni, f)))
    ib, uo, go = f32(rs.normal(0, 0.3, ni)), f32(rs.normal(0, 0.3, nu)), float(np.float32(-0.7))
    rel = []
    for x in range(nu):
        row = list(rs.choice(ni, size=rs.randint(0, 40), replace=False)) if x % 9 else []   # some rows empty
        if x % 5 == 1 and row:
            row[0] = int(indices[indptr[x]])                                 # a train item: masked
        if x % 7 == 2 and row:
            row[-1] = -1                                                     # outside the catalogue
        rel.append(np.array(row, np.int32))
    rp = np.r_[0, np.cumsum([len(x) for x in rel])].astype(np.int64)
    ri = np.concatenate(rel).astype(np.int32)
    s = ops.score_pairs_f32(table(Uh, ld), table(Vh, ld), f, dev(rp), dev(ri), item_bias=dev(ib.astype(np.float32)),
                            user_off=dev(uo.astype(np.float32)), global_off=dev(np.float32([go])), mask_indptr=dev(indptr),
                            mask_indices=dev(indices)).double().cpu().numpy()
    user = np.repeat(np.arange(nu), np.diff(rp))
    masked = np.array([ri[k] >= 0 and ri[k] in set(indices[indptr[user[k]]:indptr[user[k] + 1]]) for k in range(len(ri))],
                      dtype=bool)
    out = ri < 0
    assert masked.sum() > 5 and out.sum() > 5
    assert np.isnan(s[out]).all() and np.isneginf(s[masked]).all()
    ok = ~out & ~masked
    it = ri[ok]
    prod = Uh[user[ok]] * Vh[it]
    want = (prod.sum(1) + ib[it]) + (uo[user[ok]] + go)
    # an f-term dot, + b_i, the user offset + global offset, and their sum: f + 3 roundings on the longest chain
    bound = gamma(f + 3) * (np.abs(prod).sum(1) + np.abs(ib[it]) + np.abs(uo[user[ok]]) + abs(go))
    err = np.abs(s[ok] - want)
    assert (err <= bound).all(), err.max()
