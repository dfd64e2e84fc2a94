"""The kernels of MultiVAE, MultiDAE, NeuMF and GMF one by one against fp64 NumPy computations of the same operations, at
the shapes the models run (the reference defaults H=600, L=200; NeuMF at widths 8..128 and on a whole-epoch batch of
2^20 samples), with input dropout, the unstaged softmax, multi-slab column sums and saturated logits.  The dropout and
noise streams are pinned to the host restatement oracle/philox.py.

Tolerances are derived beside each assert from the length of the operation and the documented error of the intrinsic
it uses (CUDA C Programming Guide, intrinsic functions): with U = 2^-24 the fp32 unit roundoff and gamma(n) = nU/(1-nU)
the bound of an n-term sequential fp32 sum,
  __expf(x)  2 + floor(1.173 |x|) ulp;   __logf(x)  2^-21.41 absolute on [0.5, 2], else 3 ulp;
  __cosf(x)  2^-21.41 absolute on [-pi, pi]; the Box-Muller angle spans [0, 2 pi), where the bound used is the
             2^-20.5 of cos.approx.f32 (PTX ISA);
  bf16 rounding  2^-9 relative.
One ulp of a fp32 value v is at most 2U |v|."""
import numpy as np
import pytest
import torch

from elliot_b200 import ops
from elliot_b200._lib import EbError
from oracle import philox as ph
from oracle import tf_models as tfm

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
ULP = 2 * U                                  # one ulp of v is at most ULP * |v|
FLT_MIN = float(np.finfo(np.float32).tiny)


def gamma(n):
    return n * U / (1 - n * U)


def expf_rel(x):
    """relative error bound of __expf(x)"""
    return (2 + np.floor(1.173 * np.abs(x))) * ULP


def rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def host(t):
    return t.double().cpu().numpy()


def csr_from_rows(rows):
    indptr = np.zeros(len(rows) + 1, np.int64)
    indptr[1:] = np.cumsum([len(r) for r in rows])
    indices = np.concatenate([np.asarray(r, np.int32) for r in rows] + [np.zeros(0, np.int32)])
    return indptr, indices


def random_rows(rs, n_users, n_items, lengths):
    """sorted distinct item rows of the given lengths, cycled over n_users"""
    return [np.sort(rs.choice(n_items, size=lengths[u % len(lengths)], replace=False)).astype(np.int32) for u in range(n_users)]


# ---------------------------------------------------------------------------------------------------- Philox streams
def test_dropout_mask_is_the_restated_philox_stream():
    """Every item belongs to exactly one user, dpre1 = 1: dW1[i, 0] = scale * keep(b, p), which reads the kernel's keep
    bit back for every (batch row, position) and must equal oracle.philox.keep bit for bit."""
    rs = np.random.RandomState(0)
    lengths = [0, 1, 5, 300, 40, 1000, 17]
    nu = 70
    rows, off = [], 0
    for u in range(nu):
        n = lengths[u % len(lengths)]
        rows.append(np.arange(off, off + n, dtype=np.int32)); off += n
    indptr, indices = csr_from_rows(rows)
    I, H, seed = off, 8, 0xDEADBEEF12345
    batch = rs.permutation(nu).astype(np.int32)                     # batch row b != user id: the counter is the batch row
    for drop in (0.5, 0.2):
        dW1 = torch.zeros((I, H), device=DEV)
        dpre1 = torch.ones((nu, H), device=DEV)
        ops.vae_embed_bwd(dW1, dev(indptr), dev(indices), dev(batch), dpre1, drop, seed)
        got = host(dW1)
        for b, u in enumerate(batch):
            beg, end = indptr[u], indptr[u + 1]
            if end == beg:
                continue
            want = ph.keep(seed, b, np.arange(end - beg), drop)
            assert np.array_equal(got[beg:end, 0] != 0, want), (drop, b, u)
            # value: rsqrtf(n) (2 ulp) times 1/(1-drop) (rounded), one product
            s = 1 / np.sqrt(end - beg) / (1 - np.float32(drop))
            assert np.all(np.abs(got[beg:end, 0][want] - s) <= 4 * ULP * s)
            assert np.all(got[beg:end] == got[beg:end, :1])         # one scalar per item: every column the same
        assert 0.3 < (got[:, 0] != 0).mean() / (1 - drop) < 1.7


def _box_muller_tol(seed, step, n):
    """Per-element bound of |eps_device - eps_fp64| (Box-Muller with __logf / __cosf, see module docstring)."""
    r = ph.gen(seed, np.full(n, step, dtype=np.uint64), np.arange(n, dtype=np.uint64))
    u1 = ((r[0] >> np.uint32(8)).astype(np.float64) + 0.5) * 2.0 ** -24
    u2 = (r[1] >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
    w = -2 * np.log(u1)
    # u1 = (k + 0.5) 2^-24 is rounded in fp32 for k >= 2^23 (2 ulp of log's input at most), __logf, the rounded -2 log u1
    dlog = 2 * ULP + np.where(u1 >= 0.5, 2.0 ** -21.41, 3 * ULP * np.abs(np.log(u1))) + ULP * w
    dsq = np.minimum(dlog / (2 * np.sqrt(np.maximum(w, 1e-300))), np.sqrt(2 * dlog)) + ULP * np.sqrt(w)
    dcos = 2.0 ** -20.5 + 2 * np.pi * u2 * ULP                      # cos.approx on [0, 2 pi) plus the rounded angle
    return dsq * np.abs(np.cos(2 * np.pi * u2)) + np.sqrt(w) * dcos + 2 * ULP * np.sqrt(w)


def test_reparam_matches_fp64_with_the_restated_noise():
    rs = np.random.RandomState(1)
    B, L, seed, step, anneal = 77, 200, 0x9E3779B1, 5, 0.13
    n = B * L
    ml_full = np.zeros((B, 2 * L + 8), np.float32)                    # ldml > 2L
    ml_full[:, :L] = rs.normal(0, 0.5, (B, L)); ml_full[:, L:2 * L] = rs.uniform(-1.5, 1.5, (B, L))
    ml = dev(ml_full)[:, :2 * L]
    zbuf = torch.full((B, L + 4), 7.0, device=DEV)
    z = zbuf[:, :L]
    kl = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.vae_reparam_fwd(ml, L, z, seed, step, kl)
    mu, lv = ml_full[:, :L].astype(np.float64), ml_full[:, L:2 * L].astype(np.float64)
    eps = ph.reparam_eps(seed, step, n).reshape(B, L)
    deps = _box_muller_tol(seed, step, n).reshape(B, L)
    # recovered noise (z - mu) / exp(lv/2): the fp32 z = mu + __expf(lv/2) eps carries 2 roundings and __expf's error
    zd = host(z)
    sd = np.exp(0.5 * lv)
    got = (zd - mu) / sd
    tol = deps + np.abs(eps) * (expf_rel(0.5 * lv) + ULP) + ULP * np.abs(zd) / sd
    assert np.all(np.abs(got - eps) <= tol)
    assert np.median(np.abs(got - eps)) < 1e-6                          # ~1e-6 agreement as a rule, the bound is worst case
    assert np.all(host(zbuf)[:, L:] == 7.0)
    # KL sum: one term per thread (B L < threads of the grid), then 5 shuffle levels and fp64 atomics
    t = lv - mu ** 2 - np.exp(lv) + 1
    terr = (np.abs(lv) + mu ** 2 + np.exp(lv) + 1) * 4 * U + np.exp(lv) * expf_rel(lv)
    assert abs(kl.item() - t.sum()) <= terr.sum() + gamma(6) * np.abs(t).sum()
    # backward: dml = (dz + c mu | dz 0.5 e^{lv/2} eps + c 0.5 (e^lv - 1)), c = anneal / (B L)
    dz_full = rs.normal(0, 1, (B, L + 4)).astype(np.float32)
    dml = torch.zeros((B, 2 * L + 4), device=DEV)
    ops.vae_reparam_bwd(ml, L, dev(dz_full)[:, :L], dml[:, :2 * L], seed, step, anneal)
    dz = dz_full[:, :L].astype(np.float64)
    c = anneal / n
    got = host(dml)
    assert np.all(got[:, 2 * L:] == 0)
    dmu = dz + c * mu
    assert np.all(np.abs(got[:, :L] - dmu) <= 2 * ULP * (np.abs(dz) + c * np.abs(mu)) + 2 * ULP * c * np.abs(mu))
    a = dz * 0.5 * sd * eps
    k = c * 0.5 * (np.exp(lv) - 1)
    err = np.abs(dz * 0.5 * sd) * deps + np.abs(a) * (expf_rel(0.5 * lv) + 4 * ULP) \
        + c * 0.5 * np.exp(lv) * (expf_rel(lv) + ULP) + np.abs(k) * 4 * ULP + ULP * np.abs(a + k)
    assert np.all(np.abs(got[:, L:2 * L] - (a + k)) <= err)


def _noise_pairs(seed, steps, L):
    """Bits of the consecutive noise pairs (eps[e], eps[e+1]) the device draws at each (step, B): z = 0 + __expf(0) eps."""
    keys = []
    for step, B in steps:
        ml = torch.zeros((B, 2 * L), device=DEV)
        z = torch.empty((B, L), device=DEV)
        ops.vae_reparam_fwd(ml, L, z, seed, step)
        bits = z.reshape(-1).view(torch.int32).cpu().numpy().astype(np.uint32).astype(np.uint64)
        keys.append((bits[:-1] << np.uint64(32)) | bits[1:])
    return keys


@pytest.mark.parametrize("steps", [
    [(s, 500) for s in range(1, 13)] + [(13, 40)],                # one epoch of 6040 users at batch 500: tail of 40 last
    [(0, 500), (1, 40)],
    [(1, 40), (2, 500)],                                           # the reverse order
])
def test_reparam_noise_never_repeats_across_steps(steps):
    """Steps of different batch sizes draw disjoint noise: no consecutive pair of eps values of one step reappears in
    another (a shared Philox counter would repeat whole runs of them)."""
    keys = _noise_pairs(0x5EED, steps, 200)
    for i in range(len(keys)):
        for j in range(i + 1, len(keys)):
            common = np.intersect1d(keys[i], keys[j])
            assert common.size == 0, (steps[i], steps[j], common.size)


# ---------------------------------------------------------------------------------------------------- sparse first layer
@pytest.mark.parametrize("H", [8, 600, 2056])
@pytest.mark.parametrize("drop", [0.0, 0.5])
def test_embed_fwd_bwd_match_fp64(H, drop):
    """h1 = tanh(s_b sum_{kept p} W1[i_p] + b1) and dW1[i_p] += s_b dpre1[b] (s_b = keep_scale / sqrt(nnz_b)) against
    fp64 with the restated mask; users with 0, 1 and > 256 items; ldh, ldd > H; H = 2056 takes 3 passes of 256 float4."""
    rs = np.random.RandomState(H + int(drop * 10))
    I, nu, seed = 3000, 60, 0xABCDEF
    rows = random_rows(rs, nu, I, [0, 1, 300, 2, 20, 700, 50])
    indptr, indices = csr_from_rows(rows)
    batch = rs.permutation(nu)[:40].astype(np.int32)
    W1 = rs.normal(0, 0.05, (I, H)).astype(np.float32)
    b1 = rs.normal(0, 0.05, H).astype(np.float32)
    h1 = torch.full((len(batch), H + 4), 9.0, device=DEV)
    ops.vae_embed_fwd(dev(W1), dev(b1), dev(indptr), dev(indices), dev(batch), h1[:, :H], drop, seed)
    K = ph.csr_keep_mask(seed, indptr, indices, batch, I, drop)     # [B][I] 0/1
    nnz = np.diff(indptr)[batch].astype(np.float64)
    s = np.where(nnz > 0, 1 / np.sqrt(np.maximum(nnz, 1)), 0.0) / (1 - np.float32(drop) if drop > 0 else 1.0)
    W = W1.astype(np.float64)
    pre = s[:, None] * (K @ W) + b1
    # error: the kept-row sum (nk terms, sequential), rsqrtf (2 ulp = 4U), the keep scale and the scale product (2U each),
    # + bias (FMA or not), tanhf (2 ulp)
    nk = K.sum(1)
    perr = s[:, None] * (gamma(nk + 8)[:, None] * (K @ np.abs(W))) + ULP * np.abs(pre) + 2 * ULP * np.abs(b1)
    got = host(h1)
    assert np.all(got[:, H:] == 9.0)
    assert np.all(np.abs(got[:, :H] - np.tanh(pre)) <= perr + 2 * ULP * np.abs(np.tanh(pre)) + 1e-30)
    # backward into a zero dW1; items shared by several batch rows accumulate with fp32 atomics
    dpre1_full = rs.normal(0, 1, (len(batch), H + 8)).astype(np.float32)
    dW1 = torch.zeros((I, H), device=DEV)
    ops.vae_embed_bwd(dW1, dev(indptr), dev(indices), dev(batch), dev(dpre1_full)[:, :H], drop, seed)
    D = dpre1_full[:, :H].astype(np.float64)
    want = (K * s[:, None]).T @ D
    cnt = K.sum(0)
    berr = gamma(cnt + 8)[:, None] * ((K * s[:, None]).T @ np.abs(D))
    gotw = host(dW1)
    assert np.all(np.abs(gotw - want) <= berr + 1e-30)
    # adjoint: <dpre1, d pre1 / d W1 . W1> = <dW1, W1> under the same mask (a mask that differs between the passes fails)
    lin = np.arctanh(got[:, :H]) - b1                              # |pre| < 0.6 here, atanh is well conditioned
    lhs, rhs = (D * lin).sum(), (gotw * W).sum()
    assert abs(lhs - rhs) <= 1e-5 * (np.abs(D) * np.abs(lin)).sum()


# ---------------------------------------------------------------------------------------------------- softmax / NLL
def _softmax_case(rs, B, I, spread):
    """logits spread over +-spread, a CSR whose batch holds a user with all I items and one with none"""
    nu = max(B, 2) + 3
    lengths = [int(x) for x in rs.randint(1, min(I, 60) + 1, size=nu)]
    rows = [np.sort(rs.choice(I, size=n, replace=False)).astype(np.int32) for n in lengths]
    rows[1] = np.arange(I, dtype=np.int32)                          # all items
    rows[2] = np.zeros(0, np.int32)                                 # none
    indptr, indices = csr_from_rows(rows)
    batch = np.concatenate([[1, 2], rs.choice(np.arange(3, nu), size=B - 2, replace=False)]) if B >= 2 else np.array([1])
    logits = rs.uniform(-spread, spread, (B, I)).astype(np.float32)
    return indptr, indices, batch.astype(np.int32), logits


def _softmax_ref(logits, indptr, indices, batch):
    """fp64 lse, nll, dlogits and their per-element error bounds for the device's fp32 evaluation (either kernel: 256 or
    512 threads, so at most ceil(I / 256) terms per thread and 16 warps)"""
    B, I = logits.shape
    x = logits.astype(np.float64)
    m = x.max(1, keepdims=True)
    t = np.exp(x - m).sum(1, keepdims=True)
    lse = m + np.log(t)
    X = np.zeros((B, I))
    for b, u in enumerate(batch):
        X[b, indices[indptr[u]:indptr[u + 1]]] = 1
    nb = X.sum(1, keepdims=True)
    p = np.exp(x - lse)
    dl = (p * nb - X) / B
    nll = -((x - lse) * X).sum()
    # t: per-thread sequential sums of I/256 terms, 5 shuffle levels and a 16-warp reduction; each term with __expf's
    # error and the rounding of its argument x - m
    q = np.exp(x - m) / t
    dt = (np.ceil(I / 256) + 5 + 16) * ULP + (q * (expf_rel(x - m) + ULP * np.abs(x - m))).sum(1, keepdims=True)
    dlse = dt + np.where(t <= 2, 2.0 ** -21.41, 3 * ULP * np.abs(np.log(t))) + ULP * np.abs(lse)
    # dlogits = __expf(x - lse) nb / B (- 1/B): __expf error, lse error, two products and the subtraction
    ddl = p * nb / B * (expf_rel(x - lse) + ULP * np.abs(x - lse) + dlse + 4 * ULP) + ULP * np.abs(dl) + X * ULP / B + FLT_MIN * (nb / B + 1)
    dnll = (nb[:, 0] * dlse[:, 0]).sum() + gamma(np.ceil(nb.max() / 256) + 7) * (np.abs(x - lse) * X).sum()
    return lse[:, 0], nll, dl, dlse[:, 0], ddl, dnll


@pytest.mark.parametrize("I,B,path", [
    (1, 1, "staged"), (7, 77, "staged"), (1000, 500, "staged"), (26744, 77, "staged"), (51200, 77, "staged"),
    (51201, 77, "unstaged"), (70000, 1, "unstaged"), (70000, 77, "unstaged"),
    (1003, 77, "unstaged_ld"), (1000, 77, "unstaged_offset"),
])
def test_softmax_nll_and_gradient_match_fp64(I, B, path):
    """Both paths of eb_vae_softmax_bf16: the shared-memory staged kernel (rows up to 51200 items, 16-byte aligned rows) and
    the unstaged fallback (longer rows, ld % 4 != 0, a row start 4 bytes off 16), each with the bf16 gradient copy."""
    rs = np.random.RandomState(I + B)
    indptr, indices, batch, logits = _softmax_case(rs, B, I, 80.0)
    ld = I if path == "unstaged_ld" else (I + 3) // 4 * 4 + 4        # ld > I, a multiple of 4 unless ld % 4 is tested
    assert (ld % 4 != 0) == (path == "unstaged_ld")
    if path == "unstaged_offset":                                       # every row start 4 bytes off a 16-byte boundary
        lg = torch.zeros(B * ld + 1, device=DEV)[1:].view(B, ld)[:, :I]
    else:
        lg = torch.zeros((B, ld), device=DEV)[:, :I]
    lg.copy_(dev(logits))
    ldb = (I + 7) // 8 * 8 + 8
    gb = torch.full((B, ldb), 3.0, dtype=torch.bfloat16, device=DEV)
    nll = torch.zeros(1, dtype=torch.float64, device=DEV)
    lse = torch.empty(B, device=DEV)
    ops.vae_softmax(lg, dev(indptr), dev(indices), dev(batch), nll_sum=nll, lse_out=lse, write_grad=True, grad_bf16=gb)
    lse_ref, nll_ref, dl_ref, dlse, ddl, dnll = _softmax_ref(logits, indptr, indices, batch)
    assert np.all(np.abs(host(lse) - lse_ref) <= dlse)
    assert abs(nll.item() - nll_ref) <= dnll
    got = host(lg)
    assert np.all(np.abs(got - dl_ref) <= ddl)
    assert torch.equal(gb[:, :I], lg.to(torch.bfloat16))              # the copy is bf16(dlogits), element for element
    assert not gb[:, I:].float().any()                                # padding columns zeroed


@pytest.mark.parametrize("I", [1000, 51201])
def test_softmax_lse_alone_leaves_the_logits(I):
    rs = np.random.RandomState(5)
    indptr, indices, batch, logits = _softmax_case(rs, 77, I, 30.0)
    lg = dev(logits)
    lse = torch.empty(77, device=DEV)
    ops.vae_softmax(lg, dev(indptr), dev(indices), dev(batch), lse_out=lse, write_grad=False)
    lse_ref, _, _, dlse, _, _ = _softmax_ref(logits, indptr, indices, batch)
    assert np.all(np.abs(host(lse) - lse_ref) <= dlse)
    assert torch.equal(lg, dev(logits))


@pytest.mark.parametrize("I", [1000, 51201])
def test_softmax_bf16_copy_contract_is_the_same_on_both_paths(I):
    """ld_bf16 must be a multiple of 8 (the copy is a GEMM operand) and the buffer 16-byte aligned, staged or not: both are
    refused before any launch."""
    rs = np.random.RandomState(6)
    indptr, indices, batch, logits = _softmax_case(rs, 4, I, 5.0)
    lg = dev(logits)
    ldb = (I + 7) // 8 * 8
    for bad in (torch.zeros((4, ldb + 2), dtype=torch.bfloat16, device=DEV),                    # ld % 8 != 0
                torch.zeros(4 * ldb + 8, dtype=torch.bfloat16, device=DEV)[2:2 + 4 * ldb].view(4, ldb)):  # 4-byte aligned
        with pytest.raises(EbError):
            ops.vae_softmax(lg, dev(indptr), dev(indices), dev(batch), write_grad=True, grad_bf16=bad)
    assert torch.equal(lg, dev(logits))


# ---------------------------------------------------------------------------------------------------- column sums
@pytest.mark.parametrize("rows", [1, 8192, 8193, 1 << 20])
@pytest.mark.parametrize("cols", [1, 31, 33, 600])
def test_colsum_matches_exact_sums(rows, cols):
    """Entries k/64 with |k| <= 16: every partial sum of any order is a multiple of 2^-6 below 2^18, exact in fp32, so the
    single-slab and the multi-slab (atomics into a zeroed output, rows > 8192) sums must equal the exact sum bit for bit;
    a dropped or repeated row cannot hide.  ld > cols."""
    g = torch.Generator(device=DEV); g.manual_seed(rows * 7 + cols)
    ld = cols + 3
    k8 = torch.randint(-16, 17, (rows, ld), device=DEV, generator=g, dtype=torch.int8)
    src = (k8.float() / 64)[:, :cols]
    out = torch.full((cols,), 5.0, device=DEV)
    ops.colsum(src, out)
    want = k8[:, :cols].cpu().numpy().sum(0, dtype=np.int64) / 64.0
    assert np.array_equal(host(out), want)


@pytest.mark.parametrize("rows", [1, 8192, 8193, 100000])
def test_colsum_of_random_values_within_the_summation_bound(rows):
    """Real-valued entries: |error| <= gamma(n) sum |x|, n the longest chain of additions (rows / 8 per warp, 8 warps,
    up to rows / 1024 slabs)."""
    rs = np.random.RandomState(rows)
    cols = 600
    x = rs.normal(0, 1, (rows, cols + 5)).astype(np.float32)
    out = ops.colsum(dev(x)[:, :cols])
    xd = x[:, :cols].astype(np.float64)
    n = -(-rows // 8) + 8 + -(-rows // 1024) + 1
    assert np.all(np.abs(host(out) - xd.sum(0)) <= gamma(n) * np.abs(xd).sum(0))


# ---------------------------------------------------------------------------------------------------- elementwise kernels
def test_elementwise_kernels_match_their_formulas():
    rs = np.random.RandomState(7)
    n = 100003
    dout = rs.normal(0, 2, n).astype(np.float32)
    out = np.tanh(rs.normal(0, 2, n)).astype(np.float32)
    out[:5] = [1.0, -1.0, 0.0, 0.99999994, -0.5]
    # tanh_bwd: dout (1 - out^2): the product out*out (rounded unless contracted to an FMA), 1 - . and the final product
    got = host(ops.tanh_bwd(dev(dout), dev(out)))
    o, d = out.astype(np.float64), dout.astype(np.float64)
    want = d * (1 - o * o)
    assert np.all(np.abs(got - want) <= np.abs(d) * U * o * o + 2 * ULP * np.abs(want))
    # relu_bwd: a selection (exact), and its bf16 operand copy equals bf16(dpre)
    hr = np.maximum(rs.normal(0, 1, (257, 64)), 0).astype(np.float32)
    dr = rs.normal(0, 1, (257, 64)).astype(np.float32)
    dpre, cb = ops.relu_bwd(dev(dr), dev(hr), copy_bf16=True)
    assert np.array_equal(host(dpre), np.where(hr > 0, dr, 0).astype(np.float64))
    assert torch.equal(cb, dpre.to(torch.bfloat16))
    # sigmoid_: 1 / (1 + __expf(-x)); -inf (masked padding) -> 0, +inf -> 1
    x = rs.normal(0, 10, n).astype(np.float32)
    x[:6] = [-np.inf, np.inf, -87.0, 87.0, 0.0, -200.0]
    got = host(ops.sigmoid_(dev(x)))
    xd = x.astype(np.float64)
    with np.errstate(over="ignore"):
        want = 1 / (1 + np.exp(-xd))
    err = want * (1 - want) * np.where(np.isfinite(xd), expf_rel(xd), 0) + 2 * ULP * want + FLT_MIN
    assert got[0] == 0.0 and got[1] == 1.0
    assert np.all(np.abs(got - want) <= err)
    # gmf_scale_rows: one product per element, exact against the fp32 product; columns past f untouched
    for f in (4, 12, 128):
        src = rs.normal(0, 1, (333, 128 + 4)).astype(np.float32)
        h = rs.normal(0, 1, 128).astype(np.float32)
        o = ops.gmf_scale_rows(dev(src), dev(h), f)
        g = o.cpu().numpy()
        assert np.array_equal(g[:, :f], src[:, :f] * h[:f]) and not g[:, f:].any()


# ---------------------------------------------------------------------------------------------------- NeuMF
def _neumf_tables(rs, nu, ni, f, ld):
    T = {k: np.zeros((n, ld), np.float32) for k, n in (("U_mf", nu), ("I_mf", ni), ("U_mlp", nu), ("I_mlp", ni))}
    for k in T:
        T[k][:, :f] = rs.normal(0, 0.5, (T[k].shape[0], f))
    return T


@pytest.mark.parametrize("f", [8, 16, 64, 128])
def test_neumf_gather_and_scatter_match_fp64(f):
    rs = np.random.RandomState(f)
    nu, ni, n, ld = 300, 200, 20000, 128
    T = _neumf_tables(rs, nu, ni, f, ld)
    u = rs.randint(0, nu, n).astype(np.int32); it = rs.randint(0, ni, n).astype(np.int32)
    u[:50] = 3; it[:50] = 7                                          # a repeated (u, i) pair
    D = {k: dev(v) for k, v in T.items()}
    x0 = torch.empty((n, 2 * f), device=DEV); pm = torch.empty((n, f), device=DEV)
    ops.neumf_gather(D["U_mf"], D["I_mf"], D["U_mlp"], D["I_mlp"], f, dev(u), dev(it), x0, pm)
    a, b = T["U_mf"][u, :f], T["I_mf"][it, :f]
    assert np.array_equal(x0.cpu().numpy(), np.concatenate([T["U_mlp"][u, :f], T["I_mlp"][it, :f]], 1))
    assert np.array_equal(pm.cpu().numpy(), a * b)                   # one fp32 product: exact
    dpm = rs.normal(0, 1, (n, f)).astype(np.float32); dx0 = rs.normal(0, 1, (n, 2 * f)).astype(np.float32)
    G = {k: torch.zeros((v.shape[0], ld), device=DEV) for k, v in T.items()}
    ops.neumf_scatter(D["U_mf"], D["I_mf"], f, dev(u), dev(it), dev(dpm), dev(dx0), G["U_mf"], G["I_mf"], G["U_mlp"], G["I_mlp"])
    ad, bd, gd = a.astype(np.float64), b.astype(np.float64), dpm.astype(np.float64)
    for k, idx, contrib, rows in (("U_mf", u, gd * bd, nu), ("I_mf", it, gd * ad, ni),
                                  ("U_mlp", u, dx0[:, :f].astype(np.float64), nu), ("I_mlp", it, dx0[:, f:].astype(np.float64), ni)):
        want = np.zeros((rows, f)); mag = np.zeros((rows, f))
        np.add.at(want, idx, contrib); np.add.at(mag, idx, np.abs(contrib))
        cnt = np.bincount(idx, minlength=rows)[:, None]
        g = host(G[k])
        assert not g[:, f:].any()
        # each contribution rounded once (product), then cnt fp32 atomic additions in any order
        assert np.all(np.abs(g[:, :f] - want) <= gamma(cnt + 1) * mag), k


def _head_case(rs, n, f):
    wp = rs.normal(0, 0.5, 2 * f).astype(np.float32)
    bp = np.array([0.1], np.float32)
    pm = rs.normal(0, 0.3, (n, f)).astype(np.float32)                # |logit| < 16 (the clip) by > 7 sigma at f = 128
    h3 = np.maximum(rs.normal(0, 0.3, (n, f)), 0).astype(np.float32)
    sat = rs.choice(n, 200, replace=False)                           # logits past the 1e-7 clip, both signs
    sign = np.where(np.arange(200) % 2 == 0, 1.0, -1.0)[:, None]
    pm[sat] = (sign * 40.0 / np.abs(wp[:f]).sum() * np.sign(wp[:f])).astype(np.float32)
    h3[sat] = 0
    y = (rs.rand(n) < 0.4).astype(np.float32)
    return wp, bp, pm, h3, y, sat


@pytest.mark.parametrize("f", [8, 16, 64, 128])
def test_neumf_head_matches_fp64(f):
    """logit = bp + wp . [pm | h3], Keras BCE mean over mean_over != n samples, dl = 0 where the probability is clipped,
    dpm, dh3 (last ReLU's mask), dwp, dbp; n large enough that every warp loops."""
    rs = np.random.RandomState(100 + f)
    n, mean_over = 20000, 20037
    wp, bp, pm, h3, y, sat = _head_case(rs, n, f)
    dpm = torch.empty((n, f), device=DEV); dh3 = torch.empty((n, f), device=DEV)
    dwp = torch.zeros(2 * f, device=DEV); dbp = torch.zeros(1, device=DEV)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV); prob = torch.empty(n, device=DEV)
    ops.neumf_head(dev(pm), dev(h3), f, dev(wp), dev(bp), label=dev(y), dpm=dpm, dh3=dh3, dwp=dwp, dbp=dbp, loss=loss,
                   prob=prob, mean_over=mean_over)
    feat = np.concatenate([pm, h3], 1).astype(np.float64)
    w = wp.astype(np.float64); yd = y.astype(np.float64)
    logit = feat @ w + bp[0]
    p = 1 / (1 + np.exp(-logit))
    # logit: lane sums of 2f/32 products, 5 shuffle levels, + bias; p: __expf, one add, one IEEE division
    dlogit = gamma(-(-2 * f // 32) + 7) * (np.abs(feat) @ np.abs(w) + abs(bp[0]))
    dp = p * (1 - p) * (dlogit + expf_rel(logit)) + 2 * ULP * p
    assert np.all(np.abs(host(prob) - p) <= dp)
    open_ = (p > tfm.CLIP_LO) & (p < tfm.CLIP_HI)
    assert (~open_[sat]).all() and open_.sum() == n - 200
    inv = np.float64(np.float32(1 / mean_over))
    dl = np.where(open_, p - yd, 0.0) * inv
    ddl = (dp + ULP * np.abs(p - yd)) * inv * (1 + ULP)
    assert np.all(np.abs(host(dpm) - dl[:, None] * w[:f]) <= ddl[:, None] * np.abs(w[:f]) + ULP * np.abs(dl[:, None] * w[:f]))
    want_h3 = np.where(h3 > 0, dl[:, None] * w[f:], 0.0)
    assert np.all(np.abs(host(dh3) - want_h3) <= (h3 > 0) * (ddl[:, None] * np.abs(w[f:]) + ULP * np.abs(want_h3)))
    assert not host(dpm)[sat].any() and not host(dh3)[sat].any()
    # dwp: per-lane sums over each warp's samples, then fp32 atomics across warps: at most n additions per column
    want_w = feat.T @ dl
    bound_w = gamma(n + 1) * (np.abs(feat).T @ np.abs(dl)) + np.abs(feat).T @ ddl
    assert np.all(np.abs(host(dwp) - want_w) <= bound_w)
    assert abs(dbp.item() - dl.sum()) <= gamma(n + 1) * np.abs(dl).sum() + ddl.sum()
    pc = np.clip(p, tfm.CLIP_LO, tfm.CLIP_HI)
    bce = -(yd * np.log(pc) + (1 - yd) * np.log(1 - pc))
    # loss: __logf of the clipped probability (3 ulp / 2^-21.41), its input's error dp / pc, fp32 lane sums, fp64 atomics
    dbce = dp / np.minimum(pc, 1 - pc) + 2.0 ** -21.41 + 4 * ULP * bce
    assert abs(loss.item() - bce.sum() * inv) <= (dbce.sum() + gamma(n) * bce.sum()) * inv


@pytest.mark.parametrize("f", [8, 16, 64, 128])
def test_neumf_pair_kernels_match_fp64(f):
    """get_recs pieces: H1 = relu(Au[ub] + Ai[i] + b1) as bf16 and fp32, and prob = sigmoid(bp + w_mf . (U_mf[u0+ub] *
    I_mf[i]) + w_mlp . h3[pair]) for every pair of a user block; ldo > 4f and ldpr > n_items."""
    rs = np.random.RandomState(200 + f)
    nb, ni, u0, h = 7, 301, 5, 4 * f
    Au = rs.normal(0, 1, (nb, h + 4)).astype(np.float32); Ai = rs.normal(0, 1, (ni, h + 8)).astype(np.float32)
    b1 = rs.normal(0, 0.5, h).astype(np.float32)
    pre = (Au[:, None, :h].astype(np.float64) + Ai[None, :, :h]) + b1
    want = np.maximum(pre, 0).reshape(nb * ni, h)
    ref32 = np.maximum((Au[:, None, :h] + Ai[None, :, :h]) + b1, np.float32(0)).reshape(nb * ni, h)   # the same two fp32 adds
    out = torch.full((nb * ni, h + 8), 2.0, device=DEV)
    ops.neumf_pair_h1(dev(Au)[:, :h], dev(Ai)[:, :h], dev(b1), nb, ni, h, out[:, :h])
    got = out.cpu().numpy()
    mag = (np.abs(Au[:, None, :h]).astype(np.float64) + np.abs(Ai[None, :, :h]) + np.abs(b1)).reshape(nb * ni, h)
    assert np.all(np.abs(got[:, :h] - want) <= 2 * U * mag) and np.all(got[:, h:] == 2.0)
    assert np.array_equal(got[:, :h], ref32)
    outb = torch.full((nb * ni, h + 8), 2.0, dtype=torch.bfloat16, device=DEV)
    ops.neumf_pair_h1(dev(Au)[:, :h], dev(Ai)[:, :h], dev(b1), nb, ni, h, outb[:, :h])
    assert torch.equal(outb[:, :h], dev(ref32).to(torch.bfloat16)) and (outb[:, h:].float() == 2.0).all()
    # pair head
    ld = 128
    Umf = np.zeros((u0 + nb + 3, ld), np.float32); Umf[:, :f] = rs.normal(0, 1, (u0 + nb + 3, f))
    Imf = np.zeros((ni, ld), np.float32); Imf[:, :f] = rs.normal(0, 1, (ni, f))
    h3 = np.maximum(rs.normal(0, 1, (nb * ni, f + 4)), 0).astype(np.float32)
    wp = rs.normal(0, 0.5, 2 * f).astype(np.float32); bp = np.array([-0.2], np.float32)
    prob = torch.full((nb, ni + 5), 4.0, device=DEV)
    ops.neumf_pair_head(dev(Umf), dev(Imf), f, u0, nb, ni, dev(h3)[:, :f], dev(wp), dev(bp), prob[:, :ni])
    pmf = (Umf[u0:u0 + nb, None, :f].astype(np.float64) * Imf[None, :, :f]).reshape(nb * ni, f)
    feat = np.concatenate([pmf, h3[:, :f]], 1)
    logit = feat @ wp.astype(np.float64) + bp[0]
    p = 1 / (1 + np.exp(-logit))
    # each mf term has two products (2 roundings), the dot has 2f/32 terms per lane and 5 shuffle levels, + bias
    dlogit = gamma(-(-2 * f // 32) + 9) * (np.abs(feat) @ np.abs(wp.astype(np.float64)) + abs(bp[0]))
    dp = p * (1 - p) * (dlogit + expf_rel(logit)) + 2 * ULP * p
    gotp = host(prob)
    assert np.all(np.abs(gotp[:, :ni].reshape(-1) - p) <= dp) and np.all(gotp[:, ni:] == 4.0)


@pytest.mark.parametrize("m", [0, 3])
def test_neumf_sample_positives_exact_negatives_outside_train(m):
    """Users with empty rows between non-empty ones, one user missing a single item (every negative must be that item)."""
    rs = np.random.RandomState(300 + m)
    nu, ni = 40, 50
    rows = []
    for u in range(nu):
        if u % 4 == 1:
            rows.append(np.zeros(0, np.int32))
        elif u == 6:
            rows.append(np.delete(np.arange(ni, dtype=np.int32), 17))
        else:
            rows.append(np.sort(rs.choice(ni, size=rs.randint(1, 12), replace=False)).astype(np.int32))
    indptr, indices = csr_from_rows(rows)
    u, i, y = (t.cpu().numpy() for t in ops.neumf_sample(nu, ni, dev(indptr), dev(indices), m, 99))
    nnz = len(indices)
    assert len(u) == nnz * (1 + m)
    owner = np.repeat(np.arange(nu), np.diff(indptr))
    s = np.arange(nnz) * (1 + m)                                      # sample p (1 + m) is positive p
    assert np.array_equal(u[s], owner) and np.array_equal(i[s], indices) and (y[s] == 1).all()
    neg = np.setdiff1d(np.arange(len(u)), s)
    assert (y[neg] == 0).all() and np.array_equal(u[neg], np.repeat(owner, m))
    assert ((i[neg] >= 0) & (i[neg] < ni)).all()
    for q in neg:
        assert i[q] not in rows[u[q]]
    if m:
        assert (i[neg][u[neg] == 6] == 17).all()


# ---------------------------------------------------------------------------------------------------- GMF
@pytest.mark.parametrize("f", [4, 12, 64, 128])
def test_gmf_step_grads_match_fp64(f):
    """Fused GMF step with duplicate (u, i) pairs, saturated logits (dl = 0 on both sides) and n > 8448 warps of the grid:
    gradients to 1e-5 relative.  The loss is Keras BCE of the fp32 probability: log(1 - p) of a confident sample inherits
    the absolute error of p (rounding, __expf) divided by 1 - p, so at f >= 64, where |logit| reaches ~15, it is held to
    that derived bound instead of a flat 1e-6 (which it meets at f <= 12)."""
    rs = np.random.RandomState(400 + f)
    nu, ni, n, ld = 500, 400, 30000, 128
    Ut = np.zeros((nu, ld), np.float32); It = np.zeros((ni, ld), np.float32); h = np.zeros(ld, np.float32)
    Ut[:, :f] = rs.normal(0, 0.6, (nu, f)); It[:, :f] = rs.normal(0, 0.6, (ni, f)); h[:f] = rs.normal(0, 1, f)
    Ut[0, :f] = 8 * np.sign(h[:f]); It[0, :f] = 8                       # user 0 x item 0: logit 64 sum|h| -> p clipped to 1
    Ut[1, :f] = -8 * np.sign(h[:f]); It[1, :f] = 8                      # user 1 x item 1: clipped to 0
    u = rs.randint(2, nu, n).astype(np.int32); it = rs.randint(2, ni, n).astype(np.int32)
    u[:40] = 9; it[:40] = 9                                               # duplicates
    u[40:60] = 0; it[40:60] = 0; u[60:80] = 1; it[60:80] = 1
    y = (rs.rand(n) < 0.5).astype(np.float32)
    P = {"U": Ut[:, :f].astype(np.float64), "I": It[:, :f].astype(np.float64), "h": h[:f].astype(np.float64)}
    loss_ref, G, p = tfm.gmf_forward_backward(P, u, it, y.astype(np.float64))
    assert (p[40:80] <= tfm.CLIP_LO).sum() + (p[40:80] >= tfm.CLIP_HI).sum() == 40
    dU = torch.zeros((nu, ld), device=DEV); dI = torch.zeros((ni, ld), device=DEV); dh = torch.zeros(ld, device=DEV)
    loss = torch.zeros(1, dtype=torch.float64, device=DEV)
    ops.gmf_step_grads(dev(Ut), dev(It), dev(h), f, dev(u), dev(it), dev(y), dU, dI, dh, loss=loss)
    # logit: 4 products of two rounded products per lane, 5 shuffle levels; p: __expf, an add and a division; the BCE term:
    # its input's error dp / min(pc, 1 - pc), __logf (3 ulp / 2^-21.41); sums: ceil(n / 8448) terms per lane, fp64 atomics
    a = np.abs(P["U"][u] * P["I"][it]) @ np.abs(P["h"])
    logit = (P["U"][u] * P["I"][it]) @ P["h"]
    dp = p * (1 - p) * (gamma(12) * a + expf_rel(logit)) + 2 * ULP * p
    pc = np.clip(p, tfm.CLIP_LO, tfm.CLIP_HI)
    yd = y.astype(np.float64)
    bce = -(yd * np.log(pc) + (1 - yd) * np.log(1 - pc))
    dbce = dp / np.minimum(pc, 1 - pc) + 2.0 ** -21.41 + 4 * ULP * bce
    assert abs(loss.item() - loss_ref) <= (dbce.sum() + gamma(-(-n // 8448) + 1) * bce.sum()) / n
    if f <= 12:
        assert abs(loss.item() - loss_ref) < 1e-6 * abs(loss_ref)
    for k, t in (("U", dU), ("I", dI)):
        g = host(t)
        assert rel(g[:, :f], G[k]) < 1e-5 and not g[:, f:].any(), k
    assert rel(host(dh)[:f], G["h"]) < 1e-5 and not host(dh)[f:].any()
    assert not host(dU)[[0, 1]].any() and not host(dI)[[0, 1]].any()   # only clipped samples touch these rows


# ---------------------------------------------------------------------------------------------------- whole steps
def _vae_params(m, code):
    H, I = m.H, m.I
    g = lambda k: host(m.P[k])
    return {"W1": g("W1"), "b1": g("b1")[:H], "W2": g("W2").T, "b2": g("b2")[:code], "W3": g("W3").T, "b3": g("b3")[:H],
            "W4": g("W4").T, "b4": g("b4")[:I]}


def _big_vae_case(cls, drop, code_is_2l, seed):
    I, H, L, B, nu = 26744, 600, 200, 500, 900
    rs = np.random.RandomState(seed)
    rows = random_rows(rs, nu, I, list(rs.randint(1, 300, size=97)) + [0])
    indptr, indices = csr_from_rows(rows)
    m = cls(I, H, L, 1e-3, drop, 0.01, 11, dev(indptr), dev(indices), DEV)
    for k in ("b1", "b2", "b3", "b4"):
        m.P[k].normal_(0, 0.05)
    m._refresh()
    batch = rs.choice(nu, B, replace=False).astype(np.int32)
    X = np.zeros((B, I))
    for b, u in enumerate(batch):
        X[b, rows[u]] = 1
    return m, indptr, indices, batch, X, _vae_params(m, 2 * L if code_is_2l else L)


def _check_grads(m, G, ni, H, code, tol):
    for k, tr in (("W4", True), ("W3", True), ("W2", True), ("W1", False)):
        assert rel(host(m.G[k]), G[k].T if tr else G[k]) < tol, k
    for k, n in (("b4", ni), ("b3", H), ("b2", code), ("b1", H)):
        assert rel(host(m.G[k])[:n], G[k]) < tol, k


@pytest.mark.parametrize("drop", [0.0, 0.5])
def test_native_multivae_step_at_the_reference_shape(drop):
    """eb_vae_train_step (the production path) at I=26744, H=600, L=200, B=500 against the fp64 restatement fed with the
    restated dropout mask and noise: bf16 tolerances (loss 2e-2, gradients 5e-2 relative Frobenius)."""
    from elliot_b200.recommender.multi_vae import VariationalAutoEncoder
    m, indptr, indices, batch, X, P = _big_vae_case(VariationalAutoEncoder, drop, True, 21)
    assert m.native
    sid, anneal, L = 3, 0.13, m.L
    m._acc.zero_()
    m.compute_grads(dev(batch), anneal, sid)
    keep = ph.csr_keep_mask(m.seed * 7919 + sid, indptr, indices, batch, m.I, drop) if drop else None
    eps = ph.reparam_eps(m.seed, sid, len(batch) * L).reshape(len(batch), L)
    loss_ref, G, (_, _, _, _, nll_ref, kl_ref) = tfm.multivae_forward_backward(P, X, eps, anneal, keep=keep, rate=drop)
    kl_sum, nll_sum = m._acc.tolist()
    B = len(batch)
    loss = nll_sum / B + anneal * (-0.5 * kl_sum / (B * L))
    assert abs(loss - loss_ref) < 2e-2 * abs(loss_ref)
    assert abs(-0.5 * kl_sum / (B * L) - kl_ref) < 2e-2 * abs(kl_ref) + 1e-6
    _check_grads(m, G, m.I, m.H, 2 * L, 5e-2)


def test_multidae_step_with_dropout_at_the_reference_shape():
    from elliot_b200.recommender.multi_dae import DenoisingAutoEncoder
    drop = 0.2
    m, indptr, indices, batch, X, P = _big_vae_case(DenoisingAutoEncoder, drop, False, 22)
    sid = 4
    m._acc.zero_()
    m.compute_grads(dev(batch), 0.0, sid)
    keep = ph.csr_keep_mask(m.seed * 7919 + sid, indptr, indices, batch, m.I, drop)
    loss_ref, G, _ = tfm.multidae_forward_backward(P, X, keep=keep, rate=drop)
    assert abs(m._acc[1].item() / len(batch) - loss_ref) < 2e-2 * abs(loss_ref)
    _check_grads(m, G, m.I, m.H, m.L, 5e-2)


def _neumf_big_step(exact):
    from elliot_b200.recommender.neumf import NeuralMatrixFactorizationModel
    nu, ni, f, B = 6040, 3706, 16, 1 << 20
    with ops.exact_gemm(exact):
        m = NeuralMatrixFactorizationModel(nu, ni, f, 1e-3, 42, DEV)
        gen = torch.Generator(device=DEV); gen.manual_seed(3)           # the same step on every run
        for k in ("b1", "b2", "b3", "bp"):
            m.P[k].normal_(0, 0.05, generator=gen)
        for k in ("U_mf", "I_mf", "U_mlp", "I_mlp"):
            m.P[k].mul_(4.0)
        m._refresh()
        g = lambda k: host(m.P[k])
        P = {"U_mf": g("U_mf"), "I_mf": g("I_mf"), "U_mlp": g("U_mlp"), "I_mlp": g("I_mlp"), "W1": g("W1").T, "b1": g("b1")[:4 * f],
             "W2": g("W2").T, "b2": g("b2")[:2 * f], "W3": g("W3").T, "b3": g("b3")[:f], "wp": g("wp"), "bp": float(g("bp")[0])}
        rs = np.random.RandomState(5)
        u = rs.randint(0, nu, B).astype(np.int32); i = rs.randint(0, ni, B).astype(np.int32)
        y = (rs.rand(B) < 0.2).astype(np.float32)
        loss_ref, G, _ = tfm.neumf_forward_backward(P, u, i, y.astype(np.float64))
        loss = m.train_step((dev(u), dev(i), dev(y))).item()
    M = lambda k: host(m.M[k]) / 0.1                                      # first Adam step: m = 0.1 g
    return m, f, loss, loss_ref, G, M


def test_neumf_whole_epoch_batch_is_exact_with_the_fp32_checking_gemm():
    """batch_size -1 on a 1 M-interaction epoch: B = 2^20 samples in one step.  The bias gradients take the multi-slab
    colsum, the weight gradients contract over K = 2^20; on the fp32 checking GEMM every gradient agrees to 1e-4."""
    m, f, loss, loss_ref, G, M = _neumf_big_step(True)
    assert abs(loss - loss_ref) < 1e-5 * abs(loss_ref)
    for k in ("W3", "W2", "W1"):
        assert rel(M(k), G[k].T) < 1e-4, k
    for k, n in (("b3", f), ("b2", 2 * f), ("b1", 4 * f)):
        assert rel(M(k)[:n], G[k]) < 1e-4, k
    assert rel(M("wp"), G["wp"]) < 1e-4 and abs(M("bp")[0] - G["bp"]) < 1e-4 * abs(G["bp"]) + 1e-7
    for k in ("U_mf", "I_mf", "U_mlp", "I_mlp"):
        assert rel(M(k), G[k]) < 1e-4, k


def test_neumf_whole_epoch_batch_on_the_tensor_cores():
    """The same step on the bf16 path (split-K weight gradients over K = 2^20) at the tolerances of
    test_gpu_neumf.py::test_train_step_matches_restatement."""
    m, f, loss, loss_ref, G, M = _neumf_big_step(False)
    assert abs(loss - loss_ref) < 1e-2 * abs(loss_ref)
    for k, tol in (("W3", 5e-2), ("W2", 6e-2), ("W1", 1e-1)):
        assert rel(M(k), G[k].T) < tol, k
    for k, n, tol in (("b3", f, 5e-2), ("b2", 2 * f, 6e-2), ("b1", 4 * f, 1e-1)):
        assert rel(M(k)[:n], G[k]) < tol, k
    assert rel(M("wp"), G["wp"]) < 2e-2 and abs(M("bp")[0] - G["bp"]) < 2e-2 * abs(G["bp"]) + 1e-6
    for k, tol in (("U_mf", 2e-2), ("I_mf", 2e-2), ("U_mlp", 1e-1), ("I_mlp", 1e-1)):
        assert rel(M(k), G[k]) < tol, k


@pytest.mark.parametrize("M,N,K", [(77, 600, 3001), (512, 600, 26744)])
def test_split_k_gemm_is_bit_reproducible(M, N, K):
    """dh2 = dlogits . W4 (few output tiles, long K) splits K over the SMs; its partial tiles are summed in a fixed order, so
    repeated runs give the same bits.  (Atomic accumulation would move last bits from run to run, and the bf16 operand copy
    of the result by a whole bf16 ulp: enough to make two identical training steps diverge.)"""
    g = torch.Generator(device=DEV); g.manual_seed(M + K)
    A = ops.to_bf16(torch.randn(M, K, device=DEV, generator=g) / K ** 0.5)
    B = ops.to_bf16(torch.randn(K, N, device=DEV, generator=g))
    first = ops.gemm_bf16(A, B, M, N, K, b_rows_are_k=True)
    for _ in range(5):
        assert torch.equal(ops.gemm_bf16(A, B, M, N, K, b_rows_are_k=True), first)
    ref = A.double()[:, :K] @ B.double()[:, :N]
    assert (first.double() - ref).abs().max().item() <= gamma(K) * (A.double()[:, :K].abs() @ B.double()[:, :N].abs()).max().item()
