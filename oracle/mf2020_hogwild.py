"""Host restatement of one MF2020 throughput-mode launch (eb_mf_pointwise_step_f32, elliot_b200/csrc/mf2020.cu).
TEST INFRASTRUCTURE ONLY, in the style of oracle/philox.py.

The sample stream of an epoch:
  - `visit_order`: the affine visiting order s -> (s mul + add) mod n of the epoch (mul coprime with n, found by the same
    gcd loop as the device), with the multiplier and offset derived from (seed, epoch) in 64-bit wrapping arithmetic;
  - `sample_stream`: the (user, item, label) of positions [first, first + count): epoch slot sp = (s mul + add) mod n, the
    positive sp // (1 + m), slot sp mod (1 + m) = 0 is the positive itself (label 1), slots 1..m a uniform item
    bounded(Philox(seed, epoch n + sp, 0)[0], n_items) (label 0), with Philox from oracle/philox.py.
`apply_launch` applies one launch in fp64 with Hogwild's staleness made exact: every sample reads the tables as they
were before the launch and the global bias is the launch's starting value gb0; the row updates of all samples are
summed, and the global bias takes the closed-form finish of mf_global_bias_finish_kernel from the launch's sums.
"""
import math

import numpy as np

from . import philox

MASK64 = (1 << 64) - 1


def initial_multiplier(seed, epoch):
    """The odd multiplier in [2^22, 2^23) drawn from (seed, epoch), before it is made coprime with n."""
    h = (0x9E3779B97F4A7C15 ^ ((seed * 0xD1B54A32D192ED03 + epoch) & MASK64)) & MASK64
    return ((h >> 20) & 0x3FFFFF) | 0x400001


def visit_order(seed, epoch, n):
    """(mul, add, steps) of the epoch's affine order over n samples; steps counts the gcd loop's increments of mul."""
    mul, steps = initial_multiplier(seed, epoch), 0
    while math.gcd(mul, n) != 1:
        mul += 2
        steps += 1
    add = ((seed * 0x2545F4914F6CDD1D + epoch * 0x632BE59BD9B4E019) & MASK64) % n
    return mul, add, steps


def epoch_slots(seed, epoch, n, first, count):
    """Epoch slots sp of the positions first .. first + count - 1 (uint64; s mul < 2^40 2^23 never wraps)."""
    mul, add, _ = visit_order(seed, epoch, n)
    s = np.arange(first, first + count, dtype=np.uint64)
    return (s * np.uint64(mul) + np.uint64(add)) % np.uint64(n)


def sample_stream(pos_u, pos_i, m, n_items, seed, epoch, first=0, count=None):
    """(u, i, r) int32 arrays of positions [first, first + count) of the epoch (count None: to the end)."""
    pos_u, pos_i = np.asarray(pos_u), np.asarray(pos_i)
    n = len(pos_u) * (1 + m)
    if count is None:
        count = n - first
    sp = epoch_slots(seed, epoch, n, first, count)
    pos = (sp // np.uint64(1 + m)).astype(np.int64)
    q = sp % np.uint64(1 + m)
    u = pos_u[pos].astype(np.int32)
    x = philox.gen(seed, np.uint64(epoch * n) + sp, 0)[0]
    neg = ((x.astype(np.uint64) * np.uint64(n_items)) >> np.uint64(32)).astype(np.int32)
    i = np.where(q == 0, pos_i[pos], neg).astype(np.int32)
    return u, i, (q == 0).astype(np.int32)


def global_bias_finish(gb0, gsum, hsum, c, lr, reg):
    """mf_global_bias_finish_kernel: gb0 + (gbar - reg gb0) (1 - exp(-lr k c)) / k, gbar = gsum / c, k = hsum / c + reg."""
    if c <= 0:
        return gb0
    gbar, k = gsum / c, hsum / c + reg
    gain = -math.expm1(-lr * k * c) / k if k > 1e-12 else lr * c
    return gb0 + (gbar - reg * gb0) * gain


def apply_launch(U, V, ub, ib, gb0, u, i, r, lr, reg):
    """One launch over the samples (u, i, r) in fp64, every sample reading the pre-launch tables (U, V: rows of the
    factors, ub, ib: the biases; not modified).  Returns dict with U, V, ub, ib (new tables), gb, loss, and the launch's
    sums gsum = sum grad, hsum = sum sig (1 - sig) and per-sample pred, sig, grad."""
    a, b = U[u], V[i]
    pred = gb0 + ub[u] + ib[i] + (a * b).sum(1)
    sig = 1.0 / (1.0 + np.exp(-pred))
    grad = r - sig
    du = lr * (grad[:, None] * b - reg * a)
    dv = lr * (grad[:, None] * (a + du) - reg * b)                 # the item row sees the updated user row
    out = {"U": U.copy(), "V": V.copy(), "ub": ub.copy(), "ib": ib.copy()}
    np.add.at(out["U"], u, du)
    np.add.at(out["V"], i, dv)
    np.add.at(out["ub"], u, lr * (grad - reg * ub[u]))
    np.add.at(out["ib"], i, lr * (grad - reg * ib[i]))
    gsum, hsum = grad.sum(), (sig * (1 - sig)).sum()
    out["gb"] = global_bias_finish(gb0, gsum, hsum, len(u), lr, reg)
    out["loss"] = (np.maximum(pred, 0) - r * pred + np.log1p(np.exp(-np.abs(pred)))).sum()
    out.update(gsum=gsum, hsum=hsum, pred=pred, sig=sig, grad=grad, du=du, dv=dv)
    return out
