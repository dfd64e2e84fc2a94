"""The host restatement of MF2020's throughput-mode launch (oracle/mf2020_hogwild.py): the visiting order is a
permutation of the epoch, the stream holds every positive once with m negatives under its user, the gcd loop is
exercised, and one sample's update is the sequential reference's (oracle.mf2020_update_seq)."""
import math

import numpy as np
import pytest

import oracle
from oracle import mf2020_hogwild as hw


@pytest.mark.parametrize("n", [2, 4096, 999, 30011, 7 * 11 * 13 * 17, 1 << 20])       # even, odd, prime, composite
@pytest.mark.parametrize("seed, epoch", [(11, 0), (11, 1), (0xDEADBEEF12345, 7)])
def test_visiting_order_is_a_bijection(n, seed, epoch):
    mul, add, _ = hw.visit_order(seed, epoch, n)
    assert math.gcd(mul, n) == 1 and mul % 2 == 1 and 0 <= add < n
    sp = hw.epoch_slots(seed, epoch, n, 0, n)
    assert np.array_equal(np.sort(sp), np.arange(n, dtype=np.uint64))
    # windows are slices of the same order
    assert np.array_equal(hw.epoch_slots(seed, epoch, n, n // 3, n - n // 3), sp[n // 3:])


def test_gcd_loop_iterates():
    epoch = 2
    seed = next(s for s in range(1000) if hw.initial_multiplier(s, epoch) % 15 == 0)   # shares 3 and 5 with n below
    mul0 = hw.initial_multiplier(seed, epoch)
    assert (1 << 22) <= mul0 < (1 << 23) and mul0 % 2 == 1
    for n in (3 * 1000, 15 * 4099, 2 * mul0):
        mul, _, steps = hw.visit_order(seed, epoch, n)
        assert steps >= 1 and mul == mul0 + 2 * steps and math.gcd(mul, n) == 1, n
    n = 15 * 4099
    assert np.array_equal(np.sort(hw.epoch_slots(seed, epoch, n, 0, n)), np.arange(n, dtype=np.uint64))
    # n coprime with the first draw: no iteration
    assert hw.visit_order(seed, epoch, 1 << 20)[2] == 0


@pytest.mark.parametrize("m", [0, 1, 3])
def test_stream_holds_every_positive_once_with_m_negatives(m):
    rs = np.random.RandomState(m)
    n_users, n_items, n_pos = 60, 97, 700
    pos_u = np.sort(rs.randint(0, n_users, n_pos)).astype(np.int32)
    pos_i = rs.randint(0, n_items, n_pos).astype(np.int32)
    for epoch in (0, 1):
        u, i, r = hw.sample_stream(pos_u, pos_i, m, n_items, 5, epoch)
        assert len(u) == n_pos * (1 + m) and set(np.unique(r)) <= {0, 1}
        got = np.stack([u[r == 1], i[r == 1]], 1)
        want = np.stack([pos_u, pos_i], 1)
        assert np.array_equal(got[np.lexsort((got[:, 1], got[:, 0]))], want[np.lexsort((want[:, 1], want[:, 0]))])
        assert np.array_equal(np.bincount(u[r == 0], minlength=n_users), m * np.bincount(pos_u, minlength=n_users))
        assert i.min() >= 0 and i.max() < n_items
        # a window is the same stream
        w = hw.sample_stream(pos_u, pos_i, m, n_items, 5, epoch, first=123, count=200)
        assert all(np.array_equal(a, b[123:323]) for a, b in zip(w, (u, i, r)))
    # the negatives are the restated Philox draws of their slot
    sp = hw.epoch_slots(5, 1, n_pos * (1 + m), 0, n_pos * (1 + m))
    if m:
        neg = sp % np.uint64(1 + m) != 0
        x = oracle.philox.gen(5, np.uint64(n_pos * (1 + m)) + sp[neg], 0)[0]
        assert np.array_equal(i[neg], (x.astype(np.uint64) * np.uint64(n_items) >> np.uint64(32)).astype(np.int32))


def test_one_sample_launch_is_the_sequential_reference_step():
    """A launch of one sample reads nothing stale: its row updates are MF_model.train_step's (the item row sees the
    updated user row), and its global bias is the closed form, which for one sample differs from the plain step
    gb + lr (g - reg gb) only in the second order of lr."""
    rs = np.random.RandomState(2)
    d, lr, reg = 7, 0.05, 0.01
    U, V = rs.normal(0, 0.3, (4, d)), rs.normal(0, 0.3, (5, d))
    ub, ib, gb0 = rs.normal(0, 0.2, 4), rs.normal(0, 0.2, 5), 0.17
    for r in (0, 1):
        u, i = np.array([2]), np.array([3])
        got = hw.apply_launch(U, V, ub, ib, gb0, u, i, np.array([float(r)]), lr, reg)
        Us, Vs, ubs, ibs = U.copy(), V.copy(), ub.copy(), ib.copy()
        gb_seq, bl = oracle.mf2020_update_seq(Us, Vs, ubs, ibs, gb0, u, i, np.array([r]), lr, reg)
        for k, want in (("U", Us), ("V", Vs), ("ub", ubs), ("ib", ibs)):
            assert np.abs(got[k] - want).max() < 1e-15, k
        assert abs(got["loss"] - bl.sum()) < 1e-14
        assert abs(got["gb"] - gb_seq) < lr * lr * (got["hsum"] + reg) * abs(got["grad"][0] - reg * gb0)
        assert got["gb"] != gb_seq


def test_global_bias_finish_limits():
    # small lr c: the plain summed step; large: the launch's fixed point gb0 + (gbar - reg gb0) / k
    gb0, gsum, hsum, c, reg = 0.3, -12.0, 40.0, 200, 0.01
    plain = gb0 + 1e-9 * (gsum - reg * gb0 * c)
    assert abs(hw.global_bias_finish(gb0, gsum, hsum, c, 1e-9, reg) - plain) < 1e-15
    k = hsum / c + reg
    assert abs(hw.global_bias_finish(gb0, gsum, hsum, c, 10.0, reg) - (gb0 + (gsum / c - reg * gb0) / k)) < 1e-12
    assert hw.global_bias_finish(gb0, gsum, hsum, 0, 0.1, reg) == gb0
    # k = 0 (no curvature, no regularisation): the linear step lr c gbar
    assert hw.global_bias_finish(gb0, gsum, 0.0, c, 0.1, 0.0) == gb0 + gsum / c * 0.1 * c
