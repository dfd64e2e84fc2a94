"""Schedule prefetch of the grouped sampled BPR step (ops.set_bpr_prefetch): the next call's key pass and sort run on a side
stream while the current update runs.  A prefetched order is used only by the call it was made for; whichever order a call
applies, it emits the sampler's triples."""
import ctypes

import numpy as np
import pytest
import torch

from elliot_b200 import ops
from elliot_b200._lib import check, lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HP = (0.05, 0.0025, 0.01, 0.0025, 0.00025)


def _csr(rows):
    indptr = torch.tensor(np.cumsum([0] + [len(r) for r in rows]), dtype=torch.int64, device=DEV)
    idx = torch.tensor([x for r in rows for x in sorted(r)], dtype=torch.int32, device=DEV)
    return indptr, idx


def _rows(nu, ni, seed):
    rs = np.random.RandomState(seed)
    return [rs.choice(ni, rs.randint(1, 40), replace=False) for _ in range(nu)]


def _tables(nu, ni, d, seed):
    ld = ops.padded_dim(d)
    g = torch.Generator(device=DEV); g.manual_seed(seed)
    U = torch.zeros((nu, ld), device=DEV); U[:, :d] = torch.randn(nu, d, device=DEV, generator=g) * 0.1
    V = torch.zeros((ni, ld), device=DEV); V[:, :d] = torch.randn(ni, d, device=DEV, generator=g) * 0.1
    b = torch.randn(ni, device=DEV, generator=g) * 0.05
    return U, V, b


def _step(U, V, b, d, nu, ni, indptr, idx, n, seed, first, hp=HP, **kw):
    out = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
    ops.bpr_step_sampled_f32(U, V, b, d, nu, ni, indptr, idx, n, seed, first, *hp, out=out, **kw)
    return out


@pytest.fixture
def schedules(monkeypatch):
    """Prefetch on, and a log of every schedule enqueued: (first, made on the side stream)."""
    was = ops.set_bpr_prefetch(True)
    log = []
    orig = ops._Schedules._schedule

    def spy(self, s, n_users, n_items, indptr, n, seed, first, flags, stream):
        log.append((first, stream == self.side))
        return orig(self, s, n_users, n_items, indptr, n, seed, first, flags, stream)
    monkeypatch.setattr(ops._Schedules, "_schedule", spy)
    yield log
    ops.set_bpr_prefetch(was)


def test_consecutive_calls_emit_the_same_triples_with_prefetch_on_and_off(schedules):
    nu, ni, d, n = 3000, 700, 32, 40_000
    indptr, idx = _csr(_rows(nu, ni, 1))
    emitted = {}
    for on in (False, True):
        ops.set_bpr_prefetch(on)
        U, V, b = _tables(nu, ni, d, 2)
        emitted[on] = [_step(U, V, b, d, nu, ni, indptr, idx, n, 7, k * n) for k in range(6)]
        torch.cuda.synchronize()
        assert torch.isfinite(U).all() and torch.isfinite(V).all()
    for k in range(6):
        want = ops.bpr_sample_philox(nu, ni, indptr, idx, n, 7, k * n)
        for a, c, w in zip(emitted[False][k], emitted[True][k], want):
            assert torch.equal(a, w) and torch.equal(c, w), k
    # inline schedules for the first two calls only; from the second call on, each call prefetches the next
    assert [f for f, side in schedules if not side] == [0, n]
    assert [f for f, side in schedules if side] == [k * n for k in range(2, 7)]


@pytest.mark.parametrize("d", [16, 64])
def test_prefetched_step_is_bitwise_the_serial_step_without_conflicts(schedules, d):
    """The conflict-free batch of test_gpu_bpr_grouped (every user run one triple): the tables after a call that applies a
    prefetched order are bit-identical to those the serial step leaves.  Two lr = 0 calls (which leave the tables bit-identical)
    before it make the call at `first` a consecutive one."""
    nu = ni = 1 << 22
    n, first = 256, 1 << 20
    indptr = torch.arange(nu + 1, dtype=torch.int64, device=DEV)
    idx = torch.arange(nu, dtype=torch.int32, device=DEV)
    for seed in range(1, 40):
        u, i, j = (x.cpu().numpy() for x in ops.bpr_sample_philox(nu, ni, indptr, idx, n, seed, first))
        if len(np.unique(u)) == n and len(np.unique(np.concatenate([i, j]))) == 2 * n:
            break
    else:
        pytest.fail("no conflict-free seed")
    U0, V0, b0 = _tables(nu, ni, d, d)
    for racy in (False, True):
        tabs = {}
        for on in (False, True):
            ops.set_bpr_prefetch(on)
            U, V, b = U0.clone(), V0.clone(), b0.clone()
            for f in (first - 2 * n, first - n):
                _step(U, V, b, d, nu, ni, indptr, idx, n, seed, f, hp=(0.0,) + HP[1:], racy=racy)
            del schedules[:]
            out = _step(U, V, b, d, nu, ni, indptr, idx, n, seed, first, racy=racy)
            torch.cuda.synchronize()
            assert np.array_equal(out[0].cpu().numpy(), u) and np.array_equal(out[2].cpu().numpy(), j)
            tabs[on] = (U, V, b)
            if on:
                assert schedules == [(first + n, True)]          # the call's own order was the prefetched one
        assert not torch.equal(tabs[True][0], U0)
        for a, c in zip(tabs[False], tabs[True]):
            assert torch.equal(a, c), racy
        del tabs


def test_prefetched_order_is_not_used_by_a_different_call(schedules):
    """After two consecutive calls the slot holds the order of first + n.  A call with another seed, another n, a first that
    does not continue, or after indptr and indices were edited in place schedules inline; every call emits the sampler's
    triples."""
    nu, ni, d, n = 2000, 500, 16, 30_000
    rows = _rows(nu, ni, 3)
    indptr, idx = _csr(rows)
    ip_b, ix_b = _csr(rows[1:] + rows[:1])                     # the same rows, owned by other users
    assert not torch.equal(ip_b, indptr)
    U, V, b = _tables(nu, ni, d, 5)

    def call(seed, first, m=n):
        del schedules[:]
        out = _step(U, V, b, d, nu, ni, indptr, idx, m, seed, first)
        want = ops.bpr_sample_philox(nu, ni, indptr, idx, m, seed, first)
        assert all(torch.equal(a, w) for a, w in zip(out, want)), (seed, first, m)
        return [f for f, side in schedules if not side]

    call(1, 0); call(1, n)                                      # the slot now holds first = 2n
    assert call(2, 2 * n) == [2 * n]                            # other seed
    call(1, 2 * n); call(1, 3 * n)
    assert call(1, 4 * n, n // 2) == [4 * n]                    # other n
    call(1, 5 * n); call(1, 6 * n)
    assert call(1, 9 * n) == [9 * n]                            # a jump
    call(1, 10 * n); call(1, 11 * n)
    indptr.copy_(ip_b); idx.copy_(ix_b)                         # an in-place edit of the CSR
    assert call(1, 12 * n) == [12 * n]
    assert call(1, 13 * n) == []                                # consecutive again: prefetched on the edited CSR
    assert torch.isfinite(U).all() and torch.isfinite(V).all()


def test_apply_emits_the_sampler_triples_for_any_order():
    """The apply entry fed on purpose with an order scheduled for other inputs (another seed and first), or with a random
    permutation, still samples and emits exactly the triples of its own call."""
    nu, ni, d, n = 1500, 400, 16, 20_000
    indptr, idx = _csr(_rows(nu, ni, 6))
    ws = torch.empty(int(lib().eb_bpr_step_sampled_workspace_bytes(n, nu)), dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    off = ctypes.c_size_t(0)
    check(lib().eb_bpr_schedule_sampled(nu, ni, indptr.data_ptr(), n, 99, 12345, ws.data_ptr(), ws.numel(), ctypes.byref(off), 0, st))
    stale = ws[off.value:off.value + 4 * n].view(torch.int32).clone()
    assert torch.equal(torch.sort(stale.long()).values, torch.arange(n, device=DEV))
    for order in (stale, torch.randperm(n, device=DEV).to(torch.int32)):
        U, V, b = _tables(nu, ni, d, 7)
        out = [torch.empty(n, dtype=torch.int32, device=DEV) for _ in range(3)]
        check(lib().eb_bpr_apply_sampled_filter_f32(U.data_ptr(), V.data_ptr(), b.data_ptr(), d, U.stride(0), nu, ni,
                                                    indptr.data_ptr(), idx.data_ptr(), None, 0, n, 3, 500, *HP, None,
                                                    *(x.data_ptr() for x in out), order.data_ptr(), 0, st))
        want = ops.bpr_sample_philox(nu, ni, indptr, idx, n, 3, 500)
        assert all(torch.equal(a, w) for a, w in zip(out, want))
        assert torch.isfinite(U).all() and torch.isfinite(V).all()
