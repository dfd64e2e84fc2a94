"""Torch-tensor wrappers over the C ABI.  Torch is plumbing only (device memory, streams);
all arithmetic happens in elliot_b200/csrc/*.cu.  Every op raises if its tensors are not on a
CUDA device — there is no CPU path.

Streams: every op launches on torch's CURRENT stream of the tensors' device.  The C ABI never allocates, so these ops
keep grow-only scratch per device from call to call (_scratch): bpr_exact_f64, MtSampler.step, MtPointwiseRatioSampler.step, score_topk,
score_topk_tc, bpr_step_sampled_f32 (the schedule prefetch keeps two schedule slots of its own), gram_f64, eval_topk,
eval_topk_metrics, eval_fairness, vae_train_step, gemm_bf16_tn / gemm_bf16 (split-K partials), cml_grad_f32, dmf_head_f32, autorec_decoder_f32 and RandomStream.draws; mf_pointwise_step_f32 keeps a global-bias accumulator per
device.  Those ops must not run concurrently on two streams of the same device from one process.
"""
import ctypes
import os

import torch

from ._lib import check, lib

F32_STRIDES = (8, 16, 32, 64, 128, 256)


def padded_dim(d):
    """Row stride (in elements) the fp32 kernels need for `d` factors."""
    for s in F32_STRIDES:
        if d <= s:
            return s
    raise ValueError(f"factors={d} > 256 is not supported by the fp32 kernels")


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _stream(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("elliot_b200 ops need CUDA tensors (no CPU fallback exists)")


def _chk_idx(*ts):
    for t in ts:
        if t.dtype != torch.int32 or not t.is_contiguous():
            raise TypeError("index tensors must be contiguous int32")


def _chk_f64_rows(*ts):
    """fp64 row blocks: 2-D with unit column stride, so row-strided views pass."""
    for t in ts:
        if t.dtype != torch.float64 or t.dim() != 2 or t.stride(1) != 1:
            raise TypeError("fp64 blocks must be 2-D with unit column stride")


def _chk_f64_dense(*ts):
    """fp64 dense arrays: contiguous."""
    for t in ts:
        assert t.dtype == torch.float64 and t.is_contiguous()


def _nonempty(t):
    """The C ABI takes no NULL arrays: an empty one is passed as a one-element dummy."""
    return t if t.numel() else torch.zeros(1, dtype=t.dtype, device=t.device)


def _call(name, dev_tensor, *args):
    """Entry point `name` on dev_tensor's device, with that device's current stream appended as the last argument."""
    with torch.cuda.device(dev_tensor.device):
        check(getattr(lib(), name)(*args, _stream(dev_tensor)))


_scratch_bufs = {}


def _scratch(name, nbytes, device):
    """Grow-only device scratch of at least nbytes (and 256) bytes, one buffer per (name, device) kept from call to call;
    only ever used on the caller's current stream."""
    key = (name, device.index)
    buf = _scratch_bufs.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = _scratch_bufs[key] = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
    return buf


def _topk_out(users, n_rows, user_begin, n_sel, k, dtype, device):
    """(n_sel, idx int32 [n_sel][k], val [n_sel][k]) of a top-k over the int32 ids `users`, or else over the rows
    user_begin .. user_begin + n_sel (n_sel None: to the last of n_rows rows)."""
    if users is not None:
        _chk_idx(users)
        n_sel = users.numel()
    elif n_sel is None:
        n_sel = n_rows - user_begin
    return (n_sel, torch.empty((n_sel, k), dtype=torch.int32, device=device),
            torch.empty((n_sel, k), dtype=dtype, device=device))


def _bpr_flags(racy=False, sync=True, variant=0, deterministic=False, reserve_sms=0):
    """The flags word of the eb_bpr_step_* entry points: bit 0 plain stores (racy Hogwild), bit 1 no synchronise (host
    triples), bits 4-5 kernel variant (16 or 32), bit 6 deterministic rounds, bits 8-15 SMs the grid leaves free."""
    return ((1 if racy else 0) | (0 if sync else 2) | int(variant) | (64 if deterministic else 0)
            | ((int(reserve_sms) & 0xff) << 8))


def _out_ptrs(out):
    """Device pointers of an optional out=(u, i, j) triple of contiguous int32 tensors (NULLs when out is None)."""
    if out is None:
        return 0, 0, 0
    u, i, j = out
    _need_cuda(u, i, j); _chk_idx(u, i, j)
    return _ptr(u), _ptr(i), _ptr(j)


def device_info():
    sm = ctypes.c_int(0); cc = ctypes.c_int(0)
    check(lib().eb_device_info(ctypes.byref(sm), ctypes.byref(cc)))
    return sm.value, cc.value


def bpr_step_f32(U, V, b, d, tu, ti, tj, lr, reg_u, reg_b, reg_pos, reg_neg, loss=None, racy=False, deterministic=False):
    """Throughput-mode BPR step on materialised triples (BPRMF_model.py:87-117 semantics)."""
    _need_cuda(U, V, b, tu, ti, tj, loss)
    _chk_idx(tu, ti, tj)
    assert U.dtype == torch.float32 and V.dtype == torch.float32 and b.dtype == torch.float32
    assert U.stride(1) == 1 and V.stride(1) == 1 and U.stride(0) == V.stride(0)
    _call("eb_bpr_step_f32", U, _ptr(U), _ptr(V), _ptr(b), d, U.stride(0), _ptr(tu), _ptr(ti), _ptr(tj), tu.numel(), lr, reg_u,
          reg_b, reg_pos, reg_neg, _ptr(loss), _bpr_flags(racy=racy, deterministic=deterministic))


def bloom_build(indptr, indices, n_users, words=32):
    """Per-user membership signatures for the fused sampler (32*words bits each, see eb_bloom_build): uint32 [n_users, words]
    (kept as int32 storage).  With them the sampler draws EXACTLY the same triples, just with a shorter load chain."""
    _need_cuda(indptr, indices)
    assert indptr.dtype == torch.int64 and indices.dtype == torch.int32
    out = torch.empty((n_users, words), dtype=torch.int32, device=indptr.device)
    _call("eb_bloom_build", indptr, _ptr(indptr), _ptr(indices), n_users, words, _ptr(out))
    return out


def bpr_step_sampled_f32(U, V, b, d, n_users, n_items, indptr, indices, n, seed, first, lr, reg_u, reg_b, reg_pos,
                         reg_neg, loss=None, out=None, racy=False, reserve_sms=0, filter=None, deterministic=False, _variant=0):
    """Fused sample+update step (custom_sampler.py:24-46 distribution, Philox stream).  filter: bloom_build() output.
    The default free-running Hogwild step applies the triples grouped by user (key pass, stable sort, update; see
    eb_bpr_step_sampled_f32) with device workspace of this module.  Once two calls in a row have advanced `first` by
    exactly `n`, each call also schedules the next one (key pass and sort) on a side stream while its own update runs;
    the next call uses that schedule only if it asks for exactly those triples on the same, unmodified CSR
    (set_bpr_prefetch).  Which triples are drawn and how they are applied does not depend on it.
    deterministic: run the launch in rounds (reads, grid barrier, atomic adds, grid barrier) so the same inputs give the same
    tables on every run up to fp32 summation order; slower than the default free-running Hogwild.
    _variant (profiling): one table always runs the register-staged kernel (16 or 0); 32, the shared-memory-staged kernel,
    exists for sharded item tables only and is refused here."""
    _need_cuda(U, V, b, indptr, indices, loss, filter)
    assert indptr.dtype == torch.int64 and indices.dtype == torch.int32
    out = _out_ptrs(out)
    flags = _bpr_flags(racy=racy, variant=_variant, deterministic=deterministic, reserve_sms=reserve_sms)
    fw = 0 if filter is None else filter.shape[1]
    if _prefetch_on and not deterministic and not _variant and 1 <= n <= _SCHEDULE_MAX:
        with torch.cuda.device(U.device):
            _schedules_of(U.device).step(U, V, b, d, n_users, n_items, indptr, indices, filter, fw, n, seed, first,
                                         (lr, reg_u, reg_b, reg_pos, reg_neg), loss, out, flags)
        return
    ws = None
    if not deterministic:
        ws = _scratch("bpr_grouped", lib().eb_bpr_step_sampled_workspace_bytes(n, n_users), U.device)
    _call("eb_bpr_step_sampled_filter_f32", U, _ptr(U), _ptr(V), _ptr(b), d, U.stride(0), n_users, n_items, _ptr(indptr),
          _ptr(indices), _ptr(filter), fw, n, seed, first, lr, reg_u, reg_b, reg_pos, reg_neg, _ptr(loss), *out, _ptr(ws),
          0 if ws is None else ws.numel(), flags)


# ---- schedule prefetch of the grouped sampled step
_SCHEDULE_MAX = 2**31 - 1                     # longer calls run as sub-steps inside eb_bpr_step_sampled_f32
_prefetch_on = os.environ.get("EB_BPR_PREFETCH", "1") != "0"
_schedules = {}


def set_bpr_prefetch(enabled):
    """Schedule prefetch of bpr_step_sampled_f32 on (the default; EB_BPR_PREFETCH=0 starts with it off) or off.  Off, every
    call schedules and applies on the caller's stream as eb_bpr_step_sampled_f32 does, and the schedule slots are freed.
    Returns the previous setting."""
    global _prefetch_on
    was, _prefetch_on = _prefetch_on, bool(enabled)
    if not enabled:
        for s in _schedules.values():
            s.release()
        _schedules.clear()
    return was


def _schedules_of(device):
    i = device.index if device.index is not None else torch.cuda.current_device()
    if i not in _schedules:
        _schedules[i] = _Schedules(torch.device("cuda", i))
    return _schedules[i]


class _Schedules:
    """Two schedule slots of one device (workspace of eb_bpr_schedule_sampled each: user keys and triple indices,
    double-buffered for the sort, 16 B per triple + cub's storage) and the side stream that fills them ahead of time.

    A call applies the order in one slot.  When it continues the previous call (first advanced by exactly n), it then
    enqueues the schedule of first + n into the other slot on the side stream: after an event recorded on the caller's
    stream just before the apply (everything the caller enqueued earlier, CSR edits included, is visible) and after the
    last apply that read that slot.  The next call takes the slot if its key matches, waiting on the slot's event;
    otherwise it schedules inline.  The key holds the CSR tensors' version counters, so an in-place edit of indptr or
    indices invalidates a prefetched order."""

    def __init__(self, device):
        self.device = device
        self.side = torch.cuda.Stream(device)
        self.buf = [None, None]
        self.off = [0, 0]
        self.key = [None, None]            # call a slot's pending prefetched order was made for
        self.built = [torch.cuda.Event(), torch.cuda.Event()]   # the slot's last schedule has been written
        self.read = [torch.cuda.Event(), torch.cuda.Event()]    # the last apply that read the slot has finished
        self.ready = torch.cuda.Event()
        self.cur = 0                       # slot of the last call
        self.last = None                   # (first, n) of the last call

    def release(self):
        for e in self.built + self.read:
            e.synchronize()
        self.buf = [None, None]
        self.key = [None, None]

    def _schedule(self, s, n_users, n_items, indptr, n, seed, first, flags, stream):
        need = int(lib().eb_bpr_step_sampled_workspace_bytes(n, n_users))
        if self.buf[s] is None or self.buf[s].numel() < need:
            self.built[s].synchronize(); self.read[s].synchronize()
            self.buf[s] = None
            self.buf[s] = torch.empty(need, dtype=torch.uint8, device=self.device)
            self.buf[s].record_stream(self.side)
        off = ctypes.c_size_t(0)
        check(lib().eb_bpr_schedule_sampled(n_users, n_items, _ptr(indptr), n, seed, first, _ptr(self.buf[s]), self.buf[s].numel(),
                                            ctypes.byref(off), flags & 0xff00, stream.cuda_stream))
        self.off[s] = off.value

    def step(self, U, V, b, d, n_users, n_items, indptr, indices, filt, fw, n, seed, first, hp, loss, out, flags):
        st = torch.cuda.current_stream(self.device)
        csr = (n_users, n_items, indptr.data_ptr(), indices.data_ptr(), _ptr(filt), indptr._version, indices._version)
        key = (seed, first, n) + csr
        s = 0 if self.key[0] == key else 1 if self.key[1] == key else None
        if s is None:
            s = self.cur
            st.wait_event(self.built[s]); st.wait_event(self.read[s])
            self._schedule(s, n_users, n_items, indptr, n, seed, first, flags, st)
        else:
            st.wait_event(self.built[s])
        self.key[s] = None
        ahead = self.last == (first - n, n)
        if ahead:
            self.ready.record(st)
        order = self.buf[s].data_ptr() + self.off[s]
        check(lib().eb_bpr_apply_sampled_filter_f32(_ptr(U), _ptr(V), _ptr(b), d, U.stride(0), n_users, n_items, _ptr(indptr),
                                                    _ptr(indices), _ptr(filt), fw, n, seed, first, *hp, _ptr(loss), *out, order,
                                                    flags, st.cuda_stream))
        self.read[s].record(st)
        self.cur, self.last = s, (first, n)
        if ahead:
            o = 1 - s
            self.side.wait_event(self.ready); self.side.wait_event(self.read[o])
            self._schedule(o, n_users, n_items, indptr, n, seed, first + n, flags, self.side)
            self.built[o].record(self.side)
            indptr.record_stream(self.side)
            self.key[o] = (seed, first + n, n) + csr


def bpr_sample_philox(n_users, n_items, indptr, indices, n, seed, first=0, filter=None):
    _need_cuda(indptr, indices, filter)
    dev = indptr.device
    u = torch.empty(n, dtype=torch.int32, device=dev); i = torch.empty_like(u); j = torch.empty_like(u)
    _call("eb_bpr_sample_philox_filter", indptr, n_users, n_items, _ptr(indptr), _ptr(indices), _ptr(filter),
          0 if filter is None else filter.shape[1], n, seed, first, _ptr(u), _ptr(i), _ptr(j))
    return u, i, j


def pack_bits(n_users, n_items):
    """(bits_u, bits_i) of the packed host-triple format."""
    bu, bi = max(1, (int(n_users) - 1).bit_length()), max(1, (int(n_items) - 1).bit_length())
    if bu + 2 * bi > 64:
        raise ValueError("ids too wide for the packed 64-bit triple format")
    return bu, bi


def pack_triples(tu, ti, tj, n_users, n_items):
    """int64 tensor (same device as the inputs): u | i << bits_u | j << (bits_u + bits_i) — the host-boundary format of
    bpr_step_host_packed_f32 (8 B/triple)."""
    bu, bi = pack_bits(n_users, n_items)
    return tu.to(torch.int64) | (ti.to(torch.int64) << bu) | (tj.to(torch.int64) << (bu + bi))


def bpr_step_host_packed_f32(U, V, b, d, packed_host, n_users, n_items, lr, reg_u, reg_b, reg_pos, reg_neg, staging, loss_dev,
                             loss_host, sync=True, reserve_sms=0):
    """End-to-end step from HOST (pinned) packed triples: one H2D copy of 8 B/triple, kernel, loss D2H."""
    _need_cuda(U, V, b, staging, loss_dev)
    n = packed_host.numel()
    assert not packed_host.is_cuda and packed_host.dtype == torch.int64 and staging.dtype == torch.int64 and staging.numel() >= n
    bu, bi = pack_bits(n_users, n_items)
    _call("eb_bpr_step_host_packed_f32", U, _ptr(U), _ptr(V), _ptr(b), d, U.stride(0), _ptr(packed_host), n, bu, bi, lr, reg_u,
          reg_b, reg_pos, reg_neg, _ptr(staging), _ptr(loss_dev), _ptr(loss_host), _bpr_flags(sync=sync, reserve_sms=reserve_sms))


def bpr_exact_f64(U, V, b, d, tu, ti, tj, lr, reg_u, reg_b, reg_pos, reg_neg, loss=None):
    """Exact-mode step: identical to applying the triples one by one in order (BPRMF.py:119-127)."""
    _need_cuda(U, V, b, tu, ti, tj, loss)
    _chk_idx(tu, ti, tj)
    assert U.dtype == torch.float64 and V.dtype == torch.float64 and b.dtype == torch.float64
    n = tu.numel()
    nu, ni = U.shape[0], V.shape[0]
    ws = _scratch("bpr_exact", lib().eb_bpr_exact_workspace_bytes(n, nu, ni), U.device)
    _call("eb_bpr_exact_f64", U, _ptr(U), _ptr(V), _ptr(b), d, U.stride(0), nu, ni, _ptr(tu), _ptr(ti), _ptr(tj), n, lr, reg_u,
          reg_b, reg_pos, reg_neg, _ptr(loss), _ptr(ws), ws.numel())


class MtSampler:
    """Device replay of the reference sampler stream (custom_sampler.py:14-46).

    indptr/set_indices: the reference's `_ui_dict` in list(set(...)) order; sorted_indices: same
    CSR with rows sorted.  The MT19937 state persists across step() calls like the reference's
    global np.random state does across epochs.
    """

    def __init__(self, n_users, n_items, indptr, set_indices, sorted_indices, seed=42):
        _need_cuda(indptr, set_indices, sorted_indices)
        assert indptr.dtype == torch.int64 and set_indices.dtype == torch.int32 and sorted_indices.dtype == torch.int32
        self.n_users, self.n_items = n_users, n_items
        self.indptr, self.set_indices, self.sorted_indices = indptr, set_indices, sorted_indices
        self.state = torch.empty(625, dtype=torch.int32, device=indptr.device)
        _call("eb_mt_seed", indptr, _ptr(self.state), seed)

    def raw(self, n):
        out = torch.empty(n, dtype=torch.int32, device=self.state.device)
        _call("eb_mt_raw", out, _ptr(self.state), _ptr(out), n)
        return out

    def step(self, events):
        dev = self.state.device
        u = torch.empty(events, dtype=torch.int32, device=dev); i = torch.empty_like(u); j = torch.empty_like(u)
        ws = _scratch("mt_sampler", lib().eb_mt_sampler_workspace_bytes(events), dev)
        _call("eb_mt_sampler_step", u, _ptr(self.state), self.n_users, self.n_items, _ptr(self.indptr), _ptr(self.set_indices),
              _ptr(self.sorted_indices), events, _ptr(u), _ptr(i), _ptr(j), _ptr(ws), ws.numel())
        return u, i, j


class MtPointwiseRatioSampler:
    """Device replay of the reference's pointwise ratio sampler (samplers/pointwise_pos_neg_ratio_ratings_sampler.py,
    DMF's): (user, item, rating) samples, `neg_ratio` negatives (rating 0) per positive on average, from one MT19937 stream
    seeded at construction.  indptr/set_indices/set_ratings: the reference's `_ui_dict` in list(set(...)) order with each
    entry's train rating; sorted_indices: the same CSR with rows sorted.  The MT state persists across calls; the list
    permutation persists within an epoch, and epoch() resets it as each Sampler.step() call does.  step(events) draws
    the next `events` samples of the current epoch in windows of at most `window` samples (scratch ~2.3 KB per window
    sample at neg_ratio 5); the samples do not depend on the window."""

    WINDOW = 1 << 17

    def __init__(self, n_users, n_items, indptr, set_indices, set_ratings, sorted_indices, neg_ratio, seed=42):
        _need_cuda(indptr, set_indices, set_ratings, sorted_indices)
        assert indptr.dtype == torch.int64 and set_indices.dtype == torch.int32 and sorted_indices.dtype == torch.int32
        assert set_ratings.dtype == torch.float32 and set_ratings.numel() == set_indices.numel()
        if not 0 <= int(neg_ratio) <= 15:
            raise ValueError(f"neg_ratio={neg_ratio}: the device sampler replays lists of at most 16 slots (0 <= neg_ratio <= 15)")
        self.n_users, self.n_items, self.neg_ratio = n_users, n_items, int(neg_ratio)
        self.indptr, self.set_indices, self.set_ratings, self.sorted_indices = indptr, set_indices, set_ratings, sorted_indices
        self.state = torch.empty(625, dtype=torch.int32, device=indptr.device)
        self.list_pos = torch.empty(1, dtype=torch.int32, device=indptr.device)
        _call("eb_mt_seed", indptr, _ptr(self.state), seed)
        self.epoch()

    def epoch(self):
        """Start an epoch: the list is [0] * neg_ratio + [1] again."""
        self.list_pos.fill_(self.neg_ratio)

    def step(self, events, window=None):
        dev = self.state.device
        window = int(window or self.WINDOW)
        u = torch.empty(events, dtype=torch.int32, device=dev); i = torch.empty_like(u)
        r = torch.empty(events, dtype=torch.float32, device=dev)
        ws = _scratch("mt_pointwise", lib().eb_mt_pointwise_ratio_workspace_bytes(min(events, window), self.n_users,
                                                                                   self.neg_ratio), dev)
        for s in range(0, events, window):
            n = min(window, events - s)
            _call("eb_mt_pointwise_ratio_step", u, _ptr(self.state), _ptr(self.list_pos), self.n_users, self.n_items,
                  _ptr(self.indptr), _ptr(self.set_indices), _ptr(self.set_ratings), _ptr(self.sorted_indices),
                  self.neg_ratio, n, _ptr(u[s:]), _ptr(i[s:]), _ptr(r[s:]), _ptr(ws), ws.numel())
        return u, i, r


def score_topk(U, V, bias, d, k, mask_indptr=None, mask_indices=None, users=None, user_begin=0, n_sel=None):
    """Exact full-catalogue score + train mask + top-k (BPRMF_model.py:70-85 / BPRMF_batch_model.py:82-88)."""
    _need_cuda(U, V, bias, mask_indptr, mask_indices, users)
    assert U.dtype in (torch.float32, torch.float64) and V.dtype == U.dtype
    n_sel, idx, val = _topk_out(users, U.shape[0], user_begin, n_sel, k, U.dtype, U.device)
    n_items = V.shape[0]
    ws = _scratch("score_topk", lib().eb_score_topk_workspace_bytes(n_sel, n_items, U.element_size()), U.device)
    _call("eb_score_topk_f32" if U.dtype == torch.float32 else "eb_score_topk_f64", U, _ptr(U), _ptr(V), _ptr(bias), n_items, d,
          U.stride(0), _ptr(mask_indptr), _ptr(mask_indices), _ptr(users), user_begin, n_sel, k, _ptr(idx), _ptr(val), _ptr(ws),
          ws.numel())
    return idx, val


def score_rank(U, V, bias, d, rel_indptr, rel_items, mask_indptr=None, mask_indices=None, users=None, user_begin=0,
               n_sel=None, per_positive=False):
    """Rank of every relevant item in the full list score_topk(k=n_items) gives each selected user (the AUC / GAUC
    counts of auc.py / gauc.py): rel CSR = int64 indptr over user ids, int32 items sorted per user, -1 for items outside
    the catalogue.  Returns (n_pos, sum_c), int64 per row: the relevant items in the list, and the sum over them of the
    non-relevant entries ahead of each; per_positive=True adds, per rel CSR entry, that count or -1 (tests)."""
    _need_cuda(U, V, bias, mask_indptr, mask_indices, users, rel_indptr, rel_items)
    assert U.dtype in (torch.float32, torch.float64) and V.dtype == U.dtype
    assert rel_indptr.dtype == torch.int64 and rel_items.dtype == torch.int32 and rel_items.is_contiguous()
    if users is not None:
        _chk_idx(users)
        n_sel = users.numel()
    elif n_sel is None:
        n_sel = U.shape[0] - user_begin
    n_pos, sum_c = (torch.empty(n_sel, dtype=torch.int64, device=U.device) for _ in range(2))
    c = torch.full((rel_items.numel(),), -1, dtype=torch.int64, device=U.device) if per_positive else None
    _call("eb_score_rank_f32" if U.dtype == torch.float32 else "eb_score_rank_f64", U, _ptr(U), _ptr(V), _ptr(bias), V.shape[0],
          d, U.stride(0), _ptr(mask_indptr), _ptr(mask_indices), _ptr(rel_indptr), _ptr(_nonempty(rel_items)), _ptr(users),
          user_begin, n_sel, _ptr(n_pos), _ptr(sum_c), _ptr(c))
    return (n_pos, sum_c, c) if per_positive else (n_pos, sum_c)


def score_topk_tc(U, V, bias, d, k, mask_indptr=None, mask_indices=None, user_begin=0, n_sel=None, dump=False, stats=True):
    """Tensor-core scoring + top-k (fp32 tables); same result as score_topk().  Returns
    (idx, val, stats) with stats = {"rechecked": users re-done by the exact kernel, "kp": padded K}
    (+ "dump": dense approximate scores when dump=True, tests only).  stats=False: nothing is read back, the call
    stays asynchronous (the models' path) and the dict is empty."""
    _need_cuda(U, V, bias, mask_indptr, mask_indices)
    assert U.dtype == torch.float32 and V.dtype == torch.float32 and U.stride(0) == V.stride(0)
    n_sel, idx, val = _topk_out(None, U.shape[0], user_begin, n_sel, k, torch.float32, U.device)
    n_items = V.shape[0]
    dmp = torch.zeros((n_sel, n_items), dtype=torch.float32, device=U.device) if dump else None
    ws = _scratch("score_topk_tc", lib().eb_score_topk_tc_workspace_bytes(n_sel, n_items, d), U.device)
    st = (ctypes.c_int64 * 16)() if stats else None
    _call("eb_score_topk_tc_f32", U, _ptr(U), _ptr(V), _ptr(bias), n_items, d, U.stride(0), _ptr(mask_indptr), _ptr(mask_indices),
          user_begin, n_sel, k, _ptr(idx), _ptr(val), _ptr(dmp), _ptr(ws), ws.numel(),
          ctypes.cast(st, ctypes.c_void_p) if stats else None)
    out = {"rechecked": int(st[0]), "kp": int(st[1]), "prof": [int(x) for x in st[2:16]]} if stats else {}
    if dump:
        out["dump"] = dmp
    return idx, val, out


def bpr_batch_grad_f32(Gu, Gi, Bi, dGu, dGi, dBi, d, tu, ti, tj, l_w, l_b, loss=None):
    """Batch gradient of the BPRMF_batch loss (BPRMF_batch_model.py:57-75) into dense gradient tables."""
    _need_cuda(Gu, Gi, Bi, dGu, dGi, dBi, tu, ti, tj, loss)
    _chk_idx(tu, ti, tj)
    assert Gu.stride(0) == Gi.stride(0) == dGu.stride(0) == dGi.stride(0)
    _call("eb_bpr_batch_grad_f32", Gu, _ptr(Gu), _ptr(Gi), _ptr(Bi), _ptr(dGu), _ptr(dGi), _ptr(dBi), d, Gu.stride(0), _ptr(tu),
          _ptr(ti), _ptr(tj), tu.numel(), l_w, l_b, _ptr(loss))


def adam_dense_f32(var, m, v, grad, lr, step, beta1=0.9, beta2=0.999, eps=1e-7):
    """Keras Adam over every element (TF 2.3 semantics for sparse gradients too); clears `grad`."""
    _need_cuda(var, m, v, grad)
    n = var.numel()
    assert var.is_contiguous() and m.numel() == n and v.numel() == n and grad.numel() == n and n % 4 == 0
    _call("eb_adam_dense_f32", var, _ptr(var), _ptr(m), _ptr(v), _ptr(grad), n, lr, beta1, beta2, eps, step)


def table_delta_f32(cur, prev, delta):
    _need_cuda(cur, prev, delta)
    assert cur.is_contiguous() and prev.is_contiguous() and delta.is_contiguous() and cur.numel() % 4 == 0
    _call("eb_table_delta_f32", cur, _ptr(cur), _ptr(prev), _ptr(delta), cur.numel())


def table_apply_delta_f32(cur, prev, delta_sum, scale=1.0):
    _need_cuda(cur, prev, delta_sum)
    _call("eb_table_apply_delta_f32", cur, _ptr(cur), _ptr(prev), _ptr(delta_sum), cur.numel(), scale)


_EXACT_GEMM = False


class exact_gemm:
    """Context manager (tests only): while active, `to_bf16` hands the fp32 tensors through unchanged and the dense layers run
    on the fp32 CUDA-core checking kernel (eb_gemm_f32_ref) instead of the bf16 tensor-core GEMM.  Models built inside the
    context can then be compared with their fp64 restatements to ~1e-5 — a check of the model WIRING that bf16 rounding would
    otherwise blur to 1e-2.  Slow; the product path never enables it; the native one-call MultiVAE step ignores it."""

    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        global _EXACT_GEMM
        self.prev, _EXACT_GEMM = _EXACT_GEMM, self.on
        return self

    def __exit__(self, *a):
        global _EXACT_GEMM
        _EXACT_GEMM = self.prev


def _gemm_ref(A, B, M, N, K, a_mn, b_mn, bias, alpha, act, out):
    assert A.dtype == torch.float32 and B.dtype == torch.float32
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=A.device)
    _call("eb_gemm_f32_ref", A, _ptr(A), A.stride(0), 1 if a_mn else 0, _ptr(B), B.stride(0), 1 if b_mn else 0, _ptr(out),
          out.stride(0), M, N, K, _ptr(bias), alpha, act)
    return out


def to_bf16(src, transpose=False, out=None):
    """fp32 [R][C] -> bf16 [R][pad8(C)] or (transpose) [C][pad8(R)], zero padded, via eb_convert_bf16."""
    _need_cuda(src)
    if _EXACT_GEMM:                                       # checking mode: operands stay fp32
        return src.t().contiguous() if transpose else src
    assert src.dtype == torch.float32 and src.dim() == 2 and src.stride(1) == 1
    R, C = src.shape
    rows, cols = (C, R) if transpose else (R, C)
    ldd = (cols + 7) // 8 * 8
    if out is None:
        out = torch.empty((rows, ldd), dtype=torch.bfloat16, device=src.device)
    _call("eb_convert_bf16", src, _ptr(src), R, C, src.stride(0), _ptr(out), ldd, 1 if transpose else 0)
    return out


def _gemm_ws(device):
    """The split-K workspace of the tensor-core GEMMs on `device` (partial tiles summed in a fixed order)."""
    return _scratch("gemm_splitk", lib().eb_gemm_workspace_bytes(), device)


def gemm_bf16_tn(A, B, M, N, K, bias=None, alpha=1.0, act=0, out=None, out_bf16=False):
    """C[M][N] fp32 = act(alpha * A[M][:K] @ B[N][:K]^T + bias) on the tensor cores (A, B bf16, K-major).
    out_bf16=True: returns (C, C_bf16) — the bf16 operand copy of C written by the epilogue itself (no conversion pass)."""
    _need_cuda(A, B, bias, out)
    if A.dtype == torch.float32:                          # exact_gemm checking mode
        C = _gemm_ref(A, B, M, N, K, False, False, bias, alpha, act, out)
        return (C, C) if out_bf16 else C
    if out_bf16:
        assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
        if out is None:
            out = torch.empty((M, N), dtype=torch.float32, device=A.device)
        ldb = (N + 7) // 8 * 8
        Cb = torch.empty((M, ldb), dtype=torch.bfloat16, device=A.device) if ldb == N else torch.zeros((M, ldb), dtype=torch.bfloat16, device=A.device)
        _call("eb_gemm_bf16_out", A, _ptr(A), A.stride(0), 0, _ptr(B), B.stride(0), 0, _ptr(out), out.stride(0), _ptr(Cb), ldb, M,
              N, K, _ptr(bias), alpha, act)
        return out, Cb
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=A.device)
    ws = _gemm_ws(A.device)
    _call("eb_gemm_bf16_tn", A, _ptr(A), A.stride(0), _ptr(B), B.stride(0), _ptr(out), out.stride(0), M, N, K, _ptr(bias), alpha,
          act, _ptr(ws), ws.numel())
    return out


def gemm_bf16(A, B, M, N, K, a_rows_are_k=False, b_rows_are_k=False, bias=None, alpha=1.0, act=0, out=None):
    """C[M][N] fp32 = act(alpha * op(A) @ op(B)^T + bias): an operand flagged rows_are_k is a [K][M] (resp. [K][N]) row-major
    bf16 matrix read by the tensor cores as it lies (MN-major descriptors) — the backward GEMMs need no transposed copies."""
    _need_cuda(A, B, bias, out)
    if A.dtype == torch.float32:                          # exact_gemm checking mode
        return _gemm_ref(A, B, M, N, K, a_rows_are_k, b_rows_are_k, bias, alpha, act, out)
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=A.device)
    ws = _gemm_ws(A.device)
    _call("eb_gemm_bf16", A, _ptr(A), A.stride(0), 1 if a_rows_are_k else 0, _ptr(B), B.stride(0), 1 if b_rows_are_k else 0,
          _ptr(out), out.stride(0), M, N, K, _ptr(bias), alpha, act, _ptr(ws), ws.numel())
    return out


# ---------------------------------------------------------------- MultiVAE: whole step in one call (vae_step.cu)
class _VaeModelStruct(ctypes.Structure):
    _fields_ = ([("n_items", ctypes.c_int), ("H", ctypes.c_int), ("L", ctypes.c_int), ("reserved", ctypes.c_int)]
                + [(f"{pre}{k}", ctypes.c_void_p) for pre in ("", "g", "m", "v")
                   for k in ("W1", "b1", "W2", "b2", "W3", "b3", "W4", "b4")]
                + [(k, ctypes.c_void_p) for k in ("W2b", "W3b", "W4b", "W2t", "W3t", "W4t", "indptr", "indices")])


def vae_model_struct(n_items, H, L, P, G, M, V, bf16_copies, indptr, indices):
    """eb_vae_model over existing device tensors (which must outlive the struct and never be reallocated)."""
    _need_cuda(indptr, indices, *P.values(), *G.values(), *M.values(), *V.values(), *bf16_copies)
    st = _VaeModelStruct()
    st.n_items, st.H, st.L, st.reserved = n_items, H, L, 0
    for pre, d in (("", P), ("g", G), ("m", M), ("v", V)):
        for k in ("W1", "b1", "W2", "b2", "W3", "b3", "W4", "b4"):
            assert d[k].dtype == torch.float32 and d[k].is_contiguous()
            setattr(st, pre + k, d[k].data_ptr())
    for name, t in zip(("W2b", "W3b", "W4b"), bf16_copies):
        assert t.dtype == torch.bfloat16 and t.is_contiguous()
        setattr(st, name, t.data_ptr())
    st.W2t = st.W3t = st.W4t = None                      # unused since the backward GEMMs read the [out][in] copies directly
    assert indptr.dtype == torch.int64 and indices.dtype == torch.int32
    st.indptr, st.indices = indptr.data_ptr(), indices.data_ptr()
    st._keep = (P, G, M, V, bf16_copies, indptr, indices)
    return st


def vae_train_step(model, n_items, H, L, rows, drop_rate, noise_seed, drop_seed, step, anneal, lr, acc, phase=3):
    """eb_vae_train_step: phase bit 0 = forward+backward into the gradient buffers, bit 1 = Adam + operand refresh."""
    _need_cuda(acc, rows)
    B = rows.numel() if rows is not None else 0
    ws = None
    if phase & 1:
        _chk_idx(rows)
        ws = _scratch("vae_step", lib().eb_vae_step_workspace_bytes(n_items, H, L, B), acc.device)
    _call("eb_vae_train_step", acc, ctypes.byref(model), _ptr(rows), B, drop_rate, noise_seed, drop_seed, step, anneal, lr,
          _ptr(acc), _ptr(ws), ws.numel() if ws is not None else 0, phase)


# ---------------------------------------------------------------- MultiVAE pieces (vae.cu)
def vae_embed_fwd(W1, b1, indptr, indices, rows, h1, drop_rate=0.0, seed=0):
    _need_cuda(W1, b1, indptr, indices, rows, h1)
    _call("eb_vae_embed_fwd", W1, _ptr(W1), _ptr(b1), W1.shape[1], _ptr(indptr), _ptr(indices), _ptr(rows), rows.numel(),
          _ptr(h1), h1.stride(0), drop_rate, seed)


def vae_embed_bwd(dW1, indptr, indices, rows, dpre1, drop_rate=0.0, seed=0):
    _need_cuda(dW1, indptr, indices, rows, dpre1)
    _call("eb_vae_embed_bwd", dW1, _ptr(dW1), dW1.shape[1], _ptr(indptr), _ptr(indices), _ptr(rows), rows.numel(), _ptr(dpre1),
          dpre1.stride(0), drop_rate, seed)


def vae_reparam_fwd(ml, L, z, seed, step, kl_sum=None):
    _need_cuda(ml, z, kl_sum)
    _call("eb_vae_reparam_fwd", ml, _ptr(ml), ml.stride(0), ml.shape[0], L, _ptr(z), z.stride(0), seed, step, _ptr(kl_sum))


def vae_reparam_bwd(ml, L, dz, dml, seed, step, anneal):
    _need_cuda(ml, dz, dml)
    _call("eb_vae_reparam_bwd", ml, _ptr(ml), ml.stride(0), ml.shape[0], L, _ptr(dz), dz.stride(0), _ptr(dml), dml.stride(0),
          seed, step, anneal)


def vae_softmax(logits, indptr, indices, rows, nll_sum=None, lse_out=None, write_grad=True, grad_bf16=None):
    """grad_bf16: optional bf16 [B][ld] (ld a multiple of 8) that also receives the gradient, padding columns zeroed."""
    _need_cuda(logits, indptr, indices, rows, nll_sum, lse_out, grad_bf16)
    assert grad_bf16 is None or (grad_bf16.dtype == torch.bfloat16 and grad_bf16.stride(1) == 1)
    _call("eb_vae_softmax_bf16", logits, _ptr(logits), logits.stride(0), logits.shape[1], _ptr(indptr), _ptr(indices), _ptr(rows),
          logits.shape[0], _ptr(nll_sum), _ptr(lse_out), 1 if write_grad else 0, _ptr(grad_bf16),
          grad_bf16.stride(0) if grad_bf16 is not None else 0)


def tanh_bwd(dout, out, dpre=None):
    _need_cuda(dout, out, dpre)
    assert dout.is_contiguous() and out.is_contiguous()
    if dpre is None:
        dpre = torch.empty_like(dout)
    _call("eb_tanh_bwd", dout, _ptr(dout), _ptr(out), _ptr(dpre), dout.numel())
    return dpre


def colsum(src, out=None):
    _need_cuda(src, out)
    if out is None:
        out = torch.empty(src.shape[1], dtype=torch.float32, device=src.device)
    _call("eb_colsum", src, _ptr(src), src.shape[0], src.shape[1], src.stride(0), _ptr(out))
    return out


def csr_to_dense_bf16(indptr, indices, values, n_cols, scale=1.0, row0=0, n_rows=None, row_sq=False, col_sq=False):
    """Rows [row0, row0 + n_rows) of a CSR (values None: ones) times `scale` as a zero-filled bf16 [n_rows][pad8(n_cols)]
    matrix, plus optionally the fp32 squared norms of its rows and of its columns.  Returns (X, row_sq or None, col_sq or None)."""
    _need_cuda(indptr, indices, values)
    assert indptr.dtype == torch.int64 and indices.dtype == torch.int32 and (values is None or values.dtype == torch.float32)
    if n_rows is None:
        n_rows = indptr.numel() - 1 - row0
    dev = indptr.device
    ld = (n_cols + 7) // 8 * 8
    X = torch.empty((n_rows, ld), dtype=torch.bfloat16, device=dev)
    rs = torch.empty(n_rows, dtype=torch.float32, device=dev) if row_sq else None
    cs = torch.empty(n_cols, dtype=torch.float32, device=dev) if col_sq else None
    _call("eb_csr_to_dense_bf16", indptr, _ptr(indptr), _ptr(indices), _ptr(values), row0, n_rows, n_cols, float(scale), _ptr(X),
          ld, _ptr(rs), _ptr(cs))
    return X, rs, cs


def knn_neighbors(slab, n, row0, diag, k, cosine=True, dot_scale=1.0):
    """Neighbour lists of Gram rows row0 .. row0 + slab.shape[0] (slab: fp32 [S][>= n], overwritten with the similarity
    values): (idx int32 [S][k], val fp32 [S][k], cnt int32 [S]), value desc then column asc, -1 / 0 padded."""
    _need_cuda(slab, diag)
    assert slab.dtype == torch.float32 and slab.stride(1) == 1 and diag.dtype == torch.float32
    S = slab.shape[0]
    idx = torch.empty((S, k), dtype=torch.int32, device=slab.device)
    val = torch.empty((S, k), dtype=torch.float32, device=slab.device)
    cnt = torch.empty(S, dtype=torch.int32, device=slab.device)
    _call("eb_knn_neighbors_f32", slab, _ptr(slab), slab.stride(0), S, n, row0, _ptr(diag), 1 if cosine else 0, float(dot_scale), k,
          _ptr(idx), _ptr(val), _ptr(cnt))
    return idx, val, cnt


def knn_score_tile_cols():
    return int(lib().eb_knn_score_tile_cols())


def knn_score_topk(A, B, n_cols, k, frac_bits, mask_indptr=None, mask_indices=None, users=None, user_begin=0, n_sel=None):
    """Top k of the rows of A @ B (A, B: (indptr int64, indices int32, values fp32) CSRs on the device, B's rows sorted by
    column) with the masked columns excluded, (score desc, column asc): (idx int32 [n_sel][k], val fp32 [n_sel][k]).
    Each product is rounded to a multiple of 2^-frac_bits and the sums are exact (see eb_knn_score_topk_f32)."""
    (ap, ai, av), (bp, bi, bv) = A, B
    _need_cuda(ap, ai, av, bp, bi, bv, mask_indptr, mask_indices, users)
    assert ap.dtype == bp.dtype == torch.int64 and av.dtype == bv.dtype == torch.float32
    _chk_idx(ai, bi)
    n_sel, idx, val = _topk_out(users, ap.numel() - 1, user_begin, n_sel, k, torch.float32, ap.device)
    _call("eb_knn_score_topk_f32", ap, _ptr(ap), _ptr(ai), _ptr(av), _ptr(bp), _ptr(bi), _ptr(bv), n_cols, _ptr(mask_indptr),
          _ptr(mask_indices), _ptr(users), user_begin, n_sel, k, int(frac_bits), _ptr(idx), _ptr(val))
    return idx, val


def gram_f64(Y, d, n=None, out=None):
    """G = Y[:n, :d]^T Y[:n, :d] as a fp64 [d][d] tensor, bit-reproducible (eb_gram_f64)."""
    _need_cuda(Y, out)
    assert Y.dtype == torch.float64 and Y.stride(1) == 1
    n = Y.shape[0] if n is None else n
    if out is None:
        out = torch.empty((d, d), dtype=torch.float64, device=Y.device)
    assert out.dtype == torch.float64 and out.is_contiguous() and out.numel() == d * d
    ws = _scratch("gram", lib().eb_gram_f64_workspace_bytes(n, d), Y.device)
    _call("eb_gram_f64", Y, _ptr(Y), n, d, Y.stride(0), _ptr(out), _ptr(ws), ws.numel())
    return out


def als_small_d_max():
    """Largest d solved one row per warp by als_solve_f64 (larger d: one row per CTA)."""
    return int(lib().eb_als_small_d_max())


def als_solve_f64(G, Y, d, indptr, indices, w, c, order, reg, X):
    """X[r] = (G + sum_e w_e y_e y_e^T + reg I)^-1 sum_e c_e y_e for r in `order` (eb_als_solve_f64); the other rows of
    X are left alone.  Raises EbError (code EB_ERR_DATA) naming the smallest row whose matrix is not positive definite."""
    _need_cuda(G, Y, indptr, indices, w, c, order, X)
    assert G.dtype == Y.dtype == X.dtype == w.dtype == c.dtype == torch.float64 and indptr.dtype == torch.int64
    assert G.is_contiguous() and Y.stride(1) == 1 and X.stride(1) == 1 and w.is_contiguous() and c.is_contiguous()
    _chk_idx(indices, order)
    indices, w, c = _nonempty(indices), _nonempty(w), _nonempty(c)
    _call("eb_als_solve_f64", Y, _ptr(G), _ptr(Y), Y.stride(0), d, _ptr(indptr), _ptr(indices), _ptr(w), _ptr(c), _ptr(order),
          order.numel(), float(reg), _ptr(X), X.stride(0))
    return X


def inverse_f64(A, n=None):
    """A[:n, :n] <- its inverse in place (eb_inverse_f64; A fp64, row-major, row stride >= n; padding columns untouched).
    Raises EbError (code EB_ERR_DATA) naming the column when a pivot is zero or not finite.  The workspace is freed on
    return."""
    _need_cuda(A)
    assert A.dtype == torch.float64 and A.stride(1) == 1
    n = A.shape[0] if n is None else n
    assert A.shape[0] >= n and A.shape[1] >= n
    ws = torch.empty(max(int(lib().eb_inverse_f64_workspace_bytes(n)), 256), dtype=torch.uint8, device=A.device)
    _call("eb_inverse_f64", A, _ptr(A), n, A.stride(0), _ptr(ws), ws.numel())
    return A


def ease_normal_f64(slab, row0, count, l2_norm, scale, A):
    """Rows row0 .. row0 + slab.shape[0] of EASE^R's normal matrix into A (fp64 [n][>= n]) from an fp32 Gram slab
    [S][>= n]: off-diagonal slab * scale, diagonal fp32(count + l2_norm) (eb_ease_normal_f64)."""
    _need_cuda(slab, count, A)
    assert slab.dtype == torch.float32 and slab.stride(1) == 1 and A.dtype == torch.float64 and A.stride(1) == 1
    assert count.dtype == torch.int32 and count.is_contiguous()
    _call("eb_ease_normal_f64", A, _ptr(slab), slab.stride(0), slab.shape[0], A.shape[0], row0, _ptr(count), float(l2_norm),
          float(scale), _ptr(A), A.stride(0))
    return A


def ease_weights_f32(P, out=None):
    """B = fp32(-P / diag(P)) column by column with B[j][j] = 0 (eb_ease_weights_f32).  Raises EbError (code EB_ERR_DATA)
    naming the column when P[j][j] is zero."""
    _need_cuda(P, out)
    assert P.dtype == torch.float64 and P.stride(1) == 1
    n = P.shape[0]
    if out is None:
        out = torch.empty((n, n), dtype=torch.float32, device=P.device)
    assert out.dtype == torch.float32 and out.stride(1) == 1 and out.shape[1] >= n
    _call("eb_ease_weights_f32", P, _ptr(P), P.stride(0), n, _ptr(out), out.stride(0))
    return out


def dense_score_topk(A, B, k, frac_bits, mask_indptr=None, mask_indices=None, users=None, user_begin=0, n_sel=None):
    """knn_score_topk with a dense fp32 B [n_mid][n_cols] (row stride >= n_cols): the same fixed-point terms and selection,
    so the output equals knn_score_topk's for B as a CSR, bit for bit (eb_dense_score_topk_f32)."""
    ap, ai, av = A
    _need_cuda(ap, ai, av, B, mask_indptr, mask_indices, users)
    assert ap.dtype == torch.int64 and av.dtype == B.dtype == torch.float32 and B.stride(1) == 1
    _chk_idx(ai)
    n_sel, idx, val = _topk_out(users, ap.numel() - 1, user_begin, n_sel, k, torch.float32, ap.device)
    ai, av = _nonempty(ai), _nonempty(av)
    _call("eb_dense_score_topk_f32", ap, _ptr(ap), _ptr(ai), _ptr(av), _ptr(B), B.stride(0), B.shape[1],
          _ptr(mask_indptr), _ptr(mask_indices), _ptr(users), user_begin, n_sel, k, int(frac_bits), _ptr(idx), _ptr(val))
    return idx, val


def rp3_tile_cols():
    return int(lib().eb_rp3_tile_cols())


def rp3_row_workspace_bytes(n_cols):
    """Bytes of the row workspace rp3_similarity and rp3_score_topk allocate for n_cols columns (0 up to rp3_tile_cols())."""
    return int(lib().eb_rp3_row_workspace_bytes(n_cols))


def _rp3_row_ws(n_cols, device):
    return torch.empty(max(rp3_row_workspace_bytes(n_cols), 1), dtype=torch.uint8, device=device)


def rp3_similarity(A, B, degree, k, order=None):
    """RP3beta's neighbour lists (eb_rp3_similarity_f32): per row i of the ordered fp32 product A . B (A = Piu, B = Pui
    with rows sorted by column; (indptr int64, indices int32, values fp32) on the device), times degree (fp64) with the
    diagonal zeroed, the min(k, n) largest nonzero values in column order.  Returns (idx int32 [n][kk], val fp32 [n][kk],
    cnt int32 [n]) with kk = min(k, n)."""
    (ap, ai, av), (bp, bi, bv) = A, B
    _need_cuda(ap, ai, av, bp, bi, bv, degree, order)
    assert ap.dtype == bp.dtype == torch.int64 and av.dtype == bv.dtype == torch.float32 and degree.dtype == torch.float64
    _chk_idx(ai, bi)
    n = degree.numel()
    kk = min(k, n)
    idx = torch.empty((n, kk), dtype=torch.int32, device=ap.device)
    val = torch.empty((n, kk), dtype=torch.float32, device=ap.device)
    cnt = torch.empty(n, dtype=torch.int32, device=ap.device)
    if order is not None:
        _chk_idx(order)
    ws = _rp3_row_ws(n, ap.device)
    ai, av, bi, bv = _nonempty(ai), _nonempty(av), _nonempty(bi), _nonempty(bv)
    _call("eb_rp3_similarity_f32", ap, _ptr(ap), _ptr(ai), _ptr(av), _ptr(bp), _ptr(bi), _ptr(bv), _ptr(degree), n, _ptr(order),
          k, kk, _ptr(idx), _ptr(val), _ptr(cnt), _ptr(ws), ws.numel())
    return idx, val, cnt


def rp3_l1_rows(val, cnt):
    """val[r, :cnt[r]] <- fp32(v / sum |v|) in place, the sum in fp64 in stored order (eb_rp3_l1_rows_f32)."""
    _need_cuda(val, cnt)
    assert val.dtype == torch.float32 and val.stride(1) == 1 and cnt.dtype == torch.int32 and cnt.is_contiguous()
    _call("eb_rp3_l1_rows_f32", val, val.shape[0], val.stride(0), _ptr(cnt), _ptr(val))
    return val


def rp3_prune_cols(idx, val, cnt, k):
    """W as a CSR (indptr int64, indices int32, values fp32) from rp3_similarity's lists, keeping per column the k largest
    nonzero values, ties to the lowest row (eb_rp3_prune_cols_f32).  Rows list their columns ascending."""
    _need_cuda(idx, val, cnt)
    assert idx.is_contiguous() and val.is_contiguous() and idx.shape == val.shape
    n, stride = idx.shape
    nnz = int(cnt.sum().item())
    dev = idx.device
    indptr = torch.empty(n + 1, dtype=torch.int64, device=dev)
    indices = torch.empty(max(nnz, 1), dtype=torch.int32, device=dev)
    values = torch.empty(max(nnz, 1), dtype=torch.float32, device=dev)
    ws = torch.empty(int(lib().eb_rp3_prune_workspace_bytes(n, stride, nnz)), dtype=torch.uint8, device=dev)
    _call("eb_rp3_prune_cols_f32", idx, n, stride, _ptr(cnt), _ptr(idx), _ptr(val), nnz, k, _ptr(indptr), _ptr(indices),
          _ptr(values), _ptr(ws), ws.numel())
    m = int(indptr[-1].item())
    return indptr, indices[:m].clone(), values[:m].clone()


def rp3_score_topk(A, B, n_cols, k, mask_indptr=None, mask_indices=None, users=None, user_begin=0, n_sel=None, order=None):
    """Top k of the rows of the ordered fp32 product A . B (eb_rp3_score_topk_f32; A's rows summed in stored order, B's
    rows sorted by column) with the masked columns excluded, (score desc, column asc): (idx int32 [n_sel][k], val fp32
    [n_sel][k])."""
    (ap, ai, av), (bp, bi, bv) = A, B
    _need_cuda(ap, ai, av, bp, bi, bv, mask_indptr, mask_indices, users, order)
    assert ap.dtype == bp.dtype == torch.int64 and av.dtype == bv.dtype == torch.float32
    _chk_idx(ai, bi)
    if order is not None:
        _chk_idx(order)
    n_sel, idx, val = _topk_out(users, ap.numel() - 1, user_begin, n_sel, k, torch.float32, ap.device)
    ws = _rp3_row_ws(n_cols, ap.device)
    ai, av, bi, bv = _nonempty(ai), _nonempty(av), _nonempty(bi), _nonempty(bv)
    _call("eb_rp3_score_topk_f32", ap, _ptr(ap), _ptr(ai), _ptr(av), _ptr(bp), _ptr(bi), _ptr(bv), n_cols, _ptr(mask_indptr),
          _ptr(mask_indices), _ptr(users), user_begin, n_sel, _ptr(order), k, _ptr(idx), _ptr(val), _ptr(ws), ws.numel())
    return idx, val


def dense_topk(scores, k, mask_indptr=None, mask_indices=None, rows=None, shift=None):
    _need_cuda(scores, mask_indptr, mask_indices, rows, shift)
    n = scores.shape[0]
    idx = torch.empty((n, k), dtype=torch.int32, device=scores.device)
    val = torch.empty((n, k), dtype=torch.float32, device=scores.device)
    _call("eb_dense_topk_f32", scores, _ptr(scores), scores.stride(0), n, scores.shape[1], _ptr(mask_indptr), _ptr(mask_indices),
          _ptr(rows), _ptr(shift), k, _ptr(idx), _ptr(val))
    return idx, val


# ---------------------------------------------------------------- SLIM (slim.cu)
def slim_slots(n_users, shared_residual):
    return int(lib().eb_slim_slots(int(n_users), int(shared_residual)))


def slim_shared_residual_fits(n_users):
    return bool(lib().eb_slim_shared_residual_fits(int(n_users)))


def slim_workspace_bytes(n_users, n_items, slots, shared_residual):
    return int(lib().eb_slim_workspace_bytes(int(n_users), int(n_items), int(slots), int(shared_residual)))


def slim_fit(csc, csr, n_users, n_items, l1, l2, seed, neighborhood, tol=1e-4, max_iter=100, shared_residual=None,
             slots=None, items=None):
    """Every item's SLIM elastic net (eb_slim_fit_f32).  csc = (colptr int64, rows int32, vals fp32) of X [users][items],
    csr = (rowptr int64, cols int32) of X's pattern.  Returns (coef_t [n_items][n_items] fp32 with coef_t[i, p] the
    coefficient of item i for item p, n_iter int32, gap fp32, nnz int32, drop int32), all indexed by item.  `items`
    (begin, end) fits that range only (the other columns stay 0).  shared_residual None: shared memory when it fits."""
    cp, ri, cv = csc
    rp, ci = csr
    _need_cuda(cp, ri, cv, rp, ci)
    dev = cp.device
    with torch.cuda.device(dev):
        if shared_residual is None:
            shared_residual = slim_shared_residual_fits(n_users)
        cap = slim_slots(n_users, shared_residual)
        if cap < 1:
            raise RuntimeError(f"SLIM: no CTA fits for {n_users} users with shared_residual={shared_residual}")
        slots = cap if slots is None else max(1, min(int(slots), cap))
        coef_t = torch.zeros((n_items, n_items), dtype=torch.float32, device=dev)
        n_iter = torch.zeros(n_items, dtype=torch.int32, device=dev)
        gap = torch.zeros(n_items, dtype=torch.float32, device=dev)
        nnz = torch.zeros(n_items, dtype=torch.int32, device=dev)
        drop = torch.full((n_items,), -1, dtype=torch.int32, device=dev)
        b, e = (0, n_items) if items is None else (int(items[0]), int(items[1]))
        ws_bytes = slim_workspace_bytes(n_users, n_items, slots, shared_residual)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    _call("eb_slim_fit_f32", cp, _ptr(cp), _ptr(ri), _ptr(cv), _ptr(rp), _ptr(ci), int(n_users), int(n_items), b, e - b,
          float(l1), float(l2), float(tol), int(seed) & 0xffffffff, int(max_iter), int(neighborhood), int(shared_residual),
          int(slots), _ptr(coef_t), _ptr(n_iter), _ptr(gap), _ptr(nnz), _ptr(drop), _ptr(ws), ws_bytes)
    return coef_t, n_iter, gap, nnz, drop


def slim_weights(coef_t, drop, nnz, neighborhood):
    """W as a CSR (indptr int64, indices int32, values fp32; rows list their columns ascending) from slim_fit's outputs:
    per column p the min(nnz_p - 1, neighborhood) largest coefficients, ties to the lowest item.  The entry `drop`
    names is removed first (eb_slim_drop_f32); the rest is eb_rp3_prune_cols_f32 with k = neighborhood over W's dense
    rows.  coef_t is not modified."""
    _need_cuda(coef_t, drop, nnz)
    n = coef_t.shape[0]
    dev = coef_t.device
    vals = coef_t.clone()
    _call("eb_slim_drop_f32", vals, n, _ptr(drop), _ptr(vals))
    total = int(torch.clamp(nnz.to(torch.int64), min=0).sum().item())
    idx = torch.arange(n, dtype=torch.int32, device=dev).repeat(n)
    cnt = torch.full((n,), n, dtype=torch.int32, device=dev)
    indptr = torch.empty(n + 1, dtype=torch.int64, device=dev)
    indices = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
    values = torch.empty(max(total, 1), dtype=torch.float32, device=dev)
    ws = torch.empty(int(lib().eb_rp3_prune_workspace_bytes(n, n, total)), dtype=torch.uint8, device=dev)
    _call("eb_rp3_prune_cols_f32", vals, n, n, _ptr(cnt), _ptr(idx), _ptr(vals), total, int(neighborhood), _ptr(indptr),
          _ptr(indices), _ptr(values), _ptr(ws), ws.numel())
    m = int(indptr[-1].item())
    return indptr, indices[:m], values[:m]


# ---------------------------------------------------------------- randomized SVD pieces (pure_svd.cu)
def svd_max_width():
    """Largest block width the SVD pieces take (the limit of gram_f64)."""
    return int(lib().eb_svd_max_width())


def csr_spmm_f64(csr, X, out=None):
    """A X (eb_csr_spmm_f64) for csr = (indptr int64, indices int32, data fp32) of A and an fp64 X with one row per column
    of A; every output element summed over its row's entries in stored order.  Returns out [rows of A][X.shape[1]]."""
    indptr, indices, data = csr
    _need_cuda(indptr, indices, data, X, out)
    _chk_f64_rows(X)
    _chk_idx(indices)
    assert indptr.dtype == torch.int64 and data.dtype == torch.float32 and indptr.is_contiguous() and data.is_contiguous()
    n, w = indptr.numel() - 1, X.shape[1]
    if out is None:
        out = torch.empty((n, w), dtype=torch.float64, device=X.device)
    _chk_f64_rows(out)
    assert out.shape[0] == n and out.shape[1] >= w
    indices, data = _nonempty(indices), _nonempty(data)
    _call("eb_csr_spmm_f64", X, _ptr(indptr), _ptr(indices), _ptr(data), n, _ptr(X), w, X.stride(0), _ptr(out), out.stride(0))
    return out


def chol_pivoted_f64(G, M=None, rank=None):
    """M = P L^-T from the pivoted Cholesky factorisation P^T G P = L L^T (eb_chol_pivoted_f64), columns past the
    numerical rank zero.  `rank`: an optional int32 device tensor of one element that receives the rank."""
    _need_cuda(G, M, rank)
    w = G.shape[0]
    assert G.dtype == torch.float64 and G.is_contiguous() and G.shape == (w, w)
    if M is None:
        M = torch.empty((w, w), dtype=torch.float64, device=G.device)
    assert M.dtype == torch.float64 and M.is_contiguous() and M.shape == (w, w)
    assert rank is None or (rank.dtype == torch.int32 and rank.numel() >= 1)
    _call("eb_chol_pivoted_f64", G, _ptr(G), w, _ptr(M), _ptr(rank))
    return M


def tall_times_small_f64(X, M, out=None):
    """X M (eb_tall_times_small_f64) for a tall fp64 X [n][w] and a contiguous M [w][d]; `out` may be X itself when
    d == w."""
    _need_cuda(X, M, out)
    _chk_f64_rows(X)
    n, w = X.shape
    assert M.dtype == torch.float64 and M.is_contiguous() and M.shape[0] == w
    d = M.shape[1]
    if out is None:
        out = torch.empty((n, d), dtype=torch.float64, device=X.device)
    _chk_f64_rows(out)
    assert out.shape[0] == n and out.shape[1] >= d
    _call("eb_tall_times_small_f64", X, _ptr(X), n, w, X.stride(0), _ptr(M), d, _ptr(out), out.stride(0))
    return out


def sym_eig_f64(A):
    """(eigenvalues descending [w], eigenvectors [w][w] by column) of a symmetric fp64 A (eb_sym_eig_f64, Jacobi)."""
    _need_cuda(A)
    w = A.shape[0]
    assert A.dtype == torch.float64 and A.is_contiguous() and A.shape == (w, w)
    evals = torch.empty(w, dtype=torch.float64, device=A.device)
    evecs = torch.empty((w, w), dtype=torch.float64, device=A.device)
    ws = torch.empty(max(1, int(lib().eb_sym_eig_f64_workspace_bytes(w))), dtype=torch.uint8, device=A.device)
    _call("eb_sym_eig_f64", A, _ptr(A), w, _ptr(evals), _ptr(evecs), _ptr(ws), ws.numel())
    return evals, evecs


def svd_finish_f64(evals, user, item, scale_user_by_inv_s):
    """In place on the first d = user.shape[1] columns (eb_svd_finish_f64): the optional 1/s and s column scaling and
    the sign of each user column's largest entry; returns s [d]."""
    _need_cuda(evals, user, item)
    _chk_f64_rows(user, item)
    d = user.shape[1]
    assert evals.dtype == torch.float64 and evals.is_contiguous() and item.shape[1] == d
    s = torch.empty(d, dtype=torch.float64, device=user.device)
    _call("eb_svd_finish_f64", user, _ptr(evals), evals.numel(), d, _ptr(user), user.shape[0], user.stride(0), _ptr(item),
          item.shape[0], item.stride(0), int(bool(scale_user_by_inv_s)), _ptr(s))
    return s


# ---------------------------------------------------------------- SlopeOne (slope_one.cu)
def slope_one_dev_f64(F, M1, M2, n, s, out=None):
    """E rows = ((M1 - M2) 2^-s) / F in fp64, NaN where F = 0 (eb_slope_one_dev_f64), for fp32 slabs F, M1, M2 [rows][>= n]
    of one layout.  `out`: fp64 [rows][>= n] with unit column stride, e.g. a row range of the full E."""
    _need_cuda(F, M1, M2, out)
    for t in (F, M1, M2):
        assert t.dtype == torch.float32 and t.stride(1) == 1 and t.stride(0) == F.stride(0) and t.shape[0] == F.shape[0]
    rows = F.shape[0]
    if out is None:
        out = torch.empty((rows, n), dtype=torch.float64, device=F.device)
    assert out.dtype == torch.float64 and out.stride(1) == 1 and out.shape[0] == rows and out.shape[1] >= n
    _call("eb_slope_one_dev_f64", F, _ptr(F), _ptr(M1), _ptr(M2), F.stride(0), rows, n, int(s), _ptr(out), out.stride(0))
    return out


def slope_one_score_topk(E, train, k, mask_indptr=None, mask_indices=None, users=None, user_begin=0, n_sel=None):
    """Top k of the SlopeOne scores (eb_slope_one_score_topk_f64): E fp64 [n_items][>= n_items], train = (indptr int64,
    items int32, ratings fp32) with each user's items in summation order.  Returns (idx int32 [n_sel][k], val fp64
    [n_sel][k]), (score desc, item asc), -1 / -inf padded."""
    indptr, items, ratings = train
    _need_cuda(E, indptr, items, ratings, mask_indptr, mask_indices, users)
    assert E.dtype == torch.float64 and E.stride(1) == 1
    assert indptr.dtype == torch.int64 and ratings.dtype == torch.float32 and ratings.is_contiguous()
    _chk_idx(items)
    n_sel, idx, val = _topk_out(users, indptr.numel() - 1, user_begin, n_sel, k, torch.float64, E.device)
    items, ratings = _nonempty(items), _nonempty(ratings)
    if mask_indices is not None:
        _chk_idx(mask_indices)
        mask_indices = _nonempty(mask_indices)
    _call("eb_slope_one_score_topk_f64", E, _ptr(E), E.stride(0), E.shape[0], _ptr(indptr), _ptr(items), _ptr(ratings),
          _ptr(mask_indptr), _ptr(mask_indices), _ptr(users), user_begin, n_sel, k, _ptr(idx), _ptr(val))
    return idx, val


# ---------------------------------------------------------------- NonNegMF (nonneg_mf.cu)
def nnmf_dots_f64(P, Q, indptr, items, out=None):
    """dot_k = Q[i_k] . P[u_k] for every rating k of the CSR (indptr int64, items int32), summed in f order from +0.0
    (eb_nnmf_dots_f64).  P [n_users][F] and Q [n_items][F] fp64, contiguous."""
    _need_cuda(P, Q, indptr, items, out)
    _chk_f64_dense(P, Q)
    _chk_idx(items)
    assert indptr.dtype == torch.int64 and P.shape[1] == Q.shape[1] and indptr.numel() == P.shape[0] + 1
    if out is None:
        out = torch.empty(items.numel(), dtype=torch.float64, device=P.device)
    _chk_f64_dense(out)
    _call("eb_nnmf_dots_f64", P, _ptr(P), _ptr(Q), P.shape[1], _ptr(indptr), _ptr(items), P.shape[0], _ptr(out))
    return out


def nnmf_bias_chain_f64(indptr, items, ratings, dots, mu, lr, reg, bu, bi, out=None):
    """est_k for every rating k in order, updating bu and bi in place as the reference's loop does
    (eb_nnmf_bias_chain_f64).  ratings, dots, bu, bi: fp64 contiguous."""
    _need_cuda(indptr, items, ratings, dots, bu, bi, out)
    _chk_f64_dense(ratings, dots, bu, bi)
    _chk_idx(items)
    assert indptr.dtype == torch.int64 and indptr.numel() == bu.numel() + 1
    if out is None:
        out = torch.empty(items.numel(), dtype=torch.float64, device=bu.device)
    _chk_f64_dense(out)
    _call("eb_nnmf_bias_chain_f64", bu, _ptr(indptr), _ptr(items), _ptr(ratings), _ptr(dots), bu.numel(), bi.numel(),
          float(mu), float(lr), float(reg), _ptr(bu), _ptr(bi), _ptr(out))
    return out


def nnmf_row_update_f64(indptr, cols, pos, ratings, est, T, S, reg, out=None):
    """S * (num / den) row by row (eb_nnmf_row_update_f64): num and den the ordered sums of T[col] * r_k and
    T[col] * est_k over each row's entries (k = pos[e], or e when pos is None), den + (n reg) S.  `out` may be S."""
    _need_cuda(indptr, cols, pos, ratings, est, T, S, out)
    _chk_f64_dense(ratings, est, T, S)
    _chk_idx(cols)
    assert indptr.dtype == torch.int64 and indptr.numel() == S.shape[0] + 1 and T.shape[1] == S.shape[1]
    assert pos is None or (pos.dtype == torch.int64 and pos.is_contiguous())
    if out is None:
        out = torch.empty_like(S)
    _chk_f64_dense(out)
    _call("eb_nnmf_row_update_f64", S, _ptr(indptr), _ptr(cols), _ptr(pos), S.shape[0], _ptr(ratings), _ptr(est), _ptr(T),
          _ptr(S), _ptr(out), S.shape[1], float(reg))
    return out


# ---------------------------------------------------------------- MostPop and Random (unpersonalized.cu)
def _train_csr(indptr, train):
    _need_cuda(indptr, train)
    _chk_idx(train)
    assert indptr.dtype == torch.int64 and indptr.is_contiguous()
    return _nonempty(train)


def item_pop(indices, n_items):
    """pop [n_items] int32: the entries of each item among the train indices (eb_item_pop)."""
    _need_cuda(indices)
    _chk_idx(indices)
    pop = torch.empty(n_items, dtype=torch.int32, device=indices.device)
    _call("eb_item_pop", pop, _ptr(_nonempty(indices)), indices.numel(), n_items, _ptr(pop))
    return pop


def mostpop_topk(order, pop, k, indptr, train, users=None, user_begin=0, n_sel=None):
    """MostPop lists (eb_mostpop_topk): (idx int32 [n_sel][k], val int32 [n_sel][k] = pop, skipped int32 device scalar)
    with `order` every item by (pop desc, item asc) and the sorted train CSR as the mask; a user with |train_u| + k >=
    n_items gets a row of -1 and is counted in `skipped`."""
    train = _train_csr(indptr, train)
    _need_cuda(order, pop, users)
    _chk_idx(order, pop)
    n_sel, idx, val = _topk_out(users, indptr.numel() - 1, user_begin, n_sel, k, torch.int32, order.device)
    skipped = torch.empty((), dtype=torch.int32, device=order.device)
    _call("eb_mostpop_topk", order, _ptr(order), _ptr(pop), order.numel(), _ptr(indptr), _ptr(train), _ptr(users), user_begin,
          n_sel, k, _ptr(idx), _ptr(val), _ptr(skipped))
    return idx, val, skipped


class RandomStream:
    """The legacy np.random stream of `np.random.seed(seed)` on the device, drawn the way the reference's Random does
    (eb_random_draws): the MT19937 state, a buffer of `capacity` generated words and the position in it persist from
    call to call, as numpy's global state does."""

    def __init__(self, seed, device, capacity=1 << 20):
        self.state = torch.empty(625, dtype=torch.int32, device=device)
        self.words = torch.empty(capacity, dtype=torch.int32, device=device)
        self.pos = (ctypes.c_int64 * 2)(0, 0)
        self.consumed = 0
        _call("eb_mt_seed", self.state, _ptr(self.state), seed)

    def draws(self, k, indptr, n_items):
        """r [n_users][k] int32: each user's draws, -1 past min(k, n_u).  Reads back how far the walk got (one host
        synchronise per buffer of words)."""
        _need_cuda(indptr)
        assert indptr.dtype == torch.int64 and indptr.is_contiguous()
        n_users = indptr.numel() - 1
        r = torch.empty((n_users, k), dtype=torch.int32, device=self.state.device)
        used = ctypes.c_int64(0)
        ws = _scratch("random_walk", lib().eb_random_workspace_bytes(), r.device)
        _call("eb_random_draws", r, _ptr(self.state), _ptr(self.words), self.words.numel(), self.pos, n_users, n_items,
              _ptr(indptr), k, _ptr(r), ctypes.byref(used), _ptr(ws), ws.numel())
        self.consumed += used.value
        return r


def complement_select(r, indptr, train, users=None, user_begin=0, n_sel=None):
    """(users x k) int32: the r-th item outside each user's sorted train row for every r of r [n_users][k], -1 where
    r < 0 (eb_complement_select)."""
    train = _train_csr(indptr, train)
    _need_cuda(r, users)
    _chk_idx(r)
    k = r.shape[1]
    n_sel, out, _ = _topk_out(users, indptr.numel() - 1, user_begin, n_sel, k, torch.int32, r.device)
    _call("eb_complement_select", r, _ptr(r), _ptr(indptr), _ptr(train), _ptr(users), user_begin, n_sel, k, _ptr(out))
    return out


# ---------------------------------------------------------------- NeuMF pieces (neumf.cu)
def neumf_gather(Umf, Imf, Umlp, Imlp, f, u, it, x0, pm):
    _need_cuda(Umf, Imf, Umlp, Imlp, u, it, x0, pm)
    _call("eb_neumf_gather", Umf, _ptr(Umf), _ptr(Imf), _ptr(Umlp), _ptr(Imlp), f, Umf.stride(0), _ptr(u), _ptr(it), u.numel(),
          _ptr(x0), x0.stride(0), _ptr(pm), pm.stride(0))


def neumf_head(pm, h3, f, wp, bp, label=None, dpm=None, dh3=None, dwp=None, dbp=None, loss=None, prob=None, mean_over=None):
    """mean_over: number of samples the BinaryCrossentropy mean runs over (default: this call's batch)."""
    _need_cuda(pm, h3, wp, bp, label, dpm, dh3, dwp, dbp, loss, prob)
    _call("eb_neumf_head_norm", pm, _ptr(pm), pm.stride(0), _ptr(h3), h3.stride(0), f, _ptr(wp), _ptr(bp), _ptr(label), pm.shape[0],
          int(mean_over) if mean_over else max(int(pm.shape[0]), 1), _ptr(dpm), _ptr(dh3), _ptr(dwp), _ptr(dbp), _ptr(loss), _ptr(prob))


def relu_bwd(dout, out, copy_bf16=False):
    """dpre = dout * (out > 0); copy_bf16=True also returns dpre's bf16 operand copy, written in the same pass (row length % 8 == 0)."""
    _need_cuda(dout, out)
    dpre = torch.empty_like(dout)
    if copy_bf16 and not _EXACT_GEMM:
        assert dout.dim() == 2 and dout.shape[1] % 8 == 0 and dout.is_contiguous()
        cb = torch.empty(dout.shape, dtype=torch.bfloat16, device=dout.device)
        _call("eb_relu_bwd_copy", dout, _ptr(dout), _ptr(out), _ptr(dpre), dout.numel(), _ptr(cb))
        return dpre, cb
    _call("eb_relu_bwd", dout, _ptr(dout), _ptr(out), _ptr(dpre), dout.numel())
    return (dpre, dpre) if copy_bf16 else dpre


def neumf_scatter(Umf, Imf, f, u, it, dpm, dx0, dUmf, dImf, dUmlp, dImlp):
    _need_cuda(Umf, Imf, u, it, dpm, dx0, dUmf, dImf, dUmlp, dImlp)
    _call("eb_neumf_scatter", Umf, _ptr(Umf), _ptr(Imf), f, Umf.stride(0), _ptr(u), _ptr(it), u.numel(), _ptr(dpm), dpm.stride(0),
          _ptr(dx0), dx0.stride(0), _ptr(dUmf), _ptr(dImf), _ptr(dUmlp), _ptr(dImlp))


def neumf_sample(n_users, n_items, indptr, indices, m, seed):
    _need_cuda(indptr, indices)
    total = int(indices.numel()) * (1 + m)
    dev = indptr.device
    u = torch.empty(total, dtype=torch.int32, device=dev); i = torch.empty_like(u)
    y = torch.empty(total, dtype=torch.float32, device=dev)
    _call("eb_neumf_sample", indptr, n_users, n_items, _ptr(indptr), _ptr(indices), m, seed, total, _ptr(u), _ptr(i), _ptr(y))
    return u, i, y


def neumf_pair_h1(Au, Ai, b1, n_ub, n_items, h1, out):
    _need_cuda(Au, Ai, b1, out)
    if out.dtype == torch.float32:                        # exact_gemm checking mode: the first layer stays fp32
        _call("eb_neumf_pair_h1_f32", Au, _ptr(Au), Au.stride(0), _ptr(Ai), Ai.stride(0), _ptr(b1), n_ub, n_items, h1, _ptr(out), out.stride(0))
        return
    _call("eb_neumf_pair_h1", Au, _ptr(Au), Au.stride(0), _ptr(Ai), Ai.stride(0), _ptr(b1), n_ub, n_items, h1, _ptr(out), out.stride(0))


def neumf_pair_head(Umf, Imf, f, u0, n_ub, n_items, h3, wp, bp, prob):
    _need_cuda(Umf, Imf, h3, wp, bp, prob)
    _call("eb_neumf_pair_head", Umf, _ptr(Umf), _ptr(Imf), Umf.stride(0), f, u0, n_ub, n_items, _ptr(h3), h3.stride(0), _ptr(wp),
          _ptr(bp), _ptr(prob), prob.stride(0))


def table_apply_delta_late_f32(cur, prev, delta_sum, delta_local, scale=1.0):
    _need_cuda(cur, prev, delta_sum, delta_local)
    _call("eb_table_apply_delta_late_f32", cur, _ptr(cur), _ptr(prev), _ptr(delta_sum), _ptr(delta_local), cur.numel(),
          float(scale))


def mf_pointwise_exact_f64(U, V, ub, ib, gb, d, su, si, sr, lr, reg, batch=100000, batch_loss=None):
    """MF2020 train_step over an ordered sample list, sequentially consistent fp64 (MF_model.py:80-112)."""
    _need_cuda(U, V, ub, ib, gb, su, si, sr, batch_loss)
    _chk_idx(su, si, sr)
    for t in (U, V, ub, ib, gb):
        assert t.dtype == torch.float64
    assert U.stride(1) == 1 and V.stride(1) == 1 and U.stride(0) == V.stride(0) and ub.is_contiguous() and ib.is_contiguous()
    n = su.numel()
    if batch_loss is not None:
        assert batch_loss.dtype == torch.float64 and batch_loss.numel() >= (n + batch - 1) // batch
    _call("eb_mf_pointwise_exact_f64", U, _ptr(U), _ptr(V), _ptr(ub), _ptr(ib), _ptr(gb), d, U.stride(0), _ptr(su), _ptr(si),
          _ptr(sr), n, lr, reg, batch, _ptr(batch_loss))


_mf_gb_work = {}


def mf_pointwise_step_f32(U, V, ub, ib, gb, d, pos_u, pos_i, m, n_items, seed, epoch, lr, reg, loss=None, out=None,
                          first=0, count=None):
    """MF2020 throughput mode: positions [first, first+count) of the epoch's sample list (every positive + m uniform
    negatives, pseudo-randomly ordered) in one launch, fp32 Hogwild; count=None -> to the end of the epoch."""
    _need_cuda(U, V, ub, ib, gb, pos_u, pos_i, loss)
    _chk_idx(pos_u, pos_i)
    for t in (U, V, ub, ib, gb):
        assert t.dtype == torch.float32
    assert U.stride(1) == 1 and V.stride(1) == 1 and U.stride(0) == V.stride(0)
    out = _out_ptrs(out)
    n_epoch = pos_u.numel() * (1 + m)
    if count is None:
        count = n_epoch - first
    work = _mf_gb_work.get(U.device)
    if work is None:
        work = _mf_gb_work[U.device] = torch.zeros(4, dtype=torch.float64, device=U.device)
    _call("eb_mf_pointwise_step_f32", U, _ptr(U), _ptr(V), _ptr(ub), _ptr(ib), _ptr(gb), d, U.stride(0), _ptr(pos_u), _ptr(pos_i),
          pos_u.numel(), m, n_items, seed, epoch, first, count, lr, reg, _ptr(loss), _ptr(work), *out)


def eval_topk(topk_idx, k, rel_indptr, rel_items, rel_gains, idcg, discount, users=None, per_user=False):
    """Accuracy metrics of a (rows x >=k) int32 top-k index tensor against an item-sorted relevant-item CSR
    (evaluator.py:117-147 semantics).  Returns (out, per_user): out = device double[5]
    {evaluated users, sum nDCG, sum HR, sum Precision, sum Recall}; per_user = (rows x 4) or None."""
    _need_cuda(topk_idx, rel_indptr, rel_items, rel_gains, idcg, discount, users)
    assert topk_idx.dtype == torch.int32 and topk_idx.stride(1) == 1 and topk_idx.shape[1] >= k
    assert rel_indptr.dtype == torch.int64 and rel_items.dtype == torch.int32
    assert rel_gains.dtype == torch.float64 and idcg.dtype == torch.float64 and discount.dtype == torch.float64
    assert discount.numel() >= k
    n = topk_idx.shape[0]
    if users is not None:
        _chk_idx(users); assert users.numel() == n
    dev = topk_idx.device
    out = torch.empty(5, dtype=torch.float64, device=dev)
    pu = torch.empty(n, 4, dtype=torch.float64, device=dev) if per_user else None
    ws = _scratch("eval_topk", lib().eb_eval_topk_workspace_bytes(n, k), dev)
    _call("eb_eval_topk_f64", topk_idx, _ptr(topk_idx), n, topk_idx.stride(0), k, _ptr(users), _ptr(rel_indptr), _ptr(rel_items),
          _ptr(rel_gains), _ptr(idcg), _ptr(discount), _ptr(pu), _ptr(out), _ptr(ws), ws.numel())
    return out, pu


EVAL_METRICS_SLOTS = 29
EVAL_METRICS_PER_USER = ("nDCGRendle2020", "MRR", "MAP", "MAR", "F1", "LAUC", "NumRetrieved", "EPC", "EFD", "ARP", "APLT",
                         "ACLT")


def eval_topk_metrics(topk_idx, k, rel_indptr, rel_items, user_info, item_pop, item_long_tail, item_novelty, discount,
                      map_tail, inv_binary_idcg, users=None, per_user=False):
    """The reference's ranking, novelty, popularity-bias, coverage and diversity metrics of a (rows x >=k) int32 top-k
    index tensor (eval_metrics.cu; tables as in include/elliot_b200.h).  Returns (out, per_user): out = device
    double[29] of counts, sums and numerators; per_user = (rows x 12) in EVAL_METRICS_PER_USER order, or None."""
    _need_cuda(topk_idx, rel_indptr, rel_items, user_info, item_pop, item_long_tail, item_novelty, discount, map_tail,
               inv_binary_idcg, users)
    assert topk_idx.dtype == torch.int32 and topk_idx.stride(1) == 1 and topk_idx.shape[1] >= k
    assert rel_indptr.dtype == torch.int64 and rel_items.dtype == torch.int32
    assert user_info.dtype == torch.int32 and user_info.is_contiguous() and user_info.shape[1:] == (6,)
    assert user_info.shape[0] == rel_indptr.numel() - 1
    n_items = item_pop.numel()
    assert item_pop.dtype == torch.int32 and item_long_tail.dtype == torch.uint8 and item_long_tail.numel() == n_items
    assert item_novelty.dtype == torch.float64 and item_novelty.is_contiguous() and item_novelty.shape == (n_items, 2)
    for t in (discount, map_tail, inv_binary_idcg):
        assert t.dtype == torch.float64 and t.is_contiguous()
    assert discount.numel() >= k and map_tail.numel() >= k and inv_binary_idcg.numel() >= k + 1
    n = topk_idx.shape[0]
    if users is not None:
        _chk_idx(users); assert users.numel() == n
    dev = topk_idx.device
    out = torch.empty(EVAL_METRICS_SLOTS, dtype=torch.float64, device=dev)
    pu = torch.empty(n, len(EVAL_METRICS_PER_USER), dtype=torch.float64, device=dev) if per_user else None
    ws = _scratch("eval_metrics", lib().eb_eval_metrics_workspace_bytes(n, k, n_items), dev)
    _call("eb_eval_metrics_f64", topk_idx, _ptr(topk_idx), n, topk_idx.stride(0), k, _ptr(users), _ptr(rel_indptr),
          _ptr(rel_items), _ptr(user_info), _ptr(item_pop), _ptr(item_long_tail), _ptr(item_novelty), n_items, _ptr(discount),
          _ptr(map_tail), _ptr(inv_binary_idcg), _ptr(pu), _ptr(out), _ptr(ws), ws.numel())
    return out, pu


def eval_fairness(topk_idx, k, rel_indptr, rel_items, rel_gains, idcg, discount, has_rows, user_cluster, n_user_clusters,
                  item_cluster, n_item_clusters, scores=None, users=None):
    """Counts and sums of the reference's clustered fairness metrics over a (rows x >=k) int32 top-k index tensor
    (eval_fairness.cu; layout in include/elliot_b200.h).  scores: the lists' (rows x >=k) scores, fp64 or fp32 (cast
    once, exactly), read only by the rating sums.  Returns (counts int64, sums fp64) device tensors."""
    _need_cuda(topk_idx, rel_indptr, rel_items, rel_gains, idcg, discount, has_rows, user_cluster, item_cluster, scores,
               users)
    assert topk_idx.dtype == torch.int32 and topk_idx.stride(1) == 1 and topk_idx.shape[1] >= k
    assert rel_indptr.dtype == torch.int64 and rel_items.dtype == torch.int32
    for t in (rel_gains, idcg, discount):
        assert t.dtype == torch.float64 and t.is_contiguous()
    assert discount.numel() >= k
    n_users = rel_indptr.numel() - 1
    assert has_rows.dtype == torch.uint8 and has_rows.numel() == n_users
    _chk_idx(user_cluster, item_cluster)
    assert user_cluster.numel() == n_users and n_user_clusters >= 1 and n_item_clusters >= 1
    n = topk_idx.shape[0]
    if users is not None:
        _chk_idx(users); assert users.numel() == n
    if scores is not None:
        assert scores.shape[0] == n and scores.shape[1] >= k
        if scores.dtype != torch.float64 or scores.stride() != topk_idx.stride():
            scores = torch.empty_strided(topk_idx.shape, topk_idx.stride(), dtype=torch.float64,
                                         device=topk_idx.device).copy_(scores[:, :topk_idx.shape[1]])
    dev = topk_idx.device
    nu, ni, n_items = int(n_user_clusters), int(n_item_clusters), item_cluster.numel()
    counts = torch.empty(nu + nu * ni + 3 * ni, dtype=torch.int64, device=dev)
    sums = torch.empty(2 * nu + 2 * ni, dtype=torch.float64, device=dev)
    ws = _scratch("eval_fairness", lib().eb_eval_fairness_workspace_bytes(n, k, n_items, nu, ni), dev)
    _call("eb_eval_fairness_f64", topk_idx, _ptr(topk_idx), _ptr(scores), n, topk_idx.stride(0), k, _ptr(users),
          _ptr(rel_indptr), _ptr(rel_items), _ptr(rel_gains), _ptr(idcg), _ptr(discount), _ptr(has_rows),
          _ptr(user_cluster), nu, _ptr(_nonempty(item_cluster)), ni, n_items, _ptr(counts), _ptr(sums), _ptr(ws),
          ws.numel())
    return counts, sums


def partition_streams(device, reserve_sms, n_streams=1):
    """Streams bound to a green context that leaves >= reserve_sms SMs of `device` free (partition.cu).
    Returns (list of torch streams, SMs in the partition)."""
    arr = (ctypes.c_void_p * n_streams)()
    granted = ctypes.c_int(0)
    with torch.cuda.device(device):
        check(lib().eb_partition_streams_create(int(reserve_sms), n_streams, arr, ctypes.byref(granted)))
    return [torch.cuda.ExternalStream(int(arr[k]), device=device) for k in range(n_streams)], granted.value


# ---------------------------------------------------------------- row-sharded tables (sharded.cu)
def gather_rows_f32(table, ids, width=None, out=None):
    _need_cuda(table, ids, out); _chk_idx(ids)
    width = width or table.shape[1]
    if out is None:
        out = torch.empty((ids.numel(), table.stride(0)), dtype=torch.float32, device=table.device)
    _call("eb_gather_rows_f32", table, _ptr(table), table.stride(0), _ptr(ids), ids.numel(), width, _ptr(out), out.stride(0))
    return out


def scatter_add_rows_f32(table, ids, rows, width=None):
    _need_cuda(table, ids, rows); _chk_idx(ids)
    width = width or table.shape[1]
    _call("eb_scatter_add_rows_f32", table, _ptr(table), table.stride(0), _ptr(ids), ids.numel(), width, _ptr(rows), rows.stride(0))


def bpr_step_rows_f32(U, tu, Ri, Rj, bias_col, lr, reg_u, reg_b, reg_pos, reg_neg, loss=None):
    """BPR update against fetched item rows; returns (dRi, dRj) deltas to send back to the owners."""
    _need_cuda(U, tu, Ri, Rj, loss); _chk_idx(tu)
    dRi, dRj = torch.empty_like(Ri), torch.empty_like(Rj)
    _call("eb_bpr_step_rows_f32", U, _ptr(U), U.stride(0), _ptr(tu), _ptr(Ri), _ptr(Rj), Ri.stride(0), tu.numel(), bias_col,
          lr, reg_u, reg_b, reg_pos, reg_neg, _ptr(dRi), _ptr(dRj), _ptr(loss))
    return dRi, dRj


# ---------------------------------------------------------------- peer-addressed tables (csrc/peer.cu, bpr_train.cu PEER mode)
def _ptr_array(ptrs):
    """HOST array of device addresses (the `*_shards` arguments of the C ABI): ints, tensors, or a ready ctypes array."""
    if isinstance(ptrs, ctypes.Array):
        return ptrs, len(ptrs)
    vals = [p.data_ptr() if torch.is_tensor(p) else int(p) for p in ptrs]
    return (ctypes.c_void_p * len(vals))(*vals), len(vals)


def bpr_step_peer_f32(U, V_shards, b_shards, shard_rows, d, n_items, tu, ti, tj, lr, reg_u, reg_b, reg_pos, reg_neg, loss=None,
                      _variant=0):
    """BPR step on materialised triples, item table + biases row-sharded (shard s = rows [s*shard_rows, (s+1)*shard_rows)).
    _variant (profiling): 16 forces the register-staged kernel, 32 the shared-memory-staged one (the default)."""
    _need_cuda(U, tu, ti, tj, loss); _chk_idx(tu, ti, tj)
    va, n = _ptr_array(V_shards); ba, nb = _ptr_array(b_shards)
    assert n == nb and U.dtype == torch.float32 and U.stride(1) == 1
    _call("eb_bpr_step_peer_f32", U, _ptr(U), va, ba, n, shard_rows, d, U.stride(0), n_items, _ptr(tu), _ptr(ti), _ptr(tj),
          tu.numel(), lr, reg_u, reg_b, reg_pos, reg_neg, _ptr(loss), _bpr_flags(variant=_variant))


def bpr_step_sampled_peer_f32(U, V_shards, b_shards, shard_rows, d, n_users, n_items, indptr, indices, n, seed, first, lr, reg_u,
                              reg_b, reg_pos, reg_neg, loss=None, out=None, reserve_sms=0, filter=None, _variant=0):
    """Fused sample+update step with the item table row-sharded over the GPUs of the box (loads / atomics over NVLink).
    _variant (profiling): 16 forces the register-staged kernel, 32 the shared-memory-staged one (the default)."""
    _need_cuda(U, indptr, indices, loss)
    assert indptr.dtype == torch.int64 and indices.dtype == torch.int32 and U.dtype == torch.float32 and U.stride(1) == 1
    va, ns = _ptr_array(V_shards); ba, nb = _ptr_array(b_shards)
    assert ns == nb
    out = _out_ptrs(out)
    _call("eb_bpr_step_sampled_peer_f32", U, _ptr(U), va, ba, ns, shard_rows, d, U.stride(0), n_users, n_items, _ptr(indptr),
          _ptr(indices), _ptr(filter), 0 if filter is None else filter.shape[1], n, seed, first, lr, reg_u, reg_b, reg_pos, reg_neg,
          _ptr(loss), *out, _bpr_flags(variant=_variant, reserve_sms=reserve_sms))


def table_reconcile_peer_f32(slice_ptrs, prev_slice, scale, max_ctas=0):
    """One-kernel reconciliation of a replicated table's slice (see eb_table_reconcile_peer_f32)."""
    _need_cuda(prev_slice)
    pa, n = _ptr_array(slice_ptrs)
    _call("eb_table_reconcile_peer_f32", prev_slice, pa, n, _ptr(prev_slice), prev_slice.numel(), float(scale), int(max_ctas))


def neumf_gather_peer(Umf, Umlp, I_shards, shard_rows, ldi, f, u, it, x0, pm):
    _need_cuda(Umf, Umlp, u, it, x0, pm)
    ia, n = _ptr_array(I_shards)
    _call("eb_neumf_gather_peer", Umf, _ptr(Umf), _ptr(Umlp), Umf.stride(0), ia, n, shard_rows, ldi, f, _ptr(u), _ptr(it), u.numel(),
          _ptr(x0), x0.stride(0), _ptr(pm), pm.stride(0))


def neumf_scatter_peer(Umf, I_shards, GI_shards, shard_rows, ldi, f, u, it, dpm, dx0, dUmf, dUmlp):
    _need_cuda(Umf, u, it, dpm, dx0, dUmf, dUmlp)
    ia, n = _ptr_array(I_shards); ga, ng = _ptr_array(GI_shards)
    assert n == ng
    _call("eb_neumf_scatter_peer", Umf, _ptr(Umf), Umf.stride(0), ia, ga, n, shard_rows, ldi, f, _ptr(u), _ptr(it), u.numel(),
          _ptr(dpm), dpm.stride(0), _ptr(dx0), dx0.stride(0), _ptr(dUmf), _ptr(dUmlp))


def group_by_owner(arrays, key1, key2, shard_rows, rank, world):
    """Reorder up to three 32-bit arrays that travel together so that elements whose row (arrays[key1], and arrays[key2] if
    key2 >= 0) lives on the same owner are adjacent, starting with rank+1's rows (see eb_group_by_owner_i32: with more than four
    GPUs a peer kernel fed in this order moves rows 12x faster).  float32 payloads are carried bit for bit.  Returns new tensors."""
    arrays = list(arrays) + [None] * (3 - len(arrays))
    _need_cuda(*[x for x in arrays if x is not None])
    views = [None if x is None else x.view(torch.int32) for x in arrays]
    n = views[0].numel()
    outs = [None if v is None else torch.empty_like(v) for v in views]
    work = torch.empty(128, dtype=torch.int32, device=views[0].device)
    _call("eb_group_by_owner_i32", views[0], _ptr(views[0]), _ptr(views[1]), _ptr(views[2]), key1, key2, n, shard_rows, rank, world,
          _ptr(outs[0]), _ptr(outs[1]), _ptr(outs[2]), _ptr(work))
    return [None if o is None else o.view(x.dtype) for o, x in zip(outs, arrays)]


def gather_rows_peer_f32(shards, shard_rows, ld, ids, width, out=None):
    _need_cuda(ids, out); _chk_idx(ids)
    sa, n = _ptr_array(shards)
    if out is None:
        out = torch.empty((ids.numel(), width), dtype=torch.float32, device=ids.device)
    _call("eb_gather_rows_peer_f32", ids, sa, n, shard_rows, ld, _ptr(ids), ids.numel(), width, _ptr(out), out.stride(0))
    return out


# ---------------------------------------------------------------- GMF (csrc/gmf.cu)
def pointwise_sample_philox(n_users, n_items, indptr, indices, n, seed, first=0, filter=None):
    """(u, item, label) samples of pointwise_pos_neg_sampler.py:24-48 (Philox stream)."""
    _need_cuda(indptr, indices, filter)
    dev = indptr.device
    u = torch.empty(n, dtype=torch.int32, device=dev); i = torch.empty_like(u); y = torch.empty(n, dtype=torch.float32, device=dev)
    _call("eb_pointwise_sample_philox", indptr, n_users, n_items, _ptr(indptr), _ptr(indices), _ptr(filter),
          0 if filter is None else filter.shape[1], n, seed, first, _ptr(u), _ptr(i), _ptr(y))
    return u, i, y


def gmf_step_grads(U, I, h, f, u, it, label, dU, dI, dh, loss=None, mean_over=None):
    _need_cuda(U, I, h, u, it, label, dU, dI, dh, loss); _chk_idx(u, it)
    assert U.stride(0) == I.stride(0) == dU.stride(0) == dI.stride(0)
    _call("eb_gmf_step_grads", U, _ptr(U), _ptr(I), U.stride(0), f, _ptr(h), _ptr(u), _ptr(it), _ptr(label), u.numel(),
          int(mean_over) if mean_over else max(int(u.numel()), 1), _ptr(dU), _ptr(dI), _ptr(dh), _ptr(loss))


def gmf_scale_rows(src, h, f, out=None):
    _need_cuda(src, h, out)
    if out is None:
        out = torch.zeros_like(src)
    _call("eb_gmf_scale_rows", src, _ptr(src), src.stride(0), src.shape[0], f, _ptr(h), _ptr(out), out.stride(0))
    return out


def sigmoid_(x):
    _need_cuda(x)
    assert x.is_contiguous() and x.dtype == torch.float32
    _call("eb_sigmoid_inplace", x, _ptr(x), x.numel())
    return x


# ---------------------------------------------------------------- SVD++ / FunkSVD (csrc/rating_mf.cu)
def rated_sample_philox(n_users, n_items, indptr, indices, ratings, n, seed, first=0):
    """(u, item, rating) samples of custom_pointwise_sparse_sampler.py:24-39 (Philox stream): u uniform, item uniform over
    u's train row, its train rating; `ratings` float32 aligned with the sorted train CSR `indices`."""
    _need_cuda(indptr, indices, ratings)
    assert ratings.dtype == torch.float32 and ratings.numel() == indices.numel()
    dev = indptr.device
    u = torch.empty(n, dtype=torch.int32, device=dev); i = torch.empty_like(u); r = torch.empty(n, dtype=torch.float32, device=dev)
    _call("eb_rated_sample_philox", indptr, n_users, n_items, _ptr(indptr), _ptr(indices), _ptr(ratings), n, seed, first,
          _ptr(u), _ptr(i), _ptr(r))
    return u, i, r


def implicit_mean_f32(P, Y, f, indptr, indices, users=None, out=None):
    """Z[r] = P[u] + mean over u's train row of Y (u = users[r], or r for every row of P when users is None)."""
    _need_cuda(P, Y, indptr, indices, users, out)
    assert P.stride(0) == Y.stride(0) and P.stride(1) == 1 and Y.stride(1) == 1
    n = P.shape[0] if users is None else users.numel()
    if users is not None:
        _chk_idx(users)
    if out is None:
        out = torch.zeros((n, P.stride(0)), dtype=torch.float32, device=P.device)
    assert out.shape[0] >= n and out.stride(1) == 1
    _call("eb_implicit_mean_f32", P, _ptr(P), _ptr(Y), P.stride(0), f, _ptr(indptr), _ptr(indices), _ptr(users), n, _ptr(out),
          out.stride(0))
    return out


def rating_mf_step_f32(P, Q, bu, bi, g, f, u, it, label, dP, dQ, dbu, dbi, dg, Z=None, indptr=None, indices=None, dY=None,
                       loss=None, mean_over=None):
    """Gradient of the batch's mean squared error of z.q + b_u + b_i (+ g) into the dense gradient tables: z = Z[s] with
    dY over the train rows (SVD++), or P[u] (FunkSVD: Z, dY, g and dg None).  `loss` (fp64) gets the batch loss added."""
    _need_cuda(P, Q, bu, bi, g, u, it, label, dP, dQ, dbu, dbi, dg, Z, indptr, indices, dY, loss)
    _chk_idx(u, it)
    assert P.stride(0) == Q.stride(0) == dP.stride(0) == dQ.stride(0)
    if dY is not None:
        assert dY.stride(0) == P.stride(0)
    _call("eb_rating_mf_step_f32", P, _ptr(P), _ptr(Q), P.stride(0), f, _ptr(bu), _ptr(bi), _ptr(g), _ptr(Z),
          0 if Z is None else Z.stride(0), _ptr(indptr), _ptr(indices), _ptr(u), _ptr(it), _ptr(label), u.numel(),
          int(mean_over) if mean_over else max(int(u.numel()), 1), _ptr(dP), _ptr(dQ), _ptr(dY), _ptr(dbu), _ptr(dbi), _ptr(dg),
          _ptr(loss))


def score_pairs_f32(U, V, f, rel_indptr, rel_items, item_bias=None, user_off=None, global_off=None, mask_indptr=None,
                    mask_indices=None):
    """Per entry of the relevant-item CSR (rows = users 0 .. n-1 of U): (U[u].V[item] + item_bias) + (user_off[u] +
    global_off[0]) as the user's full list carries it; -inf for an item of the user's mask row, NaN for item -1."""
    _need_cuda(U, V, rel_indptr, rel_items, item_bias, user_off, global_off, mask_indptr, mask_indices)
    assert U.dtype == torch.float32 and V.dtype == torch.float32 and U.stride(0) == V.stride(0)
    assert rel_indptr.dtype == torch.int64 and rel_items.dtype == torch.int32 and rel_items.is_contiguous()
    n_users = rel_indptr.numel() - 1
    assert n_users <= U.shape[0]
    out = torch.empty(rel_items.numel(), dtype=torch.float32, device=U.device)
    _call("eb_score_pairs_f32", U, _ptr(U), _ptr(V), U.stride(0), f, _ptr(item_bias), _ptr(user_off), _ptr(global_off),
          _ptr(rel_indptr), _ptr(_nonempty(rel_items)), n_users, _ptr(mask_indptr), _ptr(mask_indices), _ptr(out))
    return out


def add_row_offset_(x, row_off, scalar_off=None):
    """x[r][:] += row_off[r] (+ scalar_off[0]) in place, for a 2-D fp32 x with unit column stride."""
    _need_cuda(x, row_off, scalar_off)
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1 and row_off.numel() >= x.shape[0]
    _call("eb_add_row_offset_f32", x, _ptr(x), x.shape[0], x.shape[1], x.stride(0), _ptr(row_off), _ptr(scalar_off))
    return x


def rating_error_sums(scores, ratings, items):
    """Device fp64 [sum |v - r|, sum (v - r)^2] over the entries with items >= 0 (fixed summation order)."""
    _need_cuda(scores, ratings, items)
    assert scores.dtype == torch.float32 and ratings.dtype == torch.float64 and items.dtype == torch.int32
    n = scores.numel()
    assert ratings.numel() == n and items.numel() == n
    out = torch.empty(2, dtype=torch.float64, device=scores.device)
    _call("eb_rating_error_sums_f64", scores, _ptr(_nonempty(scores)), _ptr(_nonempty(ratings)), _ptr(_nonempty(items)), n, _ptr(out))
    return out


# ---------------------------------------------------------------- PMF / LMF / FM labels (csrc/pointwise_mf.cu)
PMF_MSE, LMF_LOGPOST = 0, 1


def pointwise_mf_step_f32(P, Q, f, u, it, label, dQ, kind, dP=None, bu=None, bi=None, dbi=None, alpha=0.0, lam=0.0, loss=None,
                          mean_over=None):
    """Batch gradient of PMF's mean squared error of sigmoid(p.q) (kind PMF_MSE: into dP, dQ) or of LMF's summed log
    posterior of p.q + b_u + b_i with lam (|p|^2 + |q|^2) / 2 (kind LMF_LOGPOST: item side only, into dQ, dbi); `loss`
    (fp64) gets the batch loss added."""
    _need_cuda(P, Q, u, it, label, dQ, dP, bu, bi, dbi, loss)
    _chk_idx(u, it)
    assert P.stride(0) == Q.stride(0) == dQ.stride(0) and (dP is None or dP.stride(0) == P.stride(0))
    _call("eb_pointwise_mf_step_f32", P, _ptr(P), _ptr(Q), P.stride(0), f, _ptr(bu), _ptr(bi), _ptr(u), _ptr(it), _ptr(label),
          u.numel(), int(kind), int(mean_over) if mean_over else max(int(u.numel()), 1), float(alpha), float(lam), _ptr(dP),
          _ptr(dQ), _ptr(dbi), _ptr(loss))


def adagrad_rows_f32(var, acc, grad, rows, stamp, step, lr, width=None, bvar=None, bacc=None, bgrad=None, eps=1e-7):
    """TF's sparse Adagrad on every distinct row listed in `rows` (int32, repeats allowed), once, then those gradient rows
    (and bias entries) cleared.  stamp: int64 [n_rows] zeros at the start, kept with the tables; step: > every step this
    stamp table has seen."""
    _need_cuda(var, acc, grad, rows, stamp, bvar, bacc, bgrad)
    _chk_idx(rows)
    assert var.stride(0) == acc.stride(0) == grad.stride(0) and var.stride(1) == 1 and stamp.dtype == torch.int64
    _call("eb_adagrad_rows_f32", var, _ptr(var), _ptr(acc), _ptr(grad), var.stride(0), var.shape[1] if width is None else width,
          _ptr(bvar), _ptr(bacc), _ptr(bgrad), _ptr(rows), rows.numel(), _ptr(stamp), int(step), float(lr), float(eps))


def rating_labels_(indptr, indices, ratings, u, it, label):
    """label[s] <- the train rating of (u[s], it[s]) for every positive (label != 0) sample, in place; `ratings` float32
    aligned with the sorted train CSR `indices`."""
    _need_cuda(indptr, indices, ratings, u, it, label)
    _chk_idx(u, it)
    assert ratings.dtype == torch.float32 and ratings.numel() == indices.numel() and label.dtype == torch.float32
    _call("eb_rating_labels_f32", indptr, _ptr(indptr), _ptr(indices), _ptr(ratings), _ptr(u), _ptr(it), _ptr(label), u.numel())
    return label


def sigmoid_scores_(x):
    """sigmoid of every score of x in place; -inf (a masked item) and NaN (outside the catalogue) stay as they are."""
    _need_cuda(x)
    assert x.is_contiguous() and x.dtype == torch.float32
    _call("eb_sigmoid_scores_f32", x, _ptr(x), x.numel())
    return x


# ---------------------------------------------------------------- CML (csrc/cml.cu)
def cml_grad_f32(Gu, Gi, Bi, dGu, dGi, dBi, d, tu, ti, tj, l_w, l_b, margin, loss=None, terms=None):
    """Batch gradient of the CML loss (CML_model.py:59-98, the reference's B x B broadcast, counted by sorting) into dense
    gradient tables; `loss` (fp64) gets the batch loss added.  terms (float32, 2n): receives D then E in triple order
    (None: device scratch)."""
    _need_cuda(Gu, Gi, Bi, dGu, dGi, dBi, tu, ti, tj, loss, terms)
    _chk_idx(tu, ti, tj)
    assert Gu.stride(0) == Gi.stride(0) == dGu.stride(0) == dGi.stride(0)
    n = tu.numel()
    if terms is None:
        terms = _scratch("cml_terms", 8 * n, Gu.device)
    else:
        assert terms.dtype == torch.float32 and terms.is_contiguous() and terms.numel() >= 2 * n
    ws = _scratch("cml", lib().eb_cml_workspace_bytes(n), Gu.device)
    _call("eb_cml_grad_f32", Gu, _ptr(Gu), _ptr(Gi), _ptr(Bi), _ptr(dGu), _ptr(dGi), _ptr(dBi), d, Gu.stride(0), _ptr(tu),
          _ptr(ti), _ptr(tj), n, l_w, l_b, margin, _ptr(terms), _ptr(loss), _ptr(ws), ws.numel())


def cml_score_operands_f32(Gu, Gi, Bi, n_users, n_items):
    """(U2, item_off, user_off): 2 Gu, Bi - |Gi|^2 and -|Gu|^2 per row, so that the dot-product scorers on
    (U2, Gi, item_off) plus user_off give CML's Bi - |Gu - Gi|^2 (CML_model.py:101-106)."""
    _need_cuda(Gu, Gi, Bi)
    assert Gu.dtype == Gi.dtype == Bi.dtype == torch.float32 and Gu.is_contiguous() and Gi.is_contiguous()
    assert Gu.stride(0) == Gi.stride(0) and Gu.shape[0] >= n_users and Gi.shape[0] >= n_items and Bi.numel() >= n_items
    U2 = torch.empty((n_users, Gu.shape[1]), dtype=torch.float32, device=Gu.device)
    item_off = torch.empty(n_items, dtype=torch.float32, device=Gu.device)
    user_off = torch.empty(n_users, dtype=torch.float32, device=Gu.device)
    _call("eb_cml_score_operands_f32", Gu, _ptr(Gu), _ptr(Gi), _ptr(Bi), Gu.stride(0), n_users, n_items, _ptr(U2), _ptr(item_off),
          _ptr(user_off))
    return U2, item_off, user_off


# ---------------------------------------------------------------- DMF (csrc/dmf.cu)
def dmf_sparse_fwd(W1, b1, indptr, indices, values, rows, h1, relu):
    """h1[b] = act(X[rows[b]] . W1 + b1), X the CSR (indptr, indices, values); W1 [n_cols][H] fp32."""
    _need_cuda(W1, b1, indptr, indices, values, rows, h1)
    _chk_idx(rows)
    assert W1.is_contiguous() and h1.stride(1) == 1 and values.dtype == torch.float32
    _call("eb_dmf_sparse_fwd_f32", W1, _ptr(W1), _ptr(b1), W1.shape[1], _ptr(indptr), _ptr(indices), _ptr(values), _ptr(rows),
          rows.numel(), 1 if relu else 0, _ptr(h1), h1.stride(0))
    return h1


def dmf_sparse_bwd(dW1, indptr, indices, values, rows, dpre1):
    """dW1 += X[rows]^T . dpre1."""
    _need_cuda(dW1, indptr, indices, values, rows, dpre1)
    _chk_idx(rows)
    assert dW1.is_contiguous() and dpre1.stride(1) == 1
    _call("eb_dmf_sparse_bwd_f32", dW1, _ptr(dW1), dW1.shape[1], _ptr(indptr), _ptr(indices), _ptr(values), _ptr(rows),
          rows.numel(), _ptr(dpre1), dpre1.stride(0))


def dmf_head_f32(U, V, F, label, max_rating, cosine, loss, dU, dV, prob=None):
    """One batch of DMF's head (model.py:76-77, 93-105): batch-axis cosine (or dot), clipped BCE against label /
    max_rating; `loss` (fp64 [1]) gets the batch mean added, dU / dV the gradients.  U, V, dU, dV [B][ld] fp32."""
    _need_cuda(U, V, label, loss, dU, dV, prob)
    assert U.stride(0) == V.stride(0) and dU.stride(0) == dV.stride(0) and U.stride(1) == 1 and dU.stride(1) == 1
    B = U.shape[0]
    ws = _scratch("dmf_head", lib().eb_dmf_head_workspace_bytes(B, F), U.device)
    _call("eb_dmf_head_f32", U, _ptr(U), _ptr(V), U.stride(0), F, B, _ptr(label), float(max_rating), 1 if cosine else 0,
          _ptr(loss), _ptr(dU), _ptr(dV), dU.stride(0), _ptr(prob), _ptr(ws), ws.numel())


def dmf_score_operands_f32(Uo, Vo, F, block, cosine):
    """(Uh, Vh, Vh_last) of get_recs (model.py:106-121) for user blocks of `block`: each block's users scaled by the block's
    column norms, items by 1 / sqrt(block V^2) (Vh_last: the short last block's size; None when there is none), row
    stride padded_dim(F).  The dot-product scorers on (Uh rows of a block, Vh of that block) give the reference's scores."""
    _need_cuda(Uo, Vo)
    n_users, n_items = Uo.shape[0], Vo.shape[0]
    ld = padded_dim(F)
    Uh = torch.empty((n_users, ld), dtype=torch.float32, device=Uo.device)
    Vh = torch.empty((n_items, ld), dtype=torch.float32, device=Uo.device)
    bl = min(int(block), n_users)
    Vl = torch.empty_like(Vh) if cosine and n_users % bl else None
    _call("eb_dmf_score_operands_f32", Uo, _ptr(Uo), Uo.stride(0), _ptr(Vo), Vo.stride(0), F, n_users, n_items, bl,
          1 if cosine else 0, _ptr(Uh), _ptr(Vh), _ptr(Vl), ld)
    return Uh, Vh, Vl


# ---------------------------------------------------------------- UserAutoRec / ItemAutoRec (csrc/autorec.cu)
def autorec_decoder_f32(indptr, indices, values, rows, h, W2, b2, act, loss, dW2, db2, dpre1, scale=None, max_entries=None):
    """One training step's decoder and its backward over the observed entries of the CSR rows `rows`
    (userautorec_model.py:92-107): `loss` (fp64 [1]) gets scale sum e^2 added, dW2 / db2 the decoder gradients (added),
    dpre1 [B][H] the gradient at the encoder's pre-activation (written).  act 0 = linear, 1 = sigmoid; scale defaults to
    1 / B; max_entries (the most entries the rows can hold) defaults to the CSR's nnz, which distinct rows never pass."""
    _need_cuda(indptr, indices, values, rows, h, W2, b2, loss, dW2, db2, dpre1)
    _chk_idx(rows, indices)
    assert W2.is_contiguous() and dW2.is_contiguous() and h.stride(1) == 1 and dpre1.stride(1) == 1
    assert values.dtype == torch.float32 and loss.dtype == torch.float64
    B, H = rows.numel(), W2.shape[1]
    if max_entries is None:
        max_entries = indices.numel()
    ws = _scratch("autorec", lib().eb_autorec_decoder_workspace_bytes(B, H, max_entries), W2.device)
    _call("eb_autorec_decoder_f32", W2, _ptr(indptr), _ptr(indices), _ptr(values), _ptr(rows), B, max_entries, _ptr(h),
          h.stride(0), _ptr(W2), _ptr(b2), H, int(act), float(1.0 / max(B, 1) if scale is None else scale), _ptr(dW2),
          _ptr(db2), _ptr(dpre1), dpre1.stride(0), _ptr(loss), _ptr(ws), ws.numel())


# ---------------------------------------------------------------- ConvNeuMF (csrc/convneumf.cu)
def convneumf_widths(channels):
    """The scorer's packed channel widths: byte l - 1 = c_l."""
    w = 0
    for l, c in enumerate(channels):
        w |= int(c) << (8 * l)
    return w


def convneumf_l1_fwd(U, I, f, pu, pi, L, HL, W1, b1, c1, out):
    """Level-1 outputs of the pairs (U[pu[p]], I[pi[p]]) into out [n_pairs R_1][c1], Z-order rows; out bf16, or fp32 in
    the exact_gemm checking mode."""
    _need_cuda(U, I, pu, pi, W1, b1, out)
    _chk_idx(pu, pi)
    assert U.stride(0) == I.stride(0) and out.is_contiguous() and out.dtype in (torch.bfloat16, torch.float32)
    _call("eb_convneumf_l1_fwd", U, _ptr(U), _ptr(I), U.stride(0), f, _ptr(pu), _ptr(pi), pu.numel(), L, HL, c1, _ptr(W1),
          _ptr(b1), _ptr(out), 1 if out.dtype == torch.bfloat16 else 0)
    return out


def convneumf_l1_bwd(U, I, f, pu, pi, n_user_reg, L, HL, W1, b1, c1, dx1, l_w, dU, dI, dW1, db1):
    """Adds the level-1 gradients of the pairs (dW1, db1, dU / dI rows, plus l_w times the rows) from dx1, the gradient at
    the level-1 outputs."""
    _need_cuda(U, I, pu, pi, W1, b1, dx1, dU, dI, dW1, db1)
    _chk_idx(pu, pi)
    assert U.stride(0) == I.stride(0) == dU.stride(0) == dI.stride(0) and dx1.dtype == torch.float32 and dx1.is_contiguous()
    _call("eb_convneumf_l1_bwd", U, _ptr(U), _ptr(I), U.stride(0), f, _ptr(pu), _ptr(pi), pu.numel(), int(n_user_reg), L, HL,
          c1, _ptr(W1), _ptr(b1), _ptr(dx1), float(l_w), _ptr(dU), _ptr(dI), _ptr(dW1), _ptr(db1))


def convneumf_head(hL, RL, cL, Wd1, bd1, wd2, bd2, U, I, f, tu, ti, tj, first, n_total, p_drop, seed, l_w, loss, dWd1, dbd1,
                   dwd2, dbd2, dpre, y_out=None, mask_out=None):
    """Head, clipped BPR loss and their gradients for the triples (tu, ti, tj), triples first .. first + n of a batch of
    n_total: see include/elliot_b200.h."""
    _need_cuda(hL, Wd1, bd1, wd2, bd2, U, I, tu, ti, tj, loss, dWd1, dbd1, dwd2, dbd2, dpre, y_out, mask_out)
    _chk_idx(tu, ti, tj)
    assert hL.dtype == torch.float32 and hL.is_contiguous() and dpre.is_contiguous() and loss.dtype == torch.float64
    _call("eb_convneumf_head", hL, _ptr(hL), int(RL), cL, _ptr(Wd1), _ptr(bd1), _ptr(wd2), _ptr(bd2), _ptr(U), _ptr(I),
          U.stride(0), f, _ptr(tu), _ptr(ti), _ptr(tj), tu.numel(), int(first), int(n_total), float(p_drop), int(seed),
          float(l_w), _ptr(loss), _ptr(dWd1), _ptr(dbd1), _ptr(dwd2), _ptr(dbd2), _ptr(dpre), _ptr(y_out), _ptr(mask_out))


def convneumf_score_smem_bytes(f, L, HL, channels):
    return int(lib().eb_convneumf_score_smem_bytes(f, L, HL, convneumf_widths(channels)))


def convneumf_score(U, I, f, L, HL, channels, W1, b1, Wp, bp, Wd1, bd1, wd2, bd2, u0, n_ub, n_items, out=None):
    """Dense fp32 scores [n_ub][n_items] of users u0 .. u0 + n_ub - 1 against every item (dropout off), one fused kernel.
    Wp: bf16 W_l [c_l][4 c_(l-1)] for l = 2..L back to back (None at L = 1), bp: fp32 b_l back to back."""
    _need_cuda(U, I, W1, b1, Wp, bp, Wd1, bd1, wd2, bd2, out)
    assert U.stride(0) == I.stride(0) and (Wp is None or Wp.dtype == torch.bfloat16)
    if out is None:
        out = torch.empty((n_ub, n_items), dtype=torch.float32, device=U.device)
    _call("eb_convneumf_score", U, _ptr(U), _ptr(I), U.stride(0), f, L, HL, convneumf_widths(channels), _ptr(W1), _ptr(b1),
          _ptr(Wp), _ptr(bp), _ptr(Wd1), _ptr(bd1), _ptr(wd2), _ptr(bd2), int(u0), int(n_ub), int(n_items), _ptr(out),
          out.stride(0))
    return out


def dense_rank(scores, rel_indptr, rel_items, mask_indptr=None, mask_indices=None, rows=None, row_begin=0):
    """(n_pos, sum_c) of score_rank for the rows of a dense fp32 score block: row q is user rows[q] (or row_begin + q)."""
    _need_cuda(scores, rel_indptr, rel_items, mask_indptr, mask_indices, rows)
    assert scores.dtype == torch.float32 and scores.stride(1) == 1
    assert rel_indptr.dtype == torch.int64 and rel_items.dtype == torch.int32 and rel_items.is_contiguous()
    if rows is not None:
        _chk_idx(rows)
    n = scores.shape[0]
    n_pos, sum_c = (torch.empty(n, dtype=torch.int64, device=scores.device) for _ in range(2))
    _call("eb_dense_rank_f32", scores, _ptr(scores), scores.stride(0), n, scores.shape[1], _ptr(rows), int(row_begin),
          _ptr(mask_indptr), _ptr(mask_indices), _ptr(rel_indptr), _ptr(_nonempty(rel_items)), _ptr(n_pos), _ptr(sum_c))
    return n_pos, sum_c
