"""torchrun --nproc-per-node N tools/peer_check.py [--sections a,b,...] : the peer-addressed multi-GPU paths on real GPUs.

Sections (each records ok / numbers / error in gpurun_out/peer_check_n{N}.json; rank 0 prints the JSON):
  map        PeerBuffer mapping (which mechanism), every rank reads every other rank's block through its peer address
  p2p        raw NVLink row traffic: random 256-B rows gathered from all shards (GB/s into one GPU)
  bpr        row-sharded item table: conflict-free batch == single-table kernel; throughput of the fused
             sample+gather+update kernel at a C4-like BPR shape (1 M local users, 1 M x N items sharded, d=64)
  reconcile  replicated table (C2 size): all copies agree on base + mean of the ranks' steps; kernel time;
             C2 training step + reconcile, triples/s
  neumf      ShardedNeuMFModel vs the single-GPU model on the same global batches (rel <= 1e-3), sharded scoring,
             then the C4-shape step (users 2.5 M / GPU, 1 M items, d=64, m=4): samples/s and NVLink bytes/sample
"""
import argparse
import json
import os
import sys
import time
import traceback

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from elliot_b200 import ops                                                            # noqa: E402
from elliot_b200.parallel import PeerShardedTable, PeerTableSync, ceil_shard, shard_range   # noqa: E402
from elliot_b200.peer import PeerBuffer                                                # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--sections", default="map,p2p,bpr,reconcile,neumf")
ap.add_argument("--neumf-users", type=int, default=10_000_000)
ap.add_argument("--neumf-items", type=int, default=1_000_000)
ap.add_argument("--neumf-batch", type=int, default=1 << 20)
args = ap.parse_args()
os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)
HP = (0.05, 0.0025, 0.0, 0.0025, 0.00025)
out = {"world": world}


def barrier():
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    barrier()
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    z.record(); torch.cuda.synchronize()
    t = torch.tensor([a.elapsed_time(z) / reps], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def all_ok(flag):
    t = torch.tensor([0 if flag else 1], device=dev, dtype=torch.int32)
    if world > 1:
        dist.all_reduce(t)
    return int(t.item()) == 0


def section(name):
    def deco(fn):
        if name not in args.sections.split(","):
            return fn
        try:
            res = fn()
            out[name] = res
        except Exception as e:                                                   # noqa: BLE001
            out[name] = {"ok": False, "error": repr(e), "trace": traceback.format_exc()[-1500:]}
            sys.stderr.write(f"[rank {rank}] section {name} failed: {e!r}\n")
        barrier()
        return fn
    return deco


@section("map")
def _map():
    res = {}
    for method in ("ipc", "symm"):
        try:
            buf = PeerBuffer(1 << 20, device=dev, method=method)
            buf.local.fill_(float(rank + 1))
            buf.barrier()
            ids = torch.arange(world, dtype=torch.int32, device=dev) * (1 << 18)        # first row of every shard (4-float rows)
            rows = ops.gather_rows_peer_f32(buf.ptr_array(), 1 << 18, 4, ids, 4)
            good = all_ok(torch.equal(rows[:, 0].cpu(), torch.arange(1, world + 1, dtype=torch.float32)))
            res[method] = {"ok": good, "kind": buf.kind}
            buf.close()
        except Exception as e:                                                   # noqa: BLE001
            res[method] = {"ok": False, "error": repr(e)[:300]}
    res["ok"] = res["ipc"]["ok"] or res["symm"]["ok"]
    return res


@section("p2p")
def _p2p():
    ld, rows_per = 64, 1_000_000
    tab = PeerShardedTable(rows_per * world, ld, device=dev)
    tab.local.normal_(generator=None)
    tab.barrier()
    g = torch.Generator(device=dev); g.manual_seed(rank)
    n = 1 << 22
    ids = torch.randint(0, rows_per * world, (n,), device=dev, generator=g, dtype=torch.int32)
    dst = torch.empty((n, ld), device=dev)
    ms = timed(lambda: ops.gather_rows_peer_f32(tab.ptrs, tab.shard_rows, ld, ids, ld, out=dst), 5)
    remote = (world - 1) / world
    res = {"ok": True, "rows": n, "ms": ms, "row_GBps_total": n * 256 / ms / 1e6, "nvlink_in_GBps": n * 256 * remote / ms / 1e6}
    tab.close()
    return res


@section("bpr")
def _bpr():
    res = {}
    # (1) correctness: conflict-free batch, every rank disjoint users and disjoint items
    ni, d, nu_loc, n = 4096, 64, 512, 256
    g = torch.Generator(device=dev); g.manual_seed(5)
    V = torch.randn(ni, d, device=dev, generator=g) * 0.1
    gu = torch.Generator(device=dev); gu.manual_seed(100 + rank)
    U = torch.randn(nu_loc, d, device=dev, generator=gu) * 0.1
    items = PeerShardedTable(ni, d, device=dev)
    bias = PeerBuffer(items.shard_rows, device=dev)
    items.load_from_full(V)
    items.barrier()
    perm = torch.randperm(ni, device=dev, generator=g)
    tu = torch.arange(n, dtype=torch.int32, device=dev)
    ti = perm[rank * 2 * n: rank * 2 * n + n].to(torch.int32).contiguous(); tj = perm[rank * 2 * n + n: (rank + 1) * 2 * n].to(torch.int32).contiguous()
    U_ref, V_ref, b_ref = U.clone(), V.clone(), torch.zeros(ni, device=dev)
    ops.bpr_step_f32(U_ref, V_ref, b_ref, d, tu, ti, tj, *HP)
    ops.bpr_step_peer_f32(U, items.ptrs, bias.ptr_array(), items.shard_rows, d, ni, tu, ti, tj, *HP)
    items.barrier()
    err_u = (U - U_ref).abs().max().item()
    touched = torch.zeros(ni, dtype=torch.bool, device=dev); touched[ti.long()] = True; touched[tj.long()] = True
    mine = V_ref.clone(); mine[~touched] = 0
    cnt = touched.float()
    if world > 1:
        dist.all_reduce(mine); dist.all_reduce(cnt)
    expect = torch.where(cnt[:, None] > 0, mine, V)
    err_v = (items.local[:items.hi - items.lo] - expect[items.lo:items.hi]).abs().max().item()
    res["conflict_free_max_err_user"], res["conflict_free_max_err_item"] = err_u, err_v
    res["ok"] = all_ok(err_u < 1e-6 and err_v < 1e-6)
    items.close(); bias.close()
    # (2) throughput: 1M local users, 1M*world items sharded, d=64, 2^22 triples/step/rank, fused sampler
    nu_loc, ni_tot, per_user, B = 1_000_000, 1_000_000 * world, 50, 1 << 22
    U = torch.randn(nu_loc, d, device=dev, generator=gu) * 0.1
    items = PeerShardedTable(ni_tot, d, device=dev); items.local.normal_(); items.local.mul_(0.1)
    bias = PeerBuffer(items.shard_rows, device=dev)
    cand = (torch.rand(nu_loc, per_user, device=dev, generator=gu) ** 2 * ni_tot).to(torch.int32).clamp_(max=ni_tot - 1)
    cand, _ = torch.sort(cand, dim=1)
    keep = torch.ones_like(cand, dtype=torch.bool); keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    indptr = torch.zeros(nu_loc + 1, dtype=torch.int64, device=dev); indptr[1:] = torch.cumsum(keep.sum(1), 0)
    indices = cand[keep].contiguous()
    del cand, keep
    items.barrier()
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    ctr = [0]

    def step():
        ops.bpr_step_sampled_peer_f32(U, items.ptrs, bias.ptr_array(), items.shard_rows, d, nu_loc, ni_tot, indptr, indices, B,
                                      42 + rank, ctr[0] * B, *HP, loss=loss)
        ctr[0] += 1
    ms = timed(step, 10, warm=3)

    filt = ops.bloom_build(indptr, indices, nu_loc)

    def step_filter():
        ops.bpr_step_sampled_peer_f32(U, items.ptrs, bias.ptr_array(), items.shard_rows, d, nu_loc, ni_tot, indptr, indices, B,
                                      42 + rank, ctr[0] * B, *HP, loss=loss, filter=filt)
        ctr[0] += 1
    res["sharded_step_with_filter_ms"] = timed(step_filter, 10, warm=2)

    def step_reg():                                              # register-staged kernel instead of the shared-memory-staged default
        ops.bpr_step_sampled_peer_f32(U, items.ptrs, bias.ptr_array(), items.shard_rows, d, nu_loc, ni_tot, indptr, indices, B,
                                      42 + rank, ctr[0] * B, *HP, loss=loss, _variant=16)
        ctr[0] += 1
    res["sharded_step_register_kernel_ms"] = timed(step_reg, 10, warm=2)
    finite = all_ok(bool(torch.isfinite(items.local).all().item() and torch.isfinite(U).all().item()))
    res.update({"sharded_step_ms": ms, "triples_per_s_all_ranks": B * world / (ms * 1e-3), "triples_per_s_per_gpu": B / (ms * 1e-3),
                "finite": finite, "shape": f"{nu_loc} local users, {ni_tot} items sharded over {world} GPUs, d={d}, {B} triples/step/rank",
                "nvlink_bytes_per_triple_each_way": 2 * (256 + 4) * (world - 1) / world})
    # the same kernel with the whole table local (world=1 view of the same shape) for comparison: single-table kernel
    Vloc = torch.randn(min(ni_tot, 4_000_000), d, device=dev, generator=gu) * 0.1; bloc = torch.zeros(Vloc.shape[0], device=dev)
    idx_loc = indices.clamp(max=Vloc.shape[0] - 1)

    def step_local():
        ops.bpr_step_sampled_f32(U, Vloc, bloc, d, nu_loc, Vloc.shape[0], indptr, idx_loc, B, 42 + rank, ctr[0] * B, *HP, loss=loss)
        ctr[0] += 1
    res["single_table_same_shape_ms"] = timed(step_local, 10, warm=3)
    items.close(); bias.close()
    return res


@section("reconcile")
def _reconcile():
    res = {}
    n_items, d = 100_000, 64
    numel = n_items * d + n_items
    buf = PeerBuffer(numel, device=dev)
    g = torch.Generator(device=dev); g.manual_seed(7)
    base = torch.randn(numel, device=dev, generator=g) * 0.1
    buf.local.copy_(base)
    sync = PeerTableSync(buf)
    sync.reset()
    gr = torch.Generator(device=dev); gr.manual_seed(50 + rank)
    total = torch.zeros_like(base)
    for rnd in range(3):
        st = torch.randn(numel, device=dev, generator=gr) * 0.01 * (torch.rand(numel, device=dev, generator=gr) < 0.3)
        buf.local.add_(st)
        s = st.clone()
        if world > 1:
            dist.all_reduce(s)
        total += s / world
        sync.flush()
    err = (buf.local - (base + total)).abs().max().item()
    res["max_err_vs_mean_of_steps"] = err
    res["ok"] = all_ok(err < 1e-5)
    # kernel time with every row touched by every rank (worst case: every element corrected on every copy)
    def touch_and_sync():
        buf.local.add_(1e-3)
        sync.sync()
    res["touch_plus_reconcile_ms"] = timed(touch_and_sync, 10)
    res["touch_only_ms"] = timed(lambda: buf.local.add_(1e-3), 10)
    res["reconcile_ms_dense"] = res["touch_plus_reconcile_ms"] - res["touch_only_ms"]
    res["nvlink_bytes_per_reconcile_each_way"] = numel * 4 * (world - 1) / world
    # C2 training with the item table replicated in the peer buffer
    nu, per_user, B = 1_000_000, 100, 1 << 22
    V = buf.local[:n_items * d].view(n_items, d); b = buf.local[n_items * d:]
    buf.barrier(); buf.local.copy_(base); b.zero_(); sync.reset()
    U = torch.randn(nu, d, device=dev, generator=gr) * 0.1
    cand = (torch.rand(nu, per_user, device=dev, generator=gr) ** 2 * n_items).to(torch.int32).clamp_(max=n_items - 1)
    cand, _ = torch.sort(cand, dim=1)
    keep = torch.ones_like(cand, dtype=torch.bool); keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    indptr = torch.zeros(nu + 1, dtype=torch.int64, device=dev); indptr[1:] = torch.cumsum(keep.sum(1), 0)
    indices = cand[keep].contiguous()
    del cand, keep
    loss = torch.zeros(1, dtype=torch.float64, device=dev); ctr = [0]

    def train_only():
        ops.bpr_step_sampled_f32(U, V, b, d, nu, n_items, indptr, indices, B, 42 + rank, ctr[0] * B, *HP, loss=loss)
        ctr[0] += 1

    def train_sync():
        train_only(); sync.sync()
    res["c2_step_ms"] = timed(train_only, 10, warm=3)
    res["c2_step_plus_reconcile_ms"] = timed(train_sync, 10, warm=3)
    sync.flush()
    res["c2_triples_per_s_all_ranks"] = B * world / (res["c2_step_plus_reconcile_ms"] * 1e-3)
    res["finite"] = all_ok(bool(torch.isfinite(buf.local).all().item()))
    mx = buf.local.clone()
    if world > 1:
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
    res["copies_agree_after_flush_max_diff"] = (mx - buf.local).abs().max().item()
    buf.close()
    return res


@section("neumf")
def _neumf():
    from elliot_b200.recommender.neumf import NeuralMatrixFactorizationModel
    from elliot_b200.recommender.neumf_sharded import ShardedNeuMFModel
    res = {}
    NU, NI, F, B, STEPS = 40000, 20000, 64, 8192, 4
    sh = ShardedNeuMFModel(NU, NI, F, 1e-3, 42, dev)
    g = torch.Generator(device=dev); g.manual_seed(100 + rank)
    ulo, uhi = shard_range(NU, rank, world)
    batches = []
    for s in range(STEPS):
        u = torch.randint(0, uhi - ulo, (B,), device=dev, generator=g, dtype=torch.int32)
        it = torch.randint(0, NI, (B,), device=dev, generator=g, dtype=torch.int32)
        y = (torch.rand(B, device=dev, generator=g) < 0.3).float()
        batches.append((u, it, y))
        sh.train_step((u, it, y))
    barrier()
    allb = []
    for (u, it, y) in batches:
        parts = [[torch.empty_like(t) for _ in range(world)] for t in (u, it, y)]
        for p, t in zip(parts, ((u + ulo).contiguous(), it, y)):
            if world > 1:
                dist.all_gather(p, t)
            else:
                p[0].copy_(t)
        allb.append(tuple(torch.cat(p) for p in parts))
    ref = NeuralMatrixFactorizationModel(NU, NI, F, 1e-3, 42, dev)
    for b in allb:
        ref.train_step(b)
    rel = lambda a, b: float((a - b).norm() / b.norm().clamp_min(1e-12))
    ilo, ihi = sh.items.lo, sh.items.hi
    diffs = {"U_mf": rel(sh.P["U_mf"], ref.P["U_mf"][ulo:uhi]), "U_mlp": rel(sh.P["U_mlp"], ref.P["U_mlp"][ulo:uhi]),
             "I_mf": rel(sh.P["I"][:ihi - ilo, :F], ref.P["I_mf"][ilo:ihi]), "I_mlp": rel(sh.P["I"][:ihi - ilo, F:], ref.P["I_mlp"][ilo:ihi]),
             **{k: rel(sh.P[k], ref.P[k]) for k in ("W1", "W2", "W3", "wp")}}
    # scoring over the sharded item table vs the single-GPU model (whose weights differ by <= the diffs above)
    indptr = torch.zeros(NU + 1, dtype=torch.int64, device=dev); indices = torch.zeros(1, dtype=torch.int32, device=dev)
    i_s, v_s = sh.get_recs_topk(0, 32, 10, indptr[ulo:].contiguous(), indices)
    i_r, v_r = ref.get_recs_topk(ulo, ulo + 32, 10, indptr, indices)
    overlap = float(sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(i_s, i_r)) / (32 * 10))
    res.update({"rel_diff_vs_single_gpu": diffs, "topk_overlap_vs_single_gpu": overlap, "topk_max_prob_diff": float((v_s - v_r).abs().max()),
                "ok": all_ok(max(diffs.values()) < 1e-3 and overlap > 0.9)})
    sh.close(); del ref, sh
    torch.cuda.empty_cache()
    # C4 shape: users sharded, items sharded, d=64, m=4 negatives per positive; batch per rank per step
    NU, NI, F, B = args.neumf_users, args.neumf_items, 64, args.neumf_batch
    sh = ShardedNeuMFModel(NU, NI, F, 1e-3, 42, dev, full_init=False)
    nl = sh.uhi - sh.ulo
    u = torch.randint(0, nl, (B,), device=dev, generator=g, dtype=torch.int32)
    it = torch.randint(0, NI, (B,), device=dev, generator=g, dtype=torch.int32)
    y = (torch.arange(B, device=dev) % 5 == 0).float()                                  # 1 positive : 4 negatives
    ms = timed(lambda: sh.train_step((u, it, y)), 5, warm=2)
    adam_elems = sum(v.numel() for v in sh.P.values())
    res.update({"c4_step_ms": ms, "c4_samples_per_s_all_ranks": B * world / (ms * 1e-3), "c4_batch_per_rank": B,
                "c4_shape": f"{NU} users x {NI} items over {world} GPUs, d={F}, dense Keras Adam over {adam_elems} local elements/step",
                "c4_nvlink_bytes_per_sample_each_way": 2 * F * 4 * (world - 1) / world,
                "c4_loss_finite": bool(torch.isfinite(sh._loss).all().item())})
    # where the step goes: dense Adam alone
    def adam_only():
        for k in sh.P:
            ops.adam_dense_f32(sh.P[k], sh.M[k], sh.V[k], sh.G[k], sh.lr, sh.step + 1)
    res["c4_adam_only_ms"] = timed(adam_only, 3, warm=1)
    sh.close()
    return res


barrier()
if rank == 0:
    os.makedirs("gpurun_out", exist_ok=True)
    json.dump(out, open(f"gpurun_out/peer_check_n{world}.json", "w"), indent=1)
    print(json.dumps(out))
if world > 1:
    dist.destroy_process_group()
