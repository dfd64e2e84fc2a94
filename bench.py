#!/usr/bin/env python
"""bench.py — BPR triples/s on the C2 workload (BASELINE.json configs[1]).

One "step" = one pass of the hot path over one batch of synthetic input:
    sample B (u,i,j) triples -> gather 3 rows -> score -> log-sigmoid grad -> scatter-add
fused in ONE kernel launch (elliot_b200/csrc/bpr_train.cu, eb_bpr_step_sampled_f32).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl b200|reference] [--dump-outputs DIR]

--dump-outputs DIR: after the K timed steps, the tables the timed path leaves behind (what a caller of
eb_bpr_step_sampled_f32 receives: the updated item factors and biases, a fixed seeded sample of user rows,
the accumulated loss) are written as DIR/<name>.npy (float32 / float64), before anything else touches them.
Inputs are seeded, so two builds run with the same arguments can be compared output for output: with
--dump-outputs the timed steps run in deterministic rounds (--schedule auto), where only the fp32 order of one
round's atomic adds to a shared row varies between runs.  Free-running Hogwild, the default otherwise, reads rows
while other triples update them, so its tables differ from run to run by more than rounding.

N>1 (torchrun, one rank per GPU): every rank owns its own shard of 1M users (weak scaling;
user rows never leave their GPU), the 100K-item table is replicated and kept consistent with
one NCCL all-reduce of the per-step item deltas (the path's only exchange step).
Rank 0 prints ONE JSON result line.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# ---- workload: BASELINE.json configs[1] "BPRMF d=64 synthetic 1M x 100K interactions", one GPU
N_USERS, N_ITEMS, D = 1_000_000, 100_000, 64
PER_USER = 100
BATCH = 1 << 22                      # triples per step
HP = (0.05, 0.0025, 0.0, 0.0025, 0.00025)   # BPRMF.py:63-71 defaults
ALG_BYTES_SAMPLED = 3 * D * 4 * 2 + 16      # 1552 B/triple (SURVEY.md §8d): rows r+w, biases r+w
ALG_BYTES_MATERIALISED = ALG_BYTES_SAMPLED + 12


def load_peaks():
    """H100 SXM data-sheet peaks (700 W part): HBM3 3.35 TB/s, dense bf16 989 TFLOP/s.  Not reached figures: the
    roofline fractions below are shares of these."""
    return 3350.0, 989.0, "datasheet H100 SXM"


DUMP_USER_ROWS = 65536                      # seeded sample of the 1M user rows written by --dump-outputs


def dump_outputs(out_dir, U, V, b, loss, seed=1234):
    """The timed path's outputs after its last step, as float32 / float64 .npy files (26 MB of V + b, 16 MB of sampled U)."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    g = torch.Generator(device="cpu"); g.manual_seed(seed)
    rows = torch.randperm(U.shape[0], generator=g)[:DUMP_USER_ROWS].sort().values
    np.save(os.path.join(out_dir, "item_factors.npy"), V.float().cpu().numpy())
    np.save(os.path.join(out_dir, "item_bias.npy"), b.float().cpu().numpy())
    np.save(os.path.join(out_dir, "user_factors_sample.npy"), U[rows.to(U.device)].float().cpu().numpy())
    np.save(os.path.join(out_dir, "user_factors_sample_rows.npy"), rows.numpy().astype(np.float64))
    np.save(os.path.join(out_dir, "loss_sum.npy"), loss.double().cpu().numpy())


class ClockSampler:
    """Samples SM clock and throttle reasons DURING the timed region with NVML from a thread (2 ms period);
    nvidia-smi -lms is too coarse for a 20 ms region."""
    REASONS = {0x8: "hw_slowdown", 0x40: "hw_thermal_slowdown", 0x20: "sw_thermal_slowdown", 0x4: "sw_power_cap"}

    def __init__(self, gpu_index):
        self.idx, self.sm, self.reasons, self.stop_flag, self.th, self.mx, self.err = gpu_index, [], set(), False, None, None, None
        self.period = float(os.environ.get("EB_CLOCK_PERIOD_MS", "2")) * 1e-3

    def _loop(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(vis.split(",")[self.idx]) if vis and vis.split(",")[self.idx].isdigit() else self.idx
            h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self.mx = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
            while not self.stop_flag:
                self.sm.append(float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)))
                try:
                    r = pynvml.nvmlDeviceGetCurrentClocksEventReasons(h)
                except Exception:
                    r = pynvml.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                for bit, name in self.REASONS.items():
                    if r & bit:
                        self.reasons.add(name)
                time.sleep(self.period)
        except Exception as e:                      # noqa: BLE001
            self.err = repr(e)

    def start(self):
        self.th = threading.Thread(target=self._loop, daemon=True)
        self.th.start()
        t0 = time.time()
        while not self.sm and self.err is None and time.time() - t0 < 2.0:
            time.sleep(0.005)                       # first sample taken before the timed region starts

    def mark(self):
        """Call right before the timed region: samples before this index are ignored."""
        self.first = len(self.sm)

    def stop(self):
        self.stop_flag = True
        if self.th:
            self.th.join(timeout=2)
        sm = self.sm[getattr(self, "first", 0):]
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": self.mx, "reasons": ["no samples" + (f": {self.err}" if self.err else "")]}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": self.mx, "reasons": sorted(self.reasons), "samples": len(sm)}


def synth_csr(torch, dev, seed):
    """~PER_USER train items per user, squared-uniform popularity skew, rows sorted + deduped."""
    g = torch.Generator(device=dev); g.manual_seed(seed)
    cand = (torch.rand(N_USERS, PER_USER, device=dev, generator=g) ** 2 * N_ITEMS).to(torch.int32)
    cand.clamp_(max=N_ITEMS - 1)
    cand, _ = torch.sort(cand, dim=1)
    keep = torch.ones_like(cand, dtype=torch.bool)
    keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    lens = keep.sum(1)
    indptr = torch.zeros(N_USERS + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(lens, 0)
    return indptr, cand[keep].contiguous()


def cpu_baseline(indptr_h, indices_h, budget_s=12.0):
    """Oracle C port (kind "port") of sampler + sequential update on the host, one core
    (the algorithm is strictly sequential, BPRMF.py:80), on a bounded sample of the same
    workload; plus the interpreter-bound NumPy port whose cost profile matches the reference."""
    import numpy as np
    import oracle
    from oracle import bprmf_numpy as bn
    rs = np.random.RandomState(0)
    U = rs.normal(0, 0.1, (N_USERS, D)); V = rs.normal(0, 0.1, (N_ITEMS, D)); b = np.zeros(N_ITEMS)
    rng = oracle.Rng(42)
    n = 1_000_000
    t0 = time.perf_counter()
    u, i, j, _ = oracle.sampler_step(rng, N_USERS, N_ITEMS, indptr_h, indices_h, n)
    oracle.bpr_update_seq(U, V, b, u, i, j, *HP)
    dt = time.perf_counter() - t0
    total, total_t = n, dt
    more = int(min(40_000_000, max(0, (budget_s - dt) / dt * n)))
    if more > 0:
        t0 = time.perf_counter()
        u, i, j, _ = oracle.sampler_step(rng, N_USERS, N_ITEMS, indptr_h, indices_h, more)
        oracle.bpr_update_seq(U, V, b, u, i, j, *HP)
        total_t += time.perf_counter() - t0; total += more
    # interpreter-bound port on a small sample (reference-like cost profile)
    nn = 20000
    rows = [indices_h[indptr_h[x]:indptr_h[x + 1]].tolist() for x in range(2000)]
    m = bn.SequentialBPR(2000, N_ITEMS, D, *HP, seed=42)
    np.random.seed(42)
    t0 = time.perf_counter()
    for uu, ii, jj in bn.triple_stream(rows, N_ITEMS, nn):
        m.sgd(uu, ii, jj)
    np_rate = nn / (time.perf_counter() - t0)
    return {"value": total / total_t, "unit": "triples/s", "cores": 1, "kind": "port",
            "sample": f"{total} triples, C port of custom_sampler.py:24-46 + BPRMF_model.py:87-117 (fp64, sequential) "
                      f"on the C2 tables; host has {os.cpu_count()} cores, algorithm is single-threaded by construction",
            "numpy_port_value": np_rate,
            "numpy_port_sample": f"{nn} triples, interpreter-bound NumPy port (reference-like cost profile), "
                                 f"2000-user slice of the same CSR"}


def run_reference(args):
    """--impl reference: the reference's own CPU implementation of the path.  The reference is
    pure Python and is not installed next to this package, so this is the oracle port
    (kind "port"): the interpreter-bound NumPy restatement with the reference's per-triple cost
    profile is the headline value; the (much faster) C port is reported beside it."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import numpy as np
    import oracle
    from oracle import bprmf_numpy as bn
    rs = np.random.default_rng(0)
    n_users_s = 20000                                  # bounded slice of the 1M-user workload
    lens = np.full(n_users_s, PER_USER)
    indptr = np.zeros(n_users_s + 1, np.int64); indptr[1:] = np.cumsum(lens)
    cand = (rs.random((n_users_s, PER_USER)) ** 2 * N_ITEMS).astype(np.int32)
    rows = []
    flat = []
    for r in cand:
        ur = sorted(set(r.tolist())); rows.append(ur); flat.extend(ur)
    indptr = np.zeros(n_users_s + 1, np.int64); indptr[1:] = np.cumsum([len(r) for r in rows])
    indices = np.array(flat, np.int32)
    per_step = 20000
    m = bn.SequentialBPR(n_users_s, N_ITEMS, D, *HP, seed=42)
    np.random.seed(42)

    def step():
        for uu, ii, jj in bn.triple_stream(rows, N_ITEMS, per_step):
            m.sgd(uu, ii, jj)
    for _ in range(min(args.warmup, 1)):
        step()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step()
    dt = time.perf_counter() - t0
    rate = per_step * args.steps / dt
    # C port beside it
    U = np.random.RandomState(0).normal(0, 0.1, (n_users_s, D)); V = np.random.RandomState(1).normal(0, 0.1, (N_ITEMS, D))
    b = np.zeros(N_ITEMS); rng = oracle.Rng(42)
    t0 = time.perf_counter()
    u, i, j, _ = oracle.sampler_step(rng, n_users_s, N_ITEMS, indptr, indices, 2_000_000)
    oracle.bpr_update_seq(U, V, b, u, i, j, *HP)
    c_rate = 2_000_000 / (time.perf_counter() - t0)
    out = {"impl": "reference", "metric": "bpr_triples_per_sec", "value": rate, "unit": "triples/s",
           "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": dt / args.steps * 1e3,
           "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
           "config": {"workload": "C2: BPRMF d=64, 1M users x 100K items, ~100 train items/user "
                                  "(bounded sample: 20000-user slice, 20000 triples/step)"},
           "cpu_baseline": {"value": rate, "unit": "triples/s", "cores": 1, "kind": "port",
                            "sample": f"{per_step} triples/step x {args.steps} steps, interpreter-bound NumPy port of "
                                      "custom_sampler.py:24-46 + BPRMF_model.py:87-117 (the reference is pure Python, "
                                      "single-threaded by construction)", "c_port_value": c_rate,
                            "host_cores": os.cpu_count()},
           "e2e": {"value": rate, "unit": "triples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(out))


def bind_near_gpu(local):
    """Pin this process (and so the pages of every pinned buffer it allocates from now on: first touch) to the CPU cores of
    the GPU's NUMA node — host<->device copies then do not cross the socket interconnect.  Best effort."""
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        phys = int(vis.split(",")[local]) if vis and vis.split(",")[local].isdigit() else local
        bus = pynvml.nvmlDeviceGetPciInfo(pynvml.nvmlDeviceGetHandleByIndex(phys)).busId
        bus = (bus.decode() if isinstance(bus, bytes) else bus).lower()
        if len(bus.split(":")[0]) == 8:
            bus = bus[4:]
        node = int(open(f"/sys/bus/pci/devices/{bus}/numa_node").read())
        if node < 0:
            return "numa node unknown"
        cpus = []
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.extend(range(int(a), int(b or a) + 1))
        os.sched_setaffinity(0, set(cpus) & os.sched_getaffinity(0) or os.sched_getaffinity(0))
        return f"node {node}"
    except Exception as e:                                          # noqa: BLE001
        return f"not bound ({type(e).__name__})"


def synth_csr_n(torch, dev, seed, n_users, n_items, per_user):
    g = torch.Generator(device=dev); g.manual_seed(seed)
    cand = (torch.rand(n_users, per_user, device=dev, generator=g) ** 2 * n_items).to(torch.int32)
    cand.clamp_(max=n_items - 1)
    cand, _ = torch.sort(cand, dim=1)
    keep = torch.ones_like(cand, dtype=torch.bool)
    keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    indptr = torch.zeros(n_users + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(keep.sum(1), 0)
    return indptr, cand[keep].contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--sync", default="auto", choices=["auto", "peer", "overlap", "simple"],
                    help="N>1, how the replicated item table is reconciled: ONE peer-memory kernel per rank and step (peer), "
                         "NCCL all-reduce in line (simple) or one step late beside the next step (overlap); auto = fastest in a "
                         "short untimed trial")
    ap.add_argument("--reserve-sms", type=int, default=12, help="N>1, overlap: SMs left to the NCCL kernel")
    ap.add_argument("--schedule", default="auto", choices=["auto", "hogwild", "rounds"],
                    help="BPR step schedule: free-running Hogwild, or deterministic rounds (reads, grid barrier, atomic adds, grid "
                         "barrier); auto = rounds with --dump-outputs, Hogwild otherwise")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write the path's outputs (updated tables, loss) as DIR/<name>.npy")
    ap.add_argument("--blocks", default="all", help="comma list of extra blocks (scoring,c5,exact,large,vae,neumf,mf2020,schedules,sharded) or all/none")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args)

    os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")   # stdout carries exactly one JSON line
    import torch
    import torch.distributed as dist
    from elliot_b200 import ops

    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    numa = bind_near_gpu(local)
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    W = max(args.warmup, 3); K = args.steps
    want = lambda b: args.blocks == "all" or b in args.blocks.split(",")
    t_start = time.time()

    def allmax(x):
        t = torch.tensor([x], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return t.item()

    def timed(fn, reps, warm=2):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        z.record(); torch.cuda.synchronize()
        return allmax(a.elapsed_time(z) / reps)

    # ---- resident state (inputs are in HBM before the timed region starts)
    g = torch.Generator(device=dev); g.manual_seed(1000 + rank)
    U = torch.randn(N_USERS, D, device=dev, generator=g) * 0.1        # this rank's user shard
    n_flat = N_ITEMS * D + N_ITEMS                                      # item factors + item biases in ONE buffer
    peer_buf, peer_note = None, None
    if world > 1 and args.sync in ("auto", "peer"):
        try:
            from elliot_b200.peer import PeerBuffer
            peer_buf = PeerBuffer(n_flat, device=dev)                   # every rank's copy mapped into every other rank
            peer_note = peer_buf.kind
        except Exception as e:                                          # noqa: BLE001
            peer_note = f"unavailable: {e}"[:160]
            sys.stderr.write(f"[rank {rank}] peer memory {peer_note}\n")
    items_flat = peer_buf.local if peer_buf is not None else torch.empty(n_flat, device=dev)
    V = items_flat[:N_ITEMS * D].view(N_ITEMS, D)                      # replicated
    gv = torch.Generator(device=dev); gv.manual_seed(7)
    V.copy_(torch.randn(N_ITEMS, D, device=dev, generator=gv) * 0.1)
    b = items_flat[N_ITEMS * D:]; b.zero_()
    indptr, indices = synth_csr(torch, dev, seed=100 + rank)
    # per-user membership signatures pay off on large catalogues, not on C2's L2-resident 100 K items, so the C2 step runs
    # without them
    filt = None
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    seed = 42 + rank
    counter = [0]
    rounds = args.schedule == "rounds" or (args.schedule == "auto" and args.dump_outputs is not None)
    sm_total = ops.device_info()[0]

    # ---- N>1: schedules for the one exchange step (reconciliation of the replicated item table; deltas averaged)
    modes, partition_note = {}, None
    if world > 1:
        from elliot_b200.parallel import OverlappedTableSync, PeerTableSync, ReplicatedTableSync
        if peer_buf is not None:
            modes["peer"] = {"sync": PeerTableSync(peer_buf, n_flat), "stream": torch.cuda.current_stream(), "reserve": 0}
        if args.sync in ("simple", "auto") or not modes:
            modes["simple"] = {"sync": ReplicatedTableSync([V, b], reduce="mean", flat=items_flat),
                               "stream": torch.cuda.current_stream(), "reserve": 0}
        if args.sync in ("overlap", "auto"):
            try:
                ps, granted = ops.partition_streams(dev, args.reserve_sms, 3)
                modes["overlap"] = {"sync": OverlappedTableSync([V, b], reduce="mean", flat=items_flat),
                                    "stream": ps[0], "reserve": sm_total - granted, "e2e_streams": ps[1:]}
                partition_note = f"{granted}+{sm_total - granted} SMs"
            except Exception as e:                                      # noqa: BLE001
                partition_note = f"no SM partition ({type(e).__name__})"
    else:
        modes["single"] = {"sync": None, "stream": torch.cuda.current_stream(), "reserve": 0}

    def step(reserve):
        ops.bpr_step_sampled_f32(U, V, b, D, N_USERS, N_ITEMS, indptr, indices, BATCH, seed, counter[0] * BATCH, *HP,
                                 loss=loss, reserve_sms=reserve, filter=filt, deterministic=rounds)
        counter[0] += 1

    def run_steps(m, n, per_step_events=None):
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(m["stream"]):
            a.record()
            for k in range(n):
                if per_step_events:
                    per_step_events[0][k].record()
                step(m["reserve"])
                if per_step_events:
                    per_step_events[1][k].record()
                if m["sync"] is not None:
                    m["sync"].sync()
            if isinstance(m["sync"], OverlappedTableSync if world > 1 else ()):
                m["sync"].flush()
            z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z)

    chosen = next(iter(modes))
    tune = {}
    if len(modes) > 1:
        for name, m in modes.items():
            m["sync"].reset()
            run_steps(m, 2)
            dist.barrier()
            tune[name] = round(allmax(run_steps(m, 4)) / 4, 4)
            if name == "peer":
                m["sync"].flush()                                       # copies equal again before the next schedule starts
        chosen = args.sync if args.sync in tune else min(tune, key=tune.get)
    mode = modes[chosen]
    if mode["sync"] is not None:
        mode["sync"].reset()
    reserve = mode["reserve"]
    run_steps(mode, W)
    clocks = ClockSampler(local); clocks.start()
    ks = [torch.cuda.Event(enable_timing=True) for _ in range(K)]
    ke = [torch.cuda.Event(enable_timing=True) for _ in range(K)]
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()                                                  # ranks line up right before the timed region
    clocks.mark()
    ms_total = run_steps(mode, K, (ks, ke))
    if world > 1:
        dist.barrier()
    kern_ms = sum(s.elapsed_time(e) for s, e in zip(ks, ke)) / K
    clk = clocks.stop()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, U, V, b, loss)
    ms_total = allmax(ms_total)
    value = BATCH * K * world / (ms_total * 1e-3)

    # ---- end to end through the C ABI with HOST triples: per step ONE H2D copy of packed triples (8 B each, pinned,
    # NUMA-local) + kernel + D2H loss; three steps in flight on three streams
    DEPTH, pool = 3, 4
    host = []
    for q in range(pool):
        tu, ti, tj = ops.bpr_sample_philox(N_USERS, N_ITEMS, indptr, indices, BATCH, seed + 99, q * BATCH, filter=filt)
        host.append(ops.pack_triples(tu, ti, tj, N_USERS, N_ITEMS).cpu().pin_memory())
        del tu, ti, tj
    streams = mode.get("e2e_streams") or []
    streams = list(streams) + [torch.cuda.Stream(device=dev) for _ in range(DEPTH - len(streams))]
    e2e_sync = None
    if world > 1:
        e2e_sync = mode["sync"] if chosen in ("overlap", "peer") else OverlappedTableSync([V, b], reduce="mean", flat=items_flat)
        e2e_sync.reset()
    staging = [torch.empty(BATCH, dtype=torch.int64, device=dev) for _ in range(DEPTH)]
    loss_dev2 = [torch.zeros(1, dtype=torch.float64, device=dev) for _ in range(DEPTH)]
    loss_host = [torch.zeros(1, dtype=torch.float64).pin_memory() for _ in range(DEPTH)]

    def e2e_steps(n):
        total = 0.0
        for k in range(n):
            sl = k % DEPTH
            streams[sl].synchronize()                                   # buffers of step k-DEPTH are free, its loss is on the host
            if k >= DEPTH:
                total += loss_host[sl].item()
            with torch.cuda.stream(streams[sl]):
                ops.bpr_step_host_packed_f32(U, V, b, D, host[k % pool], N_USERS, N_ITEMS, *HP, staging[sl], loss_dev2[sl],
                                             loss_host[sl], sync=False, reserve_sms=reserve)
                if e2e_sync is not None:
                    e2e_sync.sync()
        for st_ in streams:
            st_.synchronize()
        return total
    torch.cuda.synchronize()
    e2e_steps(DEPTH + 1)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    t_e0 = time.perf_counter()
    e2e_steps(K)
    torch.cuda.synchronize()
    e2e_ms = allmax((time.perf_counter() - t_e0) * 1e3)
    e2e_value = BATCH * K * world / (e2e_ms * 1e-3)
    if e2e_sync is not None:
        e2e_sync.flush()
    finite = bool(torch.isfinite(U).all().item() and torch.isfinite(V).all().item())
    if not finite:
        raise RuntimeError("tables went non-finite during the benchmark: the numbers would be meaningless")
    del host, staging

    hbm, tflops, which = load_peaks()
    extra = {}

    def block(name, fn):
        if not want(name):
            return
        torch.cuda.empty_cache()                                        # peer buffers are plain cudaMalloc blocks: give cached memory back
        try:
            extra[name] = fn()
        except Exception as e:                                          # noqa: BLE001
            extra[name] = {"error": f"{type(e).__name__}: {e}"[:300]}
            sys.stderr.write(f"[rank {rank}] bench block {name} failed: {e!r}\n")
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    # ---- second half of the path: full-catalogue scoring + mask + top-10 on the tensor cores (+ device metrics)
    S_USERS = 132 * 128 * 2                                             # two 128-user blocks per H100 SM

    def blk_scoring():
        _, _, sst = ops.score_topk_tc(U, V, b, D, 10, indptr, indices, user_begin=0, n_sel=S_USERS)
        ms = timed(lambda: ops.score_topk_tc(U, V, b, D, 10, indptr, indices, user_begin=0, n_sel=S_USERS, stats=False), 3)
        TE = 20
        ge = torch.Generator(device=dev); ge.manual_seed(77 + rank)
        te_items, _ = torch.sort(torch.randint(0, N_ITEMS, (S_USERS, TE), device=dev, generator=ge, dtype=torch.int32), dim=1)
        te_indptr = torch.arange(0, (S_USERS + 1) * TE, TE, dtype=torch.int64, device=dev)
        disc = torch.tensor([math.log(2) / math.log(r + 2) for r in range(10)], dtype=torch.float64, device=dev)
        idcg = torch.full((S_USERS,), float(disc.sum().item()), dtype=torch.float64, device=dev)
        ev_args = (te_indptr, te_items.reshape(-1).contiguous(), torch.ones(S_USERS * TE, dtype=torch.float64, device=dev), idcg, disc)
        res = {}

        def both():
            si, _, _ = ops.score_topk_tc(U, V, b, D, 10, indptr, indices, user_begin=0, n_sel=S_USERS, stats=False)
            res["ev"], _ = ops.eval_topk(si, 10, *ev_args)
        ms_ev = timed(both, 3)
        ev = res["ev"].cpu().tolist()
        fl = 2.0 * D * N_ITEMS * S_USERS
        return {"metric": "scored_users_per_sec", "value": S_USERS * world / (ms * 1e-3), "unit": "users/s", "ms": ms,
                "config": {"workload": f"{S_USERS} users/GPU x {N_ITEMS} items, d={D}, k=10, bias + train mask, wgmma bf16 + exact fp32 re-rank",
                           "rechecked_users": sst["rechecked"], "padded_k": sst["kp"]},
                "with_device_metrics": {"value": S_USERS * world / (ms_ev * 1e-3), "unit": "users/s", "ndcg_at_10_rank0": ev[1] / max(ev[0], 1.0)},
                "roofline": {"bound": "tensor", "achieved": fl / (ms * 1e-3) / 1e12, "executed": fl * sst["kp"] / D / (ms * 1e-3) / 1e12,
                             "peak": tflops, "unit": "TFLOP/s", "frac": fl / (ms * 1e-3) / 1e12 / tflops}}
    block("scoring", blk_scoring)

    def blk_c5():
        C5_ITEMS, C5_D = 2_000_000, 128
        g5 = torch.Generator(device=dev); g5.manual_seed(55 + rank)
        U5 = torch.randn(S_USERS, C5_D, device=dev, generator=g5) * 0.1
        V5 = torch.randn(C5_ITEMS, C5_D, device=dev, generator=g5) * 0.1
        b5 = torch.randn(C5_ITEMS, device=dev, generator=g5) * 0.05
        ip5, ix5 = synth_csr_n(torch, dev, 56 + rank, S_USERS, C5_ITEMS, PER_USER)
        _, _, st5 = ops.score_topk_tc(U5, V5, b5, C5_D, 10, ip5, ix5)
        ms = timed(lambda: ops.score_topk_tc(U5, V5, b5, C5_D, 10, ip5, ix5, stats=False), 3, warm=1)
        fl = 2.0 * C5_D * C5_ITEMS * S_USERS
        return {"metric": "scored_users_per_sec", "value": S_USERS * world / (ms * 1e-3), "unit": "users/s", "ms": ms,
                "config": {"workload": f"per-GPU slice of configs[4]: {S_USERS} users/GPU x {C5_ITEMS} items, d={C5_D}, k=10, bias + mask, "
                                       "V replicated, users sharded", "rechecked_users": st5["rechecked"], "padded_k": st5["kp"]},
                "roofline": {"bound": "tensor", "achieved": fl / (ms * 1e-3) / 1e12, "executed": fl * st5["kp"] / C5_D / (ms * 1e-3) / 1e12,
                             "peak": tflops, "unit": "TFLOP/s", "frac": fl / (ms * 1e-3) / 1e12 / tflops}}
    block("c5", blk_c5)

    # ---- exact (parity) mode at the C1 shape: device MT19937 replay + sequentially consistent fp64 update
    def blk_exact():
        import numpy as np
        from elliot_b200 import synth_c1
        uu, ii, _ = synth_c1.rows()
        order = np.lexsort((ii, uu)); uu, ii = uu[order] - 1, ii[order] - 1
        nu1, ni1 = synth_c1.N_USERS, synth_c1.N_ITEMS
        ip = np.zeros(nu1 + 1, np.int64); np.cumsum(np.bincount(uu, minlength=nu1), out=ip[1:])
        srt = ii.astype(np.int32)
        setord = np.concatenate([np.array(list(set(dict.fromkeys(srt[ip[x]:ip[x + 1]].tolist()))), np.int32) for x in range(nu1)])
        ipd, sod, srd = (torch.from_numpy(a).to(dev) for a in (ip, setord, srt))
        sampler = ops.MtSampler(nu1, ni1, ipd, sod, srd, seed=42)
        rs = np.random.RandomState(42)
        U1 = torch.from_numpy(rs.normal(0, 0.1, (nu1, D))).to(dev); V1 = torch.from_numpy(rs.normal(0, 0.1, (ni1, D))).to(dev)
        b1 = torch.zeros(ni1, dtype=torch.float64, device=dev)
        T = int(ip[-1])

        def epoch():
            tu, ti, tj = sampler.step(T)
            ops.bpr_exact_f64(U1, V1, b1, D, tu, ti, tj, *HP)
        ms = timed(epoch, 3, warm=1)
        return {"metric": "bpr_triples_per_sec_exact_mode", "value": T / (ms * 1e-3), "unit": "triples/s", "ms_per_epoch": ms,
                "config": {"workload": f"C1 shape {nu1} x {ni1}, {T} triples/epoch, d={D}: eb_mt_sampler_step (bit-exact MT19937 replay) + "
                                       "eb_bpr_exact_f64 (fp64, reference order); the mode whose nDCG equals the reference's"}}
    if world == 1:
        block("exact", blk_exact)

    # ---- the HBM-bound regime: item table far larger than L2 (1M users x 2M items, V = 512 MB)
    def blk_large():
        LI = 2_000_000
        gl = torch.Generator(device=dev); gl.manual_seed(5 + rank)
        VL = torch.randn(LI, D, device=dev, generator=gl) * 0.1; bL = torch.zeros(LI, device=dev)
        ipL, ixL = synth_csr_n(torch, dev, 300 + rank, N_USERS, LI, PER_USER)
        fL = ops.bloom_build(ipL, ixL, N_USERS)
        UL = U.clone(); c = [0]

        def st():
            ops.bpr_step_sampled_f32(UL, VL, bL, D, N_USERS, LI, ipL, ixL, BATCH, seed, c[0] * BATCH, *HP, filter=fL)
            c[0] += 1
        ms = timed(st, 10, warm=3)
        ach = ALG_BYTES_SAMPLED * BATCH / (ms * 1e-3) / 1e9
        tr = traffic_of("bpr_hogwild_large")
        return {"metric": "bpr_triples_per_sec", "value": BATCH / (ms * 1e-3), "unit": "triples/s", "ms": ms,
                "config": {"workload": f"{N_USERS} users x {LI} items (V = {LI * D * 4 >> 20} MB >> 50 MB L2), d={D}, {BATCH} triples/step"},
                "roofline": {"bound": "hbm", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm, "traffic": tr,
                             "frac_dram_measured": None if tr is None else tr / (ms * 1e-3) / 1e9 / hbm},
                "finite": bool(torch.isfinite(VL).all().item())}
    if world == 1:
        block("large", blk_large)

    # ---- BASELINE configs[2]: MultiVAE [200,600] at the ML-20M shape (data parallel at N>1: weights replicated, batch split)
    def blk_vae():
        from elliot_b200.recommender.multi_vae import VariationalAutoEncoder
        nu3, ni3, B3 = 138_493, 26_744, 512
        ip3, ix3 = synth_csr_n(torch, dev, 900, nu3, ni3, 144)
        m = VariationalAutoEncoder(ni3, 600, 200, 1e-3, 0.5, 0.01, 42, ip3, ix3, dev)
        if world > 1:
            m.enable_data_parallel()
        g3 = torch.Generator(device=dev); g3.manual_seed(3 + rank)
        rows = torch.randperm(nu3, device=dev, generator=g3)[:B3].to(torch.int32)
        st = [0]

        def step3():                                                    # the step without the per-step loss read-back
            st[0] += 1; m.step += 1
            m.compute_grads(rows, 0.1, m.step)
            if m.dp is not None:
                m.dp.sync()
            m.apply_grads()
        ms = timed(step3, 20, warm=3)
        fl = 3 * 2 * B3 * ni3 * 600 + 3 * 2 * B3 * 600 * 400 + 3 * 2 * B3 * 200 * 600     # fwd+bwd dense layers (input layer is a CSR gather)
        sus = tflops
        adam_bytes = 28 * sum(v.numel() for v in m.P.values())
        return {"metric": "multivae_users_per_sec", "value": B3 * world / (ms * 1e-3), "unit": "users/s", "ms_per_step": ms,
                "config": {"workload": f"configs[2]: MultiVAE 600/200, {nu3} x {ni3} (ML-20M shape, ~144 items/user), batch {B3}/GPU, dropout 0.5, "
                                       "one native call per step phase (8 wgmma GEMMs + fused elementwise + dense Adam)",
                           "parallelism": "single GPU" if world == 1 else f"data parallel x{world}: ONE all-reduce of the flat gradient buffer"},
                "roofline": {"bound": "tensor", "achieved": fl / (ms * 1e-3) / 1e12, "peak": sus, "unit": "TFLOP/s",
                             "frac": fl / (ms * 1e-3) / 1e12 / sus, "peak_source": which,
                             "adam_hbm_floor_ms": adam_bytes / (hbm * 1e9) * 1e3},
                "finite": bool(all(torch.isfinite(v).all().item() for v in m.P.values()))}
    block("vae", blk_vae)

    # ---- BASELINE configs[3]: NeuMF d=64 over row-sharded tables (users sharded, the [items, 2f] table row-sharded in
    # peer-addressed memory: the item-row gathers/scatters ride NVLink inside the kernels); N=4 is configs[3] itself
    def blk_neumf():
        from elliot_b200.recommender.neumf_sharded import ShardedNeuMFModel
        UPG, NI4, F4, B4 = 2_500_000, 1_000_000, 64, 1 << 20
        sh = ShardedNeuMFModel(UPG * world, NI4, F4, 1e-3, 42, dev, full_init=False)
        g4 = torch.Generator(device=dev); g4.manual_seed(9 + rank)
        uu = torch.randint(0, sh.uhi - sh.ulo, (B4,), device=dev, generator=g4, dtype=torch.int32)
        it = torch.randint(0, NI4, (B4,), device=dev, generator=g4, dtype=torch.int32)
        yy = (torch.arange(B4, device=dev) % 5 == 0).float()            # m = 4 negatives per positive
        ms = timed(lambda: sh.train_step((uu, it, yy)), 5, warm=2)
        out = {"metric": "neumf_samples_per_sec", "value": B4 * world / (ms * 1e-3), "unit": "samples/s", "ms_per_step": ms,
               "config": {"workload": f"configs[3] shape: NeuMF d={F4} (GMF + MLP 128-256-128-64), {UPG * world} users x {NI4} items, m=4, "
                                      f"batch {B4}/GPU, dense Keras Adam over every owned row each step",
                          "parallelism": f"users block-sharded, item table row-sharded over {world} GPU(s) in peer-mapped memory ({sh.items.buf.kind}); "
                                         "MLP replicated, one NCCL all-reduce of its gradients",
                          "nvlink_bytes_per_sample_each_way": 2 * F4 * 4 * (world - 1) / world},
               "loss_finite": bool(torch.isfinite(sh._loss).all().item())}
        sh.close()
        return out
    block("neumf", blk_neumf)

    # ---- N>1: BPR with the ITEM table row-sharded (catalogues too large to replicate): fused kernel over peer memory
    def blk_sharded():
        from elliot_b200.parallel import PeerShardedTable
        from elliot_b200.peer import PeerBuffer
        NIS = 1_000_000 * world
        items = PeerShardedTable(NIS, D, device=dev); items.local.normal_(); items.local.mul_(0.1)
        bias = PeerBuffer(items.shard_rows, device=dev)
        ipS, ixS = synth_csr_n(torch, dev, 700 + rank, N_USERS, NIS, 50)
        fS = ops.bloom_build(ipS, ixS, N_USERS)
        US = U.clone(); c = [0]
        items.barrier()

        grouped = world > 4

        def st():
            if not grouped:      # up to 3 peers: ONE kernel samples, gathers over NVLink, updates
                ops.bpr_step_sampled_peer_f32(US, items.ptrs, bias.ptr_array(), items.shard_rows, D, N_USERS, NIS, ipS, ixS, BATCH,
                                              seed, c[0] * BATCH, *HP, filter=fS)
            else:                # more: sample, bucket the triples by the owners of (i, j), then the step over peer memory
                tu, ti, tj = ops.bpr_sample_philox(N_USERS, NIS, ipS, ixS, BATCH, seed, c[0] * BATCH, filter=fS)
                tu, ti, tj = ops.group_by_owner([tu, ti, tj], 1, 2, items.shard_rows, rank, world)
                ops.bpr_step_peer_f32(US, items.ptrs, bias.ptr_array(), items.shard_rows, D, NIS, tu, ti, tj, *HP, _variant=variant[0])
            c[0] += 1
        variant, trial = [0], {}
        if grouped:              # which row staging crosses 7 peers better is measured, not assumed: registers (16) or shared memory (32)
            for v in (16, 32):
                variant[0] = v
                trial[v] = timed(st, 3, warm=2)
            variant[0] = min(trial, key=trial.get)
        ms = timed(st, 10, warm=3)
        out = {"metric": "bpr_triples_per_sec_sharded_items", "value": BATCH * world / (ms * 1e-3), "unit": "triples/s", "ms": ms,
               "per_gpu": BATCH / (ms * 1e-3),
               "config": {"workload": f"{N_USERS} users/GPU, {NIS} items row-sharded over {world} GPUs, d={D}, {BATCH} triples/step/GPU; item rows "
                                      f"loaded and atomically updated in their owner's memory over NVLink inside the training kernel ({items.buf.kind})"
                                      + ("; triples bucketed by the owners of (i, j) first (more than 4 GPUs)" if grouped else ""),
                          "nvlink_bytes_per_triple_each_way": 2 * (D * 4 + 4) * (world - 1) / world},
               "finite": bool(torch.isfinite(items.local).all().item())}
        if grouped:
            out["config"]["row_staging_trial_ms"] = {"registers": trial[16], "shared_memory": trial[32]}
        items.close(); bias.close()
        return out
    if world > 1:
        block("sharded", blk_sharded)

    # ---- sibling model on the same gather/dot/scatter shape: MF2020 pointwise logistic step (N=1)
    def blk_mf2020():
        lens = (indptr[1:] - indptr[:-1])
        pos_u = torch.repeat_interleave(torch.arange(N_USERS, dtype=torch.int32, device=dev), lens)
        Um, Vm = U.clone(), V.clone()
        ubm = torch.zeros(N_USERS, device=dev); ibm = torch.zeros(N_ITEMS, device=dev); gbm = torch.zeros(1, device=dev)
        c = [0]

        def st():
            ops.mf_pointwise_step_f32(Um, Vm, ubm, ibm, gbm, D, pos_u, indices, 1, N_ITEMS, 9, 0, 0.05, 0.0025, first=c[0] * BATCH, count=BATCH)
            c[0] += 1
        ms = timed(st, 5, warm=3)
        byt = 2 * (2 * D * 4 + 2 * 4)
        return {"metric": "mf2020_samples_per_sec", "value": BATCH / (ms * 1e-3), "unit": "samples/s", "ms": ms,
                "roofline": {"bound": "hbm", "alg_bytes_per_sample": byt, "achieved": byt * BATCH / (ms * 1e-3) / 1e9, "unit": "GB/s",
                             "frac": byt * BATCH / (ms * 1e-3) / 1e9 / hbm},
                "finite": bool(torch.isfinite(Um).all().item() and torch.isfinite(gbm).all().item())}
    if world == 1:
        block("mf2020", blk_mf2020)

    # ---- the C2 step under both schedules (on copies of the tables): what determinism costs
    def blk_schedules():
        Uc, Vc, bc = U.clone(), V.clone(), b.clone(); c = [0]
        res = {}
        for name, det in (("hogwild", False), ("rounds", True)):
            def st():
                ops.bpr_step_sampled_f32(Uc, Vc, bc, D, N_USERS, N_ITEMS, indptr, indices, BATCH, seed + 7, c[0] * BATCH, *HP,
                                         deterministic=det)
                c[0] += 1
            ms = timed(st, 10, warm=3)
            res[name] = {"ms_per_step": ms, "value": BATCH / (ms * 1e-3), "unit": "triples/s"}
        return {"config": {"workload": "C2 step as in the headline, free-running Hogwild vs deterministic rounds"}, **res}
    if world == 1:
        block("schedules", blk_schedules)

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    achieved = ALG_BYTES_SAMPLED * BATCH / (kern_ms * 1e-3) / 1e9
    traffic = traffic_of("bpr_hogwild")
    launches_per_step = 1 if world == 1 else (2 if chosen == "peer" else 3)
    par = "single GPU"
    if world > 1:
        par = ("user rows sharded per GPU; item table + biases replicated, deltas averaged every step: "
               + {"peer": "ONE kernel per rank reads its slice of every copy over NVLink and pushes corrections with vector atomics (no collective)",
                  "simple": "delta kernel -> NCCL all-reduce -> apply kernel, in line",
                  "overlap": "NCCL all-reduce one step late beside the next step (SM partition)"}[chosen])
    out = {
        "metric": "bpr_triples_per_sec", "value": value, "unit": "triples/s", "n_gpus": world, "steps": K, "warmup": W,
        "ms_per_step": ms_total / K, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"C2: BPRMF d=64, 1M users x 100K items per GPU, ~100 train items/user, {BATCH} triples/step, "
                               "fused sample+gather+score+grad+scatter kernel, vector atomics, "
                               + ("deterministic rounds" if rounds else "free-running Hogwild"),
                   "global_batch": BATCH * world, "parallelism": par,
                   "sync_schedule": {"chosen": chosen, "trial_ms": tune, "peer": peer_note, "partition": partition_note},
                   "l2": "inputs larger than L2 (256 MB user table + 400 MB CSR per GPU vs 50 MB), fresh random rows every step"},
        "roofline": {"bound": "hbm", "achieved": achieved, "peak": hbm, "unit": "GB/s", "frac": achieved / hbm,
                     "traffic": traffic, "frac_dram_measured": None if traffic is None else traffic / (kern_ms * 1e-3) / 1e9 / hbm,
                     "peak_source": which, "kernel": "bpr_hogwild_kernel<64,SAMPLE,ATOMIC>", "kernel_ms": kern_ms,
                     "alg_bytes_per_triple": ALG_BYTES_SAMPLED,
                     "note": "the 25.6 MB item table fits the 50 MB L2 at C2, so DRAM moves fewer bytes than the algorithmic count; "
                             "the `large` block is the regime where the two agree"},
        "e2e": {"value": e2e_value, "unit": "triples/s", "h2d_bytes_per_step": 8 * BATCH, "d2h_bytes_per_step": 8,
                "h2d_GBps_per_gpu": 8 * BATCH * K / (e2e_ms * 1e-3) / 1e9, "numa": numa,
                "path": "eb_bpr_step_host_packed_f32: pinned packed triples (8 B) -> ONE H2D -> kernel -> D2H loss; 3 steps in flight"},
        "gpu_launches": K * launches_per_step, "clocks": clk, "finite": finite, "loss_sum": loss.item(),
        "seconds_total": round(time.time() - t_start, 1),
    }
    ren = {"scoring": "scoring", "c5": "scoring_c5_slice", "exact": "exact_c1", "large": "c2_large_catalog", "vae": "multivae_c3",
           "neumf": "neumf_c4", "sharded": "sharded_bpr", "mf2020": "mf2020",
           "schedules": "c2_schedules"}
    for k, v in extra.items():
        out[ren[k]] = v
    if world == 1 and not args.no_cpu_baseline:
        out["cpu_baseline"] = cpu_baseline(indptr.cpu().numpy(), indices.cpu().numpy())
    print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


def traffic_of(name):
    """dram bytes per launch of a kernel from a stored capture (profiles/traffic_<name>.json) if one exists, else None."""
    tp = os.path.join(ROOT, "profiles", f"traffic_{name}.json")
    if os.path.exists(tp):
        return json.load(open(tp)).get("dram_bytes_per_launch")
    return None


if __name__ == "__main__":
    main()
