"""A/B of the grouped C2 step with and without the schedule prefetch (ops.set_bpr_prefetch), separate from bench.py: alternating
runs of consecutive steps, then one torch.profiler run per arrangement that splits the kernel time into update, key pass and
sort and measures how much of the key pass and sort ran while an update kernel was running.  Prints one JSON object.

    python tools/bpr_prefetch_probe.py [--rounds R] [--steps K] [--trace-dir DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import BATCH, D, HP, N_ITEMS, N_USERS, synth_csr   # noqa: E402
from elliot_b200 import ops                                   # noqa: E402

ARMS = {"serial": False, "prefetch": True}


def kernel_class(name):
    if "bpr_grouped_kernel" in name:
        return "update"
    if "user_key_kernel" in name:
        return "key"
    if "DeviceRadixSort" in name or "memset" in name.lower():
        return "sort"
    return None


def overlap(a, b):
    """total length of the intersection of two lists of (start, end) intervals"""
    tot = 0.0
    for s, e in a:
        for t, f in b:
            if f > s and t < e:
                tot += min(e, f) - max(s, t)
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--trace-dir", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator(device=dev); g.manual_seed(1000)
    U = torch.randn(N_USERS, D, device=dev, generator=g) * 0.1
    V = torch.randn(N_ITEMS, D, device=dev, generator=g) * 0.1
    b = torch.zeros(N_ITEMS, device=dev)
    indptr, indices = synth_csr(torch, dev, seed=100)
    c = [0]

    def steps(k):
        for _ in range(k):
            ops.bpr_step_sampled_f32(U, V, b, D, N_USERS, N_ITEMS, indptr, indices, BATCH, 42, c[0] * BATCH, *HP)
            c[0] += 1

    def timed(k):
        steps(4)
        torch.cuda.synchronize()
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); steps(k); z.record()
        torch.cuda.synchronize()
        return a.elapsed_time(z) / k

    res = {name: [] for name in ARMS}
    for _ in range(args.rounds):
        for name, on in ARMS.items():
            ops.set_bpr_prefetch(on)
            res[name].append(round(timed(args.steps), 4))
    out = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip(),
           "ms_per_step": res, "median": {k: sorted(v)[len(v) // 2] for k, v in res.items()}}

    from torch.profiler import ProfilerActivity, profile
    prof_out = {}
    tdir = args.trace_dir or tempfile.mkdtemp()
    os.makedirs(tdir, exist_ok=True)
    for name, on in ARMS.items():
        ops.set_bpr_prefetch(on)
        steps(4); torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            steps(10); torch.cuda.synchronize()
        path = os.path.join(tdir, f"bpr_prefetch_{name}.json")
        prof.export_chrome_trace(path)
        ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") in ("kernel", "gpu_memset")]
        iv = {}
        for e in ev:
            k = kernel_class(e["name"])
            if k:
                iv.setdefault(k, []).append((e["ts"], e["ts"] + e["dur"]))
        span = max(e["ts"] + e["dur"] for e in ev) - min(e["ts"] for e in ev)
        prof_out[name] = {"ms_per_step_traced": round(span / 10 / 1e3, 4),
                          **{f"{k}_ms": round(sum(f - s for s, f in v) / 10 / 1e3, 4) for k, v in iv.items()},
                          "key_sort_overlapped_with_update_ms": round(
                              overlap(iv.get("key", []) + iv.get("sort", []), iv.get("update", [])) / 10 / 1e3, 4)}
    out["profile"] = prof_out
    ops.set_bpr_prefetch(True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
