"""Does applying one step's BPR triples grouped by user pay, at the C2 shape?  (separate from bench.py)

Draws one step's 4M triples with the Philox sampler, then times the materialised-triple step (eb_bpr_step_f32) on
(a) the triples in sampler order and (b) the same triples stably sorted by user, alternating a and b on fresh copies of the
tables, with the L2 flushed before every launch.  Also times the sort, the sampler alone and the fused sampled step.
Prints one JSON object, with the card name and power limit read in the same run."""
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from elliot_b200 import ops                                                            # noqa: E402

dev = "cuda:0"
HP = (0.05, 0.0025, 0.0, 0.0025, 0.00025)
NU, NI, D, B = 1_000_000, 100_000, 64, 1 << 22
WARM, REPS = 3, 12


def csr(seed):
    g = torch.Generator(device=dev); g.manual_seed(seed)
    cand = (torch.rand(NU, 100, device=dev, generator=g) ** 2 * NI).to(torch.int32).clamp_(max=NI - 1)
    cand, _ = torch.sort(cand, dim=1)
    keep = torch.ones_like(cand, dtype=torch.bool); keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    indptr = torch.zeros(NU + 1, dtype=torch.int64, device=dev); indptr[1:] = torch.cumsum(keep.sum(1), 0)
    return indptr, cand[keep].contiguous()


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                                                              # noqa: BLE001
        return f"unknown ({type(e).__name__})"


def event_ms(fn):
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); z.record(); torch.cuda.synchronize()
    return a.elapsed_time(z)


def summary(xs):
    return {"median_ms": round(statistics.median(xs), 4), "min_ms": round(min(xs), 4), "max_ms": round(max(xs), 4), "n": len(xs)}


def main():
    g = torch.Generator(device=dev); g.manual_seed(1000)
    U0 = torch.randn(NU, D, device=dev, generator=g) * 0.1
    V0 = torch.randn(NI, D, device=dev, generator=g) * 0.1
    b0 = torch.zeros(NI, device=dev)
    U, V, b = U0.clone(), V0.clone(), b0.clone()
    flush = torch.empty(128 << 20, dtype=torch.uint8, device=dev)                     # > 50 MB L2
    indptr, indices = csr(100)

    tu, ti, tj = ops.bpr_sample_philox(NU, NI, indptr, indices, B, 42)
    key, perm = torch.sort(tu, stable=True)
    su, si, sj = key.contiguous(), ti[perm].contiguous(), tj[perm].contiguous()

    def fresh():
        U.copy_(U0); V.copy_(V0); b.copy_(b0); flush.zero_(); torch.cuda.synchronize()

    runs = {"a_sampler_order": lambda: ops.bpr_step_f32(U, V, b, D, tu, ti, tj, *HP),
            "b_user_sorted": lambda: ops.bpr_step_f32(U, V, b, D, su, si, sj, *HP)}
    times = {k: [] for k in runs}
    for it in range(WARM + REPS):
        for k, fn in runs.items():                                                     # a, b alternate
            fresh()
            ms = event_ms(fn)
            if it >= WARM:
                times[k].append(ms)

    def sort_only():
        k_, p_ = torch.sort(tu, stable=True)
        return ti[p_], tj[p_]
    sort_ms, samp_ms, fused_ms = [], [], []
    c = [0]

    def fused():
        ops.bpr_step_sampled_f32(U, V, b, D, NU, NI, indptr, indices, B, 42, c[0] * B, *HP)
        c[0] += 1
    for it in range(WARM + REPS):
        flush.zero_()
        s = event_ms(sort_only)
        flush.zero_()
        p = event_ms(lambda: ops.bpr_sample_philox(NU, NI, indptr, indices, B, 42, it * B))
        fresh()
        f = event_ms(fused)
        if it >= WARM:
            sort_ms.append(s); samp_ms.append(p); fused_ms.append(f)

    a, bb = times["a_sampler_order"], times["b_user_sorted"]
    half = len(a) // 2
    out = {"card": card(), "shape": f"{NU} users x {NI} items, d={D}, {B} triples",
           "step_f32": {k: summary(v) for k, v in times.items()},
           "a_vs_a_spread": round(abs(statistics.median(a[:half]) - statistics.median(a[half:])) / statistics.median(a), 4),
           "speedup_b_over_a": round(statistics.median(a) / statistics.median(bb), 3),
           "torch_stable_sort_and_gather": summary(sort_ms),
           "sampler_alone": summary(samp_ms),
           "fused_sampled_step": summary(fused_ms),
           "distinct_users": int(torch.unique(tu).numel())}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
