"""A/B of the fused Hogwild step on one GPU (separate from bench.py): with / without the per-user membership signatures (an
L2 prefetch of the rows was tried and removed: -10 %); C2 shape and the large-catalogue shape.  Prints one JSON object."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from elliot_b200 import ops                                                            # noqa: E402

dev = "cuda:0"
HP = (0.05, 0.0025, 0.0, 0.0025, 0.00025)
nu, d, B = 1_000_000, 64, 1 << 22


def csr(ni, seed):
    g = torch.Generator(device=dev); g.manual_seed(seed)
    cand = (torch.rand(nu, 100, device=dev, generator=g) ** 2 * ni).to(torch.int32).clamp_(max=ni - 1)
    cand, _ = torch.sort(cand, dim=1)
    keep = torch.ones_like(cand, dtype=torch.bool); keep[:, 1:] = cand[:, 1:] != cand[:, :-1]
    indptr = torch.zeros(nu + 1, dtype=torch.int64, device=dev); indptr[1:] = torch.cumsum(keep.sum(1), 0)
    return indptr, cand[keep].contiguous()


def timed(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    z.record(); torch.cuda.synchronize()
    return a.elapsed_time(z) / reps


out = {}
for ni in (100_000, 2_000_000):
    U = torch.randn(nu, d, device=dev) * 0.1; V = torch.randn(ni, d, device=dev) * 0.1; b = torch.zeros(ni, device=dev)
    ip, ix = csr(ni, 100)
    filt = ops.bloom_build(ip, ix, nu)
    c = [0]
    res = {}
    for name, f in (("filter", filt), ("no filter", None)):
        def st():
            ops.bpr_step_sampled_f32(U, V, b, d, nu, ni, ip, ix, B, 42, c[0] * B, *HP, filter=f)
            c[0] += 1
        ms = timed(st)
        res[name] = {"ms": round(ms, 4), "G_triples_per_s": round(B / ms / 1e6, 3)}
    res["finite"] = bool(torch.isfinite(U).all().item() and torch.isfinite(V).all().item())
    out[f"items_{ni}"] = res
    del U, V, b, ip, ix, filt
    torch.cuda.empty_cache()
print(json.dumps(out, indent=1))
