#!/usr/bin/env python
"""NonNegMF epoch timings on one GPU; prints one JSON line per data set and a summary line.

For each data set NonNegMFModel (elliot_b200/recommender/nonneg_mf.py) trains one epoch to warm up and then --epochs
epochs, each followed by the masked top-10 of every user.  Each phase is timed with CUDA events and the medians are
reported: the dots (eb_nnmf_dots_f64), the bias chain (eb_nnmf_bias_chain_f64, one thread), the item and the user
row updates (eb_nnmf_row_update_f64) and the scoring.  Beside the chain: its nanoseconds per rating, and whether bi
was staged in shared memory (n_items doubles within the opt-in limit) or read in global memory.  The card's name,
power limit and SM clock are read in the same run.

Data sets (tools/knn_bench.py's generators): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706,
1-5 stars); ML-20M-shaped = 138 493 x 26 744, 20 M half-star ratings (bi fits shared memory); the same ratings over a
53 488-item catalogue (item i of user u becomes 2 i + u mod 2), where bi does not fit.

    python tools/nonneg_mf_bench.py [--epochs N] [--skip-ml20m]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from elliot_b200.recommender.nonneg_mf import NonNegMFModel  # noqa: E402
from knn_bench import c1_matrix, ml20m_matrix  # noqa: E402

DEV = "cuda:0"


class _Data:
    """The fields dict_order_csr reads: users, items and the grouped (user, item, rating) arrays."""

    def __init__(self, u, i, r, U, I):
        o = np.argsort(u, kind="stable")
        self._tr = (u[o].astype(np.int64), i[o].astype(np.int64), r[o].astype(np.float64))
        self.users, self.items = list(range(U)), list(range(I))


def smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "not read"


def one_epoch(m, mask):
    marks = []

    def mark(phase):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        marks.append((phase, e))
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    m.train_step(mark)
    m.topk(10, *mask)
    mark("scoring")
    torch.cuda.synchronize()
    ms, prev = {}, start
    for phase, e in marks:
        ms[phase] = prev.elapsed_time(e)
        prev = e
    ms["epoch"] = start.elapsed_time(marks[-2][1])
    return ms


def run(name, u, i, r, U, I, epochs):
    mu = np.float32(r.astype(np.float64).sum() / (U * I))
    m = NonNegMFModel(_Data(u, i, r, U, I), U, I, mu, 10, 0.1, 0.001, random_seed=42, device=DEV)
    srt = np.lexsort((i, u))
    indptr = np.zeros(U + 1, np.int64)
    np.cumsum(np.bincount(u, minlength=U), out=indptr[1:])
    mask = (torch.from_numpy(indptr).to(DEV), torch.from_numpy(i[srt].astype(np.int32)).to(DEV))
    one_epoch(m, mask)                                            # warm-up
    runs = [one_epoch(m, mask) for _ in range(epochs)]
    med = {k: round(float(np.median([x[k] for x in runs])), 3) for k in runs[0]}
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    row = {"data": name, "users": U, "items": I, "nnz": m.nnz, "factors": 10, "ms": med,
           "chain_ns_per_rating": round(med["chain"] * 1e6 / m.nnz, 2),
           "bi_in": "shared" if I * 8 <= optin else "global", "chain_share_of_epoch": round(med["chain"] / med["epoch"], 3)}
    print(json.dumps(row), flush=True)
    del m
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--skip-ml20m", action="store_true")
    args = ap.parse_args()
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"), "sm_clock_mhz": smi("clocks.sm"),
           "sm_clock_max_mhz": smi("clocks.max.sm")}
    rows = [run("C1", *c1_matrix(), args.epochs)]
    if not args.skip_ml20m:
        u, i, r, U, I = ml20m_matrix()
        rows.append(run("ML-20M-shape", u, i, r, U, I, max(1, args.epochs - 2)))
        rows.append(run("ML-20M-ratings-53488-items", u, 2 * i + u % 2, r, U, 2 * I, max(1, args.epochs - 2)))
    res["runs"] = rows
    res["sm_clock_mhz_after"] = smi("clocks.sm")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
