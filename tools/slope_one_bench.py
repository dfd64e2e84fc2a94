#!/usr/bin/env python
"""SlopeOne phase timings on one GPU; prints one JSON line per data set and a summary line.

For each data set SlopeOneModel.initialize (elliot_b200/recommender/slope_one.py) runs once to warm up and then --repeat
times, each followed by the masked top-10 of every user; each phase is timed with CUDA events and the medians are
reported: the upload of the dict-order CSR, the two bf16 operands (ratings times 2^s and the entry pattern), the three
exact tensor-core products per row slab (B^T B, X^T B, B^T X), the fp64 deviation kernel, and the scoring.

Arithmetic lower bounds printed beside them (not measurements): the scorer reads one fp64 row of E per train entry and
candidate tile, nnz x n_items x 8 bytes, at the data sheet's 3.35 TB/s HBM3 peak (less whatever L2 serves); the products
are 3 x 2 n_items^2 n_users flops.  The card's name, power limit and SM clock are read in the same run.

Data sets (tools/knn_bench.py's generators): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, 1-5
stars); ML-20M-shaped = 138 493 x 26 744, 20 M half-star ratings.

    python tools/slope_one_bench.py [--repeat N] [--skip-ml20m]
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
from elliot_b200.recommender.slope_one import SlopeOneModel  # noqa: E402
from knn_bench import c1_matrix, ml20m_matrix  # noqa: E402

DEV = "cuda:0"
HBM_PEAK = 3.35e12


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


def one_run(m, mask):
    marks = []

    def mark(phase):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        marks.append((phase, e))
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    m.initialize(mark)
    m.topk(10, *mask)
    mark("scoring")
    torch.cuda.synchronize()
    ms, prev = {}, start
    for phase, e in marks:
        ms[phase] = ms.get(phase, 0.0) + prev.elapsed_time(e)
        prev = e
    ms["initialize"] = start.elapsed_time([e for p, e in marks if p == "dev"][-1])
    return ms


def run(name, u, i, r, U, I, repeat):
    data = _Data(u, i, r, U, I)
    m = SlopeOneModel(data, DEV)
    srt = np.lexsort((i, u))
    indptr = np.zeros(U + 1, np.int64)
    np.cumsum(np.bincount(u, minlength=U), out=indptr[1:])
    mask = (torch.from_numpy(indptr).to(DEV), torch.from_numpy(i[srt].astype(np.int32)).to(DEV))
    one_run(m, mask)                                              # warm-up
    runs = [one_run(m, mask) for _ in range(repeat)]
    med = {k: round(float(np.median([x[k] for x in runs])), 3) for k in runs[0]}
    read = m.nnz * I * 8
    flops = 3 * 2.0 * I * I * U
    row = {"data": name, "users": U, "items": I, "nnz": m.nnz, "s": int(m.s), "slab_rows": m.slab_rows, "ms": med,
           "scoring_E_bytes_GB": round(read / 1e9, 1), "scoring_bound_ms_at_hbm_peak": round(read / HBM_PEAK * 1e3, 1),
           "scoring_TB_per_s": round(read / (med["scoring"] * 1e-3) / 1e12, 3),
           "products_TFLOP": round(flops / 1e12, 2), "products_TFLOP_per_s": round(flops / (med["products"] * 1e-3) / 1e12, 1)}
    print(json.dumps(row), flush=True)
    del m
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--skip-ml20m", action="store_true")
    args = ap.parse_args()
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"), "sm_clock_mhz": smi("clocks.sm"),
           "sm_clock_max_mhz": smi("clocks.max.sm")}
    rows = [run("C1", *c1_matrix(), args.repeat)]
    if not args.skip_ml20m:
        rows.append(run("ML-20M-shape", *ml20m_matrix(), max(1, args.repeat - 2)))
    res["runs"] = rows
    res["sm_clock_mhz_after"] = smi("clocks.sm")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
