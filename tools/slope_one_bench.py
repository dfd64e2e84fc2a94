#!/usr/bin/env python
"""SlopeOne phase timings on one GPU; prints one JSON line per data set and a summary line.

For each data set SlopeOneModel.initialize (elliot_b200/recommender/slope_one.py) runs once to warm up and then --repeat
times, each followed by the masked top-10 of every user; each phase is timed through the model's marks
(tools/benchlib.py) and the medians are reported: the upload of the dict-order CSR, the two bf16 operands (ratings times
2^s and the entry pattern), the three exact tensor-core products per row slab (B^T B, X^T B, B^T X), the fp64 deviation
kernel, the scoring, and `initialize`, the sum of the first four.

Arithmetic lower bounds printed beside them (not measurements): the scorer reads one fp64 row of E per train entry and
candidate tile, nnz x n_items x 8 bytes, at the data sheet's 3.35 TB/s HBM3 peak (less whatever L2 serves); the products
are 3 x 2 n_items^2 n_users flops.  The card's name, power limit and SM clock are read in the same run.

Data sets (benchlib): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, 1-5 stars); ML-20M-shaped =
138 493 x 26 744, ~18.4 M half-star ratings.

    python tools/slope_one_bench.py [--repeat N] [--skip-ml20m]
"""
import argparse
import json

import torch

import benchlib as bl
from elliot_b200.recommender.slope_one import SlopeOneModel

HBM_PEAK = 3.35e12


def run(name, u, i, r, U, I, repeat):
    m, mask = SlopeOneModel(bl.Data(u, i, r, U, I), bl.DEV), bl.train_mask(u, i, U)

    def one_run(mark):
        m.initialize(mark)
        m.topk(10, *mask)
        mark("scoring")
    t = bl.repeat(one_run, repeat)
    t["initialize"] = sum(v for k, v in t.items() if k != "scoring")
    med = {k: round(v, 3) for k, v in t.items()}
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
    res = bl.card()
    rows = [run("C1", *bl.c1_matrix(), args.repeat)]
    if not args.skip_ml20m:
        rows.append(run("ML-20M-shape", *bl.ml20m_matrix(), max(1, args.repeat - 2)))
    res["runs"] = rows
    res["sm_clock_mhz_after"] = bl.card()["sm_clock_mhz"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
