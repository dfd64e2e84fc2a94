#!/usr/bin/env python
"""NonNegMF epoch timings on one GPU; prints one JSON line per data set and a summary line.

For each data set NonNegMFModel (elliot_b200/recommender/nonneg_mf.py) trains one epoch to warm up and then --epochs
epochs, each followed by the masked top-10 of every user.  Each phase is timed through the model's marks
(tools/benchlib.py) and the medians are reported: the dots (eb_nnmf_dots_f64), the bias chain (eb_nnmf_bias_chain_f64,
one thread), the item and the user row updates (eb_nnmf_row_update_f64), `epoch`, the sum of those four, and the
scoring.  Beside the chain: its nanoseconds per rating, and whether bi was staged in shared memory (n_items doubles
within the opt-in limit) or read in global memory.  The card's name, power limit and SM clock are read in the same run.

Data sets (benchlib): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, 1-5 stars); ML-20M-shaped =
138 493 x 26 744, ~18.4 M half-star ratings (bi fits shared memory); the same ratings over a 53 488-item catalogue
(item i of user u becomes 2 i + u mod 2), where bi does not fit.

    python tools/nonneg_mf_bench.py [--epochs N] [--skip-ml20m]
"""
import argparse
import json

import numpy as np
import torch

import benchlib as bl
from elliot_b200.recommender.nonneg_mf import NonNegMFModel


def run(name, u, i, r, U, I, epochs):
    mu = np.float32(r.astype(np.float64).sum() / (U * I))
    m = NonNegMFModel(bl.Data(u, i, r, U, I), U, I, mu, 10, 0.1, 0.001, random_seed=42, device=bl.DEV)
    mask = bl.train_mask(u, i, U)

    def one_epoch(mark):
        m.train_step(mark)
        m.topk(10, *mask)
        mark("scoring")
    t = bl.repeat(one_epoch, epochs)
    t["epoch"] = sum(v for k, v in t.items() if k != "scoring")
    med = {k: round(v, 3) for k, v in t.items()}
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
    res = bl.card()
    rows = [run("C1", *bl.c1_matrix(), args.epochs)]
    if not args.skip_ml20m:
        u, i, r, U, I = bl.ml20m_matrix()
        rows.append(run("ML-20M-shape", u, i, r, U, I, max(1, args.epochs - 2)))
        rows.append(run("ML-20M-ratings-53488-items", u, 2 * i + u % 2, r, U, 2 * I, max(1, args.epochs - 2)))
    res["runs"] = rows
    res["sm_clock_mhz_after"] = bl.card()["sm_clock_mhz"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
