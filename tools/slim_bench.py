#!/usr/bin/env python
"""SLIM stage timings on one GPU; prints one JSON line.

With recsys_config.yml's Slim parameters (l1_ratio 0.0000119, alpha 0.0788, neighborhood 544), SlimModel.initialize()
(elliot_b200/recommender/slim.py) and the masked top-10 of every user (eb_rp3_score_topk_f32) are timed through the
model's phase marks (tools/benchlib.py): the operands (the memory check and the CSC upload), the batched coordinate
descent of every item (eb_slim_fit_f32), W's assembly (eb_slim_drop_f32 + eb_rp3_prune_cols_f32) and the top-10.  At C1
one run warms up, then --repeat runs are timed and the median is reported, with the epoch counts.

At ML-20M shape the whole fit is not run: one wave of problems (items 0 .. --ml20m-items - 1, the most popular items
of the generator, so the longest columns) is timed with the global-residual path, and the per-item rate is reported.  The card's
name, power limit and SM clocks are read in the same run.

Data sets (benchlib): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, ~1.0 M ratings 1-5, no test
split); ML-20M-shaped = 138 493 x 26 744 with ~18.4 M half-star ratings.

    python tools/slim_bench.py [--skip-ml20m] [--repeat N]
"""
import argparse
import json

import numpy as np
import torch

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.recommender._device import upload_csr
from elliot_b200.recommender.slim import SlimModel, seed_state

PARAMS = dict(l1_ratio=0.0000119, alpha=0.0788, neighborhood=544, seed=42)


def ml20m_wave(m, n_items):
    # a partial fit over the first `slots` items, which no model call offers: the one direct op call of the benches
    C = m.R.tocsc()
    C.sort_indices()
    csc, csr = upload_csr(C.indptr, C.indices, C.data, m.device), (m.urm[0], m.urm[1])
    slots = min(ops.slim_slots(m.n_users, False), n_items)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    _, n_iter, _, _, _ = ops.slim_fit(csc, csr, m.n_users, m.n_items, m.l1, m.l2, seed_state(m.seed), m.k,
                                      shared_residual=False, slots=slots, items=(0, slots))
    b.record()
    torch.cuda.synchronize()
    s = a.elapsed_time(b) / 1e3
    it = n_iter.cpu().numpy()[:slots]
    return {"items_timed": slots, "seconds": s, "items_per_s": slots / s, "epochs_median": float(np.median(it)),
            "epochs_max": int(it.max()), "note": "items 0 .. items_timed - 1 only, one wave; the full fit was not run"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-ml20m", action="store_true")
    ap.add_argument("--repeat", type=int, default=1)
    ap.add_argument("--ml20m-items", type=int, default=1056, help="items timed at ML-20M shape (one wave at most)")
    args = ap.parse_args()
    out = bl.card()
    out["clocks_sm_mhz"], out["clocks_max_sm_mhz"] = out["sm_clock_mhz"], out["sm_clock_max_mhz"]
    u, i, r, U, I = bl.c1_matrix()
    m, mask = SlimModel(bl.Data(u, i, r, U, I), device=bl.DEV, **PARAMS), bl.train_mask(u, i, U)

    def run(mark):
        m.initialize(mark=mark)
        m.topk(10, *mask)
        mark("score_top10")
    t = bl.repeat(run, args.repeat, seconds=True)
    t["gpu_total"] = sum(t.values())
    it = m.n_iter.cpu().numpy()
    out["c1"] = {"users": U, "items": I, "ratings": int(m.R.nnz), "w_nnz": int(m.W[1].numel()),
                 "shared_residual": ops.slim_shared_residual_fits(U), "slots": ops.slim_slots(U, True),
                 "epochs_median": float(np.median(it)), "epochs_max": int(it.max()), **t}
    del m
    torch.cuda.empty_cache()
    if not args.skip_ml20m:
        u, i, r, U, I = bl.ml20m_matrix()
        m = SlimModel(bl.Data(u, i, r, U, I), device=bl.DEV, **PARAMS)
        out["ml20m_shape"] = {"users": U, "items": I, "ratings": int(m.R.nnz), **ml20m_wave(m, args.ml20m_items)}
    out["reference_c1_slim_seconds"] = bl.reference_seconds("slim_c1.npz")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
