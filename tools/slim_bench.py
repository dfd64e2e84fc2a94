#!/usr/bin/env python
"""SLIM stage timings on one GPU; prints one JSON line.

With recsys_config.yml's Slim parameters (l1_ratio 0.0000119, alpha 0.0788, neighborhood 544), the stages of
SlimModel.initialize() and of scoring (elliot_b200/recommender/slim.py), each timed with CUDA events: the batched
coordinate descent of every item (eb_slim_fit_f32), W's assembly (eb_slim_drop_f32 + eb_rp3_prune_cols_f32) and the
masked top-10 of every user (eb_rp3_score_topk_f32).  At C1 one run warms up, then --repeat runs are timed and the
median is reported, with the epoch counts.

At ML-20M shape the whole fit is not run: one wave of problems (items 0 .. --ml20m-items - 1, the most popular items
of the generator, so the longest columns) is timed with the global-residual path, and the per-item rate is reported.  The card's
name, power limit and SM clocks are read in the same run.

Data sets (tools/knn_bench.py's generators): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, ~1.0 M
ratings 1-5, no test split); ML-20M-shaped = 138 493 x 26 744 with ~20 M half-star ratings.

    python tools/slim_bench.py [--skip-ml20m] [--repeat N]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from elliot_b200 import ops  # noqa: E402
from elliot_b200.recommender._device import upload_csr  # noqa: E402
from elliot_b200.recommender.slim import SlimModel, seed_state  # noqa: E402
from knn_bench import c1_matrix, ml20m_matrix  # noqa: E402

DEV = "cuda:0"
PARAMS = dict(l1_ratio=0.0000119, alpha=0.0788, neighborhood=544, seed=42)


class _Data:
    def __init__(self, u, i, r, U, I):
        self.sp_i_train_ratings = sp.csr_matrix((r, (u, i)), shape=(U, I), dtype=np.float32)


def _operands(m):
    C = m.R.tocsc()
    C.sort_indices()
    return upload_csr(C.indptr, C.indices, C.data, m.device), (m.urm[0], m.urm[1])


def run_once(m):
    names = ("fit", "weights", "score_top10")
    ev = {n: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for n in names}
    csc, csr = _operands(m)
    torch.cuda.synchronize()
    a, b = ev["fit"]
    a.record()
    coef_t, n_iter, gap, nnz, drop = ops.slim_fit(csc, csr, m.n_users, m.n_items, m.l1, m.l2, seed_state(m.seed), m.k)
    b.record()
    a, b = ev["weights"]
    a.record(); m.W = ops.slim_weights(coef_t, drop, nnz, m.k); b.record()
    a, b = ev["score_top10"]
    a.record(); ti, _ = m.topk(10, m.urm[0], m.urm[1]); b.record()
    torch.cuda.synchronize()
    t = {k: v[0].elapsed_time(v[1]) / 1e3 for k, v in ev.items()}
    return t, n_iter.cpu().numpy()


def ml20m_wave(m, n_items):
    csc, csr = _operands(m)
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


def _smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "not read"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-ml20m", action="store_true")
    ap.add_argument("--repeat", type=int, default=1)
    ap.add_argument("--ml20m-items", type=int, default=1056, help="items timed at ML-20M shape (one wave at most)")
    args = ap.parse_args()
    out = {"gpu": torch.cuda.get_device_properties(0).name, "power_limit_w": _smi("power.limit"),
           "clocks_sm_mhz": _smi("clocks.sm"), "clocks_max_sm_mhz": _smi("clocks.max.sm")}
    u, i, r, U, I = c1_matrix()
    m = SlimModel(_Data(u, i, r, U, I), device=DEV, **PARAMS)
    run_once(m)                                                                # warm-up
    runs = [run_once(m) for _ in range(args.repeat)]
    t = {k: float(np.median([x[0][k] for x in runs])) for k in runs[0][0]}
    t["gpu_total"] = sum(t.values())
    it = runs[0][1]
    out["c1"] = {"users": U, "items": I, "ratings": int(m.R.nnz), "w_nnz": int(m.W[1].numel()),
                 "shared_residual": ops.slim_shared_residual_fits(U), "slots": ops.slim_slots(U, True),
                 "epochs_median": float(np.median(it)), "epochs_max": int(it.max()), **t}
    del m
    torch.cuda.empty_cache()
    if not args.skip_ml20m:
        u, i, r, U, I = ml20m_matrix()
        m = SlimModel(_Data(u, i, r, U, I), device=DEV, **PARAMS)
        out["ml20m_shape"] = {"users": U, "items": I, "ratings": int(m.R.nnz), **ml20m_wave(m, args.ml20m_items)}
    g = np.load(os.path.join(ROOT, "tests", "golden", "slim_c1.npz"))
    out["reference_c1_slim_seconds"] = {"value": float(g["reference_seconds"]),
                                        "note": "whole reference run_experiment on one host core, minted with the golden, not this run"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
