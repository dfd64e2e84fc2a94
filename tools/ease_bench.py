#!/usr/bin/env python
"""EASE^R phase timings on one GPU; prints one JSON line.

Per data set, CUDA-event times of the phases of EASEModel.initialize() and of scoring (elliot_b200/recommender/ease.py):
Gram (densify + the exact bf16 tensor-core Gram in slabs + the fp64 normal matrix, eb_ease_normal_f64), inverse
(eb_inverse_f64), weights (eb_ease_weights_f32) and the masked top-10 of every user (eb_dense_score_topk_f32).  One run
warms up, then --repeat runs are timed and the median is reported.  The card's name and power limit are read in the same
run.

Rates are counted from shapes: the inverse costs 2 n^3 fp64 FLOP (Gauss-Jordan inversion), against 67 TFLOP/s (the H100
SXM data-sheet fp64 tensor-core peak, at 700 W; a data-sheet figure, not one reached); scoring reads 4 nnz n bytes of B
rows (one fp32 row of B per rating), against 3.35 TB/s (data-sheet HBM3 bandwidth).

The reference's C1 seconds come from tests/golden/ease_c1.npz: the whole reference run_experiment of the EASER block on
one host core, timed when the golden was minted, not in this run.

Data sets (tools/knn_bench.py's generators): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, ~1.0 M
ratings 1-5, no test split); ML-20M-shaped = 138 493 x 26 744 with ~18.4 M half-star ratings.

    python tools/ease_bench.py [--skip-ml20m] [--repeat N]
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
from elliot_b200.recommender import knn  # noqa: E402
from elliot_b200.recommender.ease import EASEModel  # noqa: E402
from knn_bench import c1_matrix, ml20m_matrix  # noqa: E402

DEV = "cuda:0"
PEAK_FP64_TC = 67e12
PEAK_HBM = 3.35e12


class _Data:
    def __init__(self, u, i, r, U, I):
        self.sp_i_train_ratings = sp.csr_matrix((r, (u, i)), shape=(U, I), dtype=np.float32)


def run_once(m):
    names = ("gram", "inverse", "weights", "score_top10")
    ev = {n: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for n in names}
    n = m.n_items
    torch.cuda.synchronize()
    a, b = ev["gram"]
    a.record()
    X, s, _ = knn.dense_operand(m.urm, m.n_users, n, "items")
    A = torch.empty((n, n), dtype=torch.float64, device=DEV)
    for j0, C in knn.gram_slabs(X, m.n_users, n, "items"):
        ops.ease_normal_f64(C, j0, m.count, m.l2_norm, 4.0 ** -s, A)
    b.record()
    del X, C
    a, b = ev["inverse"]
    a.record(); ops.inverse_f64(A); b.record()
    m.B = None
    a, b = ev["weights"]
    a.record(); m.B = ops.ease_weights_f32(A); b.record()
    del A
    m.frac_bits = knn.frac_bits(knn._bound(m.urm, (None, None, m.B.view(-1))))
    a, b = ev["score_top10"]
    a.record(); m.topk(10, m.urm[0], m.urm[1]); b.record()
    torch.cuda.synchronize()
    assert torch.isfinite(m.B).all()
    return {k: v[0].elapsed_time(v[1]) / 1e3 for k, v in ev.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-ml20m", action="store_true")
    ap.add_argument("--repeat", type=int, default=1)
    args = ap.parse_args()
    out = {"gpu": torch.cuda.get_device_properties(0).name}
    try:
        out["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                              capture_output=True, text=True).stdout.strip()
    except OSError:
        out["power_limit_w"] = "not read"
    sets = {"c1": c1_matrix}
    if not args.skip_ml20m:
        sets["ml20m_shape"] = ml20m_matrix
    for name, make in sets.items():
        u, i, r, U, I = make()
        m = EASEModel(_Data(u, i, r, U, I), 1e3, DEV)
        nnz = int(m.urm[2].numel())
        run_once(m)                                                            # warm-up
        runs = [run_once(m) for _ in range(args.repeat)]
        t = {k: float(np.median([x[k] for x in runs])) for k in runs[0]}
        t["total"] = sum(t.values())
        t["inverse_tflops"] = 2.0 * I ** 3 / t["inverse"] / 1e12
        t["inverse_share_of_fp64_tc_peak"] = 2.0 * I ** 3 / PEAK_FP64_TC / t["inverse"]
        t["score_b_bytes"] = 4.0 * nnz * I
        t["score_tb_per_s"] = 4.0 * nnz * I / t["score_top10"] / 1e12
        t["score_share_of_hbm_peak"] = 4.0 * nnz * I / PEAK_HBM / t["score_top10"]
        out[name] = {"users": U, "items": I, "ratings": nnz, **t}
        del m
        torch.cuda.empty_cache()
    g = np.load(os.path.join(ROOT, "tests", "golden", "ease_c1.npz"))
    out["reference_c1_easer_seconds"] = {"value": float(g["reference_seconds"]),
                                         "note": "whole reference run_experiment on one host core, minted with the golden, not this run"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
