#!/usr/bin/env python
"""RP3beta stage timings on one GPU; prints one JSON line.

Per data set, with recsys_config.yml's RP3beta parameters (neighborhood 546, alpha 1.0807, beta 0.7029,
normalize_similarity True), the stages of RP3Model.initialize() and of scoring (elliot_b200/recommender/rp3beta.py):
host preparation (Pui, Piu, degree and the powers in numpy; a host clock), upload, similarity (eb_rp3_similarity_f32),
row normalisation (eb_rp3_l1_rows_f32), column prune (eb_rp3_prune_cols_f32) and the masked top-10 of every user
(eb_rp3_score_topk_f32), each timed with CUDA events.  One run warms up, then --repeat runs are timed and the median is
reported.  The card's name and power limit are read in the same run.

Rates are counted from the data: the similarity makes sum_u |u|^2 ordered fp32 multiply-adds (every user's right row
once per item the user rated), scoring sum_u sum_{i in u} |W_i|.

Data sets (tools/knn_bench.py's generators): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, ~1.0 M
ratings 1-5, no test split); ML-20M-shaped = 138 493 x 26 744 with ~20 M half-star ratings.

    python tools/rp3beta_bench.py [--skip-ml20m] [--repeat N]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from elliot_b200 import ops  # noqa: E402
from elliot_b200.recommender._device import upload, upload_csr  # noqa: E402
from elliot_b200.recommender.rp3beta import RP3Model  # noqa: E402
from knn_bench import c1_matrix, ml20m_matrix  # noqa: E402

DEV = "cuda:0"
PARAMS = dict(neighborhood=546, alpha=1.0807, beta=0.7029, normalize_similarity=True)


class _Data:
    def __init__(self, u, i, r, U, I):
        self.sp_i_train_ratings = sp.csr_matrix((r, (u, i)), shape=(U, I), dtype=np.float32)


def run_once(m):
    names = ("upload", "similarity", "normalize", "prune", "score_top10")
    ev = {n: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for n in names}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pui, piu, degree = m.host_operands()
    R = m.R
    work = np.bincount(R.indices, weights=np.diff(R.indptr)[np.repeat(np.arange(m.n_users), np.diff(R.indptr))],
                       minlength=m.n_items)
    order_np = np.argsort(-work, kind="stable")
    host = time.perf_counter() - t0
    a, b = ev["upload"]
    a.record()
    Pui, Piu = upload_csr(*pui, m.device), upload_csr(*piu, m.device)
    deg, order = upload(degree, m.device, torch.float64), upload(order_np, m.device, torch.int32)
    b.record()
    a, b = ev["similarity"]
    a.record(); idx, val, cnt = ops.rp3_similarity(Piu, Pui, deg, m.k, order=order); b.record()
    a, b = ev["normalize"]
    a.record(); ops.rp3_l1_rows(val, cnt); b.record()
    a, b = ev["prune"]
    a.record(); m.W = ops.rp3_prune_cols(idx, val, cnt, m.k); b.record()
    del idx, val, Pui, Piu
    a, b = ev["score_top10"]
    a.record(); ti, _ = m.topk(10, m.urm[0], m.urm[1]); b.record()
    torch.cuda.synchronize()
    assert (ti >= 0).all()
    t = {k: v[0].elapsed_time(v[1]) / 1e3 for k, v in ev.items()}
    t["host_prepare"] = host
    return t, int(cnt.sum().item())


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
        m = RP3Model(_Data(u, i, r, U, I), device=DEV, **PARAMS)
        R = m.R
        lens = np.diff(R.indptr).astype(np.float64)
        sim_adds = float((lens ** 2).sum())
        run_once(m)                                                            # warm-up
        runs = [run_once(m) for _ in range(args.repeat)]
        t = {k: float(np.median([x[0][k] for x in runs])) for k in runs[0][0]}
        wl = np.diff(m.W[0].cpu().numpy())
        score_adds = float(wl[R.indices].sum())
        t["gpu_total"] = sum(v for k, v in t.items() if k != "host_prepare")
        t["similarity_ordered_adds"] = sim_adds
        t["similarity_adds_per_s"] = sim_adds / t["similarity"]
        t["score_ordered_adds"] = score_adds
        t["score_adds_per_s"] = score_adds / t["score_top10"]
        out[name] = {"users": U, "items": I, "ratings": int(R.nnz), "similarity_entries": runs[0][1],
                     "w_nnz": int(m.W[1].numel()), **t}
        del m
        torch.cuda.empty_cache()
    g = np.load(os.path.join(ROOT, "tests", "golden", "rp3beta_c1.npz"))
    out["reference_c1_rp3beta_seconds"] = {"value": float(g["reference_seconds"]),
                                           "note": "whole reference run_experiment on one host core, minted with the golden, not this run"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
