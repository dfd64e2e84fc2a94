#!/usr/bin/env python
"""RP3beta stage timings on one GPU; prints one JSON line.

Per data set, with recsys_config.yml's RP3beta parameters (neighborhood 546, alpha 1.0807, beta 0.7029,
normalize_similarity True), RP3Model.initialize() (elliot_b200/recommender/rp3beta.py) and the masked top-10 of every
user (eb_rp3_score_topk_f32) are timed through the model's phase marks (tools/benchlib.py): host preparation (the
memory check, Pui, Piu, degree, the powers and the row work order in numpy; the device is idle, so its interval is the
host time), upload, similarity (eb_rp3_similarity_f32), row normalisation (eb_rp3_l1_rows_f32), column prune
(eb_rp3_prune_cols_f32) and the top-10.  One run warms up, then --repeat runs are timed and the median is reported.  The
card's name and power limit are read in the same run.

Rates are counted from the data: the similarity makes sum_u |u|^2 ordered fp32 multiply-adds (every user's right row
once per item the user rated), scoring sum_u sum_{i in u} |W_i|.

Data sets (benchlib): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, ~1.0 M ratings 1-5, no test
split); ML-20M-shaped = 138 493 x 26 744 with ~18.4 M half-star ratings.

    python tools/rp3beta_bench.py [--skip-ml20m] [--repeat N]
"""
import argparse
import json

import numpy as np
import torch

import benchlib as bl
from elliot_b200.recommender.rp3beta import RP3Model

PARAMS = dict(neighborhood=546, alpha=1.0807, beta=0.7029, normalize_similarity=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-ml20m", action="store_true")
    ap.add_argument("--repeat", type=int, default=1)
    args = ap.parse_args()
    out = bl.card()
    sets = {"c1": bl.c1_matrix}
    if not args.skip_ml20m:
        sets["ml20m_shape"] = bl.ml20m_matrix
    for name, make in sets.items():
        u, i, r, U, I = make()
        m, mask = RP3Model(bl.Data(u, i, r, U, I), device=bl.DEV, **PARAMS), bl.train_mask(u, i, U)

        def run(mark):
            m.initialize(mark)
            m.topk(10, *mask)
            mark("score_top10")
        t = bl.repeat(run, args.repeat, seconds=True)
        assert (m.topk(10, *mask)[0] >= 0).all()
        R = m.R
        sim_adds = float((np.diff(R.indptr).astype(np.float64) ** 2).sum())
        score_adds = float(np.diff(m.W[0].cpu().numpy())[R.indices].sum())
        t["gpu_total"] = sum(v for k, v in t.items() if k != "host_prepare")
        t["similarity_ordered_adds"] = sim_adds
        t["similarity_adds_per_s"] = sim_adds / t["similarity"]
        t["score_ordered_adds"] = score_adds
        t["score_adds_per_s"] = score_adds / t["score_top10"]
        out[name] = {"users": U, "items": I, "ratings": int(R.nnz), "w_nnz": int(m.W[1].numel()), **t}
        del m
        torch.cuda.empty_cache()
    out["reference_c1_rp3beta_seconds"] = bl.reference_seconds("rp3beta_c1.npz")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
