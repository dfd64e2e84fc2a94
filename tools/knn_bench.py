#!/usr/bin/env python
"""ItemKNN / UserKNN phase timings on one GPU; prints one JSON line.

Per model (items / users) and data set, KNNModel.initialize (elliot_b200/recommender/knn.py) and the top-10 of every user
are timed through the model's phase marks (tools/benchlib.py): densify (eb_csr_to_dense_bf16 and the exactness checks),
Gram (eb_gemm_bf16 over all row slabs), neighbours (eb_knn_neighbors_f32), transpose (the index sort into W's CSR and the
scoring bound), score + top-10 of every user (eb_knn_score_topk_f32), and end to end, their sum.  Each configuration
runs once as warm-up and is then timed once (--repeat to time more runs; the median is reported).

The Gram rate is stated as DENSE algorithmic flops on a sparse matrix, 2 U I^2 (items) or 2 U^2 I (users), over the Gram
time, and as a share of the H100 SXM data-sheet dense bf16 peak (989 TFLOP/s at 700 W).  The reference's C1 seconds come
from tests/golden/itemknn_c1.npz: the whole reference run_experiment of the hello-world ItemKNN block on one host core,
minted when the golden was made, not in this run.

Data sets (benchlib): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, ~1.0 M ratings 1-5, no test
split); ML-20M-shaped = 138 493 x 26 744 with ~18.4 M distinct half-star ratings, generated from a seed.

    python tools/knn_bench.py [--skip-ml20m] [--repeat N]
"""
import argparse
import json

import torch

import benchlib as bl
from elliot_b200.recommender.knn import KNNModel

PEAK_BF16 = 989e12


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
        data, mask = bl.Data(u, i, r, U, I), bl.train_mask(u, i, U)
        out[name] = {"users": U, "items": I, "ratings": int(data.sp_i_train_ratings.nnz)}
        for over in ("items", "users"):
            m = KNNModel(data, 50, "cosine", False, over, bl.DEV)

            def run(mark):
                m.initialize(mark)
                m.topk(10, *mask)
                mark("score_topk")
            t = bl.repeat(run, args.repeat, seconds=True)
            t["end_to_end"] = sum(t.values())
            flops = 2.0 * U * I * I if over == "items" else 2.0 * U * U * I
            t["gram_dense_tflops"] = flops / t["gram"] / 1e12
            t["gram_share_of_bf16_peak"] = flops / t["gram"] / PEAK_BF16
            out[name][("itemknn" if over == "items" else "userknn")] = t
            del m
            torch.cuda.empty_cache()
    out["reference_c1_itemknn_seconds"] = bl.reference_seconds("itemknn_c1.npz")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
