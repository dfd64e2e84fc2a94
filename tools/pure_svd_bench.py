#!/usr/bin/env python
"""PureSVD phase timings on one GPU; prints one JSON line.

For each data set and factors in --factors, PureSVDModel.train_step (elliot_b200/recommender/pure_svd.py) runs once to
warm up and then --repeat times, each followed by the masked top-10 of every user (eb_score_topk_f64); each phase is
timed through the model's marks (tools/benchlib.py) and the medians are reported: the upload of both CSRs and the start
block, the 2 n_iter + 3 sparse products (eb_csr_spmm_f64), the orthonormalisations (Gram, pivoted Cholesky, X M), the
eigensolve with Q W, the sign/scale epilogue, `fit`, the sum of those, and the top-10.  The sparse products' rate is
given as gathered bytes per second: every stored entry reads one w-wide fp64 row of X (8 w bytes) plus its 8 bytes of
index and value, over the data sheet's 3.35 TB/s HBM3 peak.

--host also runs sklearn's randomized_svd (what the reference calls) on the same float32 matrix on one host core
(threadpoolctl limits BLAS to one thread): a HOST measurement, not a GPU one.  The card's name, power limit and SM
clock are read in the same run.

Data sets (benchlib, binarised as sp_i_train is): C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706);
ML-20M-shaped = 138 493 x 26 744.

    python tools/pure_svd_bench.py [--factors 10,50,190] [--repeat N] [--skip-ml20m] [--host]
"""
import argparse
import json
import time

import benchlib as bl
from elliot_b200.recommender.pure_svd import PureSVDModel


def run(name, u, i, r, U, I, factors, repeat, host):
    data, mask = bl.Data(u, i, r, U, I), bl.train_mask(u, i, U)
    A = data.sp_i_train
    out = []
    for f in factors:
        m = PureSVDModel(f, data, 42, bl.DEV)

        def one_fit(mark):
            m.train_step(mark)
            m.topk(10, *mask)
            mark("topk10")
        t = bl.repeat(one_fit, repeat)
        t["fit"] = sum(v for k, v in t.items() if k != "topk10")
        n_spmm = 2 * m.n_iter + 3
        gathered = (2 * m.n_iter + 2) * A.nnz * (8 * m.w + 8) + A.nnz * (8 * m.d + 8)
        rate = gathered / (t["spmm"] * 1e-3)
        row = {"data": name, "users": U, "items": I, "nnz": int(A.nnz), "factors": f, "w": m.w,
               "n_iter": m.n_iter, "transposed": m.transpose, "n_spmm": n_spmm, "ms": {k: round(v, 3) for k, v in t.items()},
               "spmm_gathered_GB": round(gathered / 1e9, 3), "spmm_TB_per_s": round(rate / 1e12, 3),
               "spmm_share_of_hbm_peak": round(rate / 3.35e12, 3)}
        if host:
            from sklearn.utils.extmath import randomized_svd
            from threadpoolctl import threadpool_limits
            with threadpool_limits(1):
                t0 = time.time()
                randomized_svd(A, n_components=f, random_state=42)
                row["host_sklearn_one_core_s"] = round(time.time() - t0, 3)
        print(json.dumps(row), flush=True)
        out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--factors", default="10,50,190")
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--skip-ml20m", action="store_true")
    ap.add_argument("--host", action="store_true")
    args = ap.parse_args()
    factors = [int(x) for x in args.factors.split(",")]
    res = bl.card()
    rows = run("C1", *bl.c1_matrix(), factors, args.repeat, args.host)
    if not args.skip_ml20m:
        rows += run("ML-20M-shape", *bl.ml20m_matrix(), factors, args.repeat, args.host)
    res["runs"] = rows
    res["sm_clock_mhz_after"] = bl.card()["sm_clock_mhz"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
