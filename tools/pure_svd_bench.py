#!/usr/bin/env python
"""PureSVD phase timings on one GPU; prints one JSON line.

For each data set and factors in --factors, PureSVDModel.train_step (elliot_b200/recommender/pure_svd.py) runs once to
warm up and then --repeat times; each phase is timed with CUDA events and the medians are reported: the upload of both
CSRs and the start block, the 2 n_iter + 3 sparse products (eb_csr_spmm_f64), the orthonormalisations (Gram, pivoted
Cholesky, X M), the eigensolve with Q W, the sign/scale epilogue, and the masked top-10 of every user
(eb_score_topk_f64).  The sparse products' rate is given as gathered bytes per second: every stored entry reads one
w-wide fp64 row of X (8 w bytes) plus its 8 bytes of index and value, over the data sheet's 3.35 TB/s HBM3 peak.

--host also runs sklearn's randomized_svd (what the reference calls) on the same float32 matrix on one host core
(threadpoolctl limits BLAS to one thread): a HOST measurement, not a GPU one.  The card's name, power limit and SM
clock are read in the same run.

Data sets (tools/knn_bench.py's generators, binarised as sp_i_train is): C1 = every rating of elliot_b200/synth_c1.py's
file (6 040 x 3 706); ML-20M-shaped = 138 493 x 26 744.

    python tools/pure_svd_bench.py [--factors 10,50,190] [--repeat N] [--skip-ml20m] [--host]
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
from elliot_b200.recommender.pure_svd import PureSVDModel  # noqa: E402
from knn_bench import c1_matrix, ml20m_matrix  # noqa: E402

DEV = "cuda:0"
HBM_PEAK = 3.35e12


class _Data:
    def __init__(self, A):
        self.sp_i_train = A


def binary(u, i, r, U, I):
    A = sp.csr_matrix((np.ones(len(u), np.float32), (u, i)), shape=(U, I), dtype=np.float32)
    A.sum_duplicates()
    A.data[:] = 1.0
    return A


def smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "not read"


def one_fit(A, f):
    m = PureSVDModel(f, _Data(A), 42, DEV)
    marks = []

    def mark(phase):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        marks.append((phase, e))
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    m.train_step(mark)
    mask = (torch.from_numpy(A.indptr).to(DEV, torch.int64), torch.from_numpy(A.indices).to(DEV, torch.int32))
    t0 = torch.cuda.Event(enable_timing=True)
    t0.record()
    m.topk(10, *mask)
    t1 = torch.cuda.Event(enable_timing=True)
    t1.record()
    torch.cuda.synchronize()
    ms = {}
    prev = start
    for phase, e in marks:
        ms[phase] = ms.get(phase, 0.0) + prev.elapsed_time(e)
        prev = e
    ms["fit"] = start.elapsed_time(marks[-1][1])
    ms["topk10"] = t0.elapsed_time(t1)
    n_spmm = 2 * m.n_iter + 3
    gathered = (2 * m.n_iter + 2) * A.nnz * (8 * m.w + 8) + A.nnz * (8 * m.d + 8)
    return ms, n_spmm, gathered, m


def run(name, A, factors, repeat, host):
    out = []
    for f in factors:
        one_fit(A, f)                                             # warm-up
        runs = [one_fit(A, f) for _ in range(repeat)]
        keys = runs[0][0].keys()
        med = {k: float(np.median([r[0][k] for r in runs])) for k in keys}
        _, n_spmm, gathered, m = runs[0]
        rate = gathered / (med["spmm"] * 1e-3)
        row = {"data": name, "users": A.shape[0], "items": A.shape[1], "nnz": int(A.nnz), "factors": f, "w": m.w,
               "n_iter": m.n_iter, "transposed": m.transpose, "n_spmm": n_spmm, "ms": {k: round(v, 3) for k, v in med.items()},
               "spmm_gathered_GB": round(gathered / 1e9, 3), "spmm_TB_per_s": round(rate / 1e12, 3),
               "spmm_share_of_hbm_peak": round(rate / HBM_PEAK, 3)}
        if host:
            from sklearn.utils.extmath import randomized_svd
            from threadpoolctl import threadpool_limits
            with threadpool_limits(1):
                t = time.time()
                randomized_svd(A, n_components=f, random_state=42)
                row["host_sklearn_one_core_s"] = round(time.time() - t, 3)
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
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"), "sm_clock_mhz": smi("clocks.sm"),
           "sm_clock_max_mhz": smi("clocks.max.sm")}
    rows = run("C1", binary(*c1_matrix()), factors, args.repeat, args.host)
    if not args.skip_ml20m:
        rows += run("ML-20M-shape", binary(*ml20m_matrix()), factors, args.repeat, args.host)
    res["runs"] = rows
    res["sm_clock_mhz_after"] = smi("clocks.sm")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
