#!/usr/bin/env python
"""ItemKNN / UserKNN phase timings on one GPU; prints one JSON line.

Per model (items / users) and data set, CUDA-event times of the phases the models run (elliot_b200/recommender/knn.py):
densify (eb_csr_to_dense_bf16), Gram (eb_gemm_bf16 over all row slabs), neighbours (eb_knn_neighbors_f32), transpose (the
index sort into W's CSR), score + top-10 of every user (eb_knn_score_topk_f32), and end to end.  Each configuration runs
once as warm-up and is then timed once (--repeat to time more runs; the median is reported).

The Gram rate is stated as DENSE algorithmic flops on a sparse matrix, 2 U I^2 (items) or 2 U^2 I (users), over the Gram
time, and as a share of the H100 SXM data-sheet dense bf16 peak (989 TFLOP/s at 700 W).  The reference's C1 seconds come
from tests/golden/itemknn_c1.npz: the whole reference run_experiment of the hello-world ItemKNN block on one host core,
minted when the golden was made, not in this run.

Data sets: C1 = every rating of elliot_b200/synth_c1.py's file (6 040 x 3 706, ~1.0 M ratings 1-5, no test split);
ML-20M-shaped = 138 493 x 26 744 with ~18.4 M distinct half-star ratings (20 M draws before duplicate
(user, item) pairs are dropped; popularity capped at ML-20M's largest item count, 67 310), generated from a seed.

    python tools/knn_bench.py [--skip-ml20m] [--repeat N]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elliot_b200 import ops, synth_c1  # noqa: E402
from elliot_b200.recommender import knn  # noqa: E402

DEV = "cuda:0"
PEAK_BF16 = 989e12


def c1_matrix():
    u, i, r = synth_c1.rows()
    return u - 1, i - 1, r.astype(np.float32), synth_c1.N_USERS, synth_c1.N_ITEMS


def ml20m_matrix(seed=20):
    U, I, N, cap = 138493, 26744, 20_000_263, 67310
    g = np.random.default_rng(seed)
    pop = 1.0 / np.arange(1, I + 1) ** 0.9
    for _ in range(4):
        pop = np.minimum(pop / pop.sum(), cap / N)
    pop /= pop.sum()
    act = np.clip(g.lognormal(np.log(80.0), 1.1, U), 20, 9000)
    act /= act.sum()
    u = g.choice(U, size=int(N * 1.02), p=act)
    i = g.choice(I, size=u.size, p=pop)
    key = np.unique(u.astype(np.int64) * I + i)[:N]
    u, i = key // I, key % I
    r = g.integers(1, 11, size=u.size) / 2.0
    return u, i, r.astype(np.float32), U, I


def to_dev(u, i, r, U, I):
    import scipy.sparse as sp
    m = sp.csr_matrix((r, (u, i)), shape=(U, I), dtype=np.float32)
    m.sort_indices()
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)
    return t(m.indptr, torch.int64), t(m.indices, torch.int32), t(m.data, torch.float32)


def run_once(urm, U, I, over, k_nn=50, k=10):
    ev = {name: (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for name in
          ("densify", "gram", "neighbours", "transpose", "score_topk", "end_to_end")}
    acc = {name: 0.0 for name in ev}

    def timed(name, fn):
        a, b = ev[name]
        a.record(); out = fn(); b.record(); torch.cuda.synchronize()
        acc[name] += a.elapsed_time(b)
        return out
    items = over == "items"
    n = I if items else U
    start = torch.cuda.Event(enable_timing=True); end = torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    s = knn.exactness_scale(urm[2].cpu().numpy())
    X, rs, cs = timed("densify", lambda: ops.csr_to_dense_bf16(*urm, I, scale=float(1 << s), row_sq=not items, col_sq=items))
    diag = cs if items else rs
    S = max(8, knn.SLAB_BYTES // (4 * n) // 8 * 8)
    slab = torch.empty((min(S, n), n), dtype=torch.float32, device=DEV)
    idx = torch.empty((n, k_nn), dtype=torch.int32, device=DEV)
    val = torch.empty((n, k_nn), dtype=torch.float32, device=DEV)
    for j0 in range(0, n, S):
        m = min(S, n - j0)
        C = slab[:m]
        if items:
            timed("gram", lambda: ops.gemm_bf16(X[:, j0:], X, m, n, U, a_rows_are_k=True, b_rows_are_k=True, out=C))
        else:
            timed("gram", lambda: ops.gemm_bf16(X[j0:], X, m, n, I, out=C))
        i_, v_, _ = timed("neighbours", lambda: ops.knn_neighbors(C, n, j0, diag, k_nn, cosine=True))
        idx[j0:j0 + m], val[j0:j0 + m] = i_, v_
    del X, slab
    W = timed("transpose", lambda: knn.transpose_lists(idx, val))
    A, B = (urm, W) if items else (W, urm)
    f = knn.frac_bits(knn._bound(A, B))
    timed("score_topk", lambda: ops.knn_score_topk(A, B, I, k, f, urm[0], urm[1]))
    end.record(); torch.cuda.synchronize()
    acc["end_to_end"] = start.elapsed_time(end)
    return {name: v / 1e3 for name, v in acc.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-ml20m", action="store_true")
    ap.add_argument("--repeat", type=int, default=1)
    args = ap.parse_args()
    props = torch.cuda.get_device_properties(0)
    out = {"gpu": props.name}
    try:
        import subprocess
        out["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                                              capture_output=True, text=True).stdout.strip()
    except OSError:
        out["power_limit_w"] = "not read"
    sets = {"c1": c1_matrix}
    if not args.skip_ml20m:
        sets["ml20m_shape"] = ml20m_matrix
    for name, make in sets.items():
        u, i, r, U, I = make()
        urm = to_dev(u, i, r, U, I)
        out[name] = {"users": U, "items": I, "ratings": int(urm[2].numel())}
        for over in ("items", "users"):
            run_once(urm, U, I, over)                                       # warm-up
            runs = [run_once(urm, U, I, over) for _ in range(args.repeat)]
            t = {key: float(np.median([x[key] for x in runs])) for key in runs[0]}
            flops = 2.0 * U * I * I if over == "items" else 2.0 * U * U * I
            t["gram_dense_tflops"] = flops / t["gram"] / 1e12
            t["gram_share_of_bf16_peak"] = flops / t["gram"] / PEAK_BF16
            out[name][("itemknn" if over == "items" else "userknn")] = t
        del urm
        torch.cuda.empty_cache()
    g = np.load(os.path.join(ROOT, "tests", "golden", "itemknn_c1.npz"))
    out["reference_c1_itemknn_seconds"] = {"value": float(g["reference_seconds"]),
                                           "note": "whole reference run_experiment on one host core, minted with the golden, not this run"}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
