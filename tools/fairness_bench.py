"""Time the device pass of the clustered fairness metrics (eb_eval_fairness_f64: BiasDisparityBR / BD, User/ItemMAD
rating and ranking, REO, RSP) next to the 19-metric pass (eb_eval_metrics_f64) on the same lists, at the C1 shape
(6 040 x 3 706) and the ML-20M shape (138 493 x 26 744), k = 10 and 100.  Synthetic data and lists as
eval_metrics_bench.py; 2 user clusters and 4 item popularity clusters (the shape of the reference's ML-1M
u_happy.tsv / i_pop.tsv), scores on every list.  CUDA events around `--iters` calls after `--warmup`; prints one JSON
line per shape and k, with the card, its power limit and SM clock.

    python tools/fairness_bench.py [--iters 50] [--warmup 5] [--out results/fairness_bench.json]
"""
import argparse
import json
import os
from types import SimpleNamespace

import numpy as np
import torch

import benchlib as bl
from eval_metrics_bench import SHAPES, lists, synth, timed
from elliot_b200 import ops
from elliot_b200.evaluation import ideal_dcg, metric_tables, position_tables


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = torch.device("cuda:0")
    gpu = bl.card()
    ref = np.load(os.path.join(bl.ROOT, "tests", "golden", "fairness_c1.npz"))
    rows = []
    for shape, (n_users, n_items, nnz) in SHAPES.items():
        train, test, logp = synth(n_users, n_items, nnz)
        cs = (test.indptr.astype(np.int64), test.indices.astype(np.int64), np.ones(test.nnz))
        has_rows = np.diff(test.indptr) > 0
        tab = metric_tables(SimpleNamespace(sp_i_train=train, transactions=train.nnz), cs, has_rows)
        t = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x)).to(dev, dt)
        g = np.random.default_rng(3)
        ucl = t(g.integers(0, 2, n_users), torch.int32)
        pop_rank = np.argsort(np.argsort(-np.asarray(train.sum(0)).ravel(), kind="stable"), kind="stable")
        icl = t(np.minimum(pop_rank * 4 // n_items, 3), torch.int32)
        for k in (10, 100):
            idx = lists(train, logp, k, dev)
            val = torch.rand(idx.shape, device=dev, dtype=torch.float64)
            disc, tail, inv = position_tables(k)
            base = (t(cs[0], torch.int64), t(cs[1], torch.int32))
            nineteen = base + (t(tab.user_info, torch.int32), t(tab.pop, torch.int32), t(tab.long_tail, torch.uint8),
                               t(tab.nov, torch.float64), t(disc, torch.float64), t(tail, torch.float64), t(inv, torch.float64))
            fair = base + (t(cs[2], torch.float64), t(ideal_dcg(cs, k), torch.float64), t(disc, torch.float64),
                           t(has_rows, torch.uint8), ucl, 2, icl, 4)
            ms19 = timed(lambda: ops.eval_topk_metrics(idx, k, *nineteen), a.iters, a.warmup)
            msf = timed(lambda: ops.eval_fairness(idx, k, *fair, scores=val), a.iters, a.warmup)
            c1, s1 = ops.eval_fairness(idx, k, *fair, scores=val)
            c2, s2 = ops.eval_fairness(idx, k, *fair, scores=val)
            row = {"shape": shape, "users": n_users, "items": n_items, "train_nnz": int(train.nnz), "k": k,
                   "fairness_ms": round(msf, 4), "nineteen_metric_ms": round(ms19, 4), "ratio": round(msf / ms19, 2),
                   "rerun_bit_identical": bool(torch.equal(c1, c2) and s1.cpu().numpy().tobytes() == s2.cpu().numpy().tobytes()),
                   "gpu": gpu}
            if shape == "C1":
                row["reference_evaluator_c1_top20_three_cutoffs_s"] = round(float(ref["reference_seconds"]), 2)
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
