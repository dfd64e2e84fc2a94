"""Time the device evaluation of top-k lists: the 19-metric pass (eb_eval_metrics_f64) against the four-metric kernel
(eb_eval_topk_f64, nDCG / HR / Precision / Recall), at the C1 shape (6 040 x 3 706) and the ML-20M shape
(138 493 x 26 744), k = 10 and 100.  Synthetic data: a popularity-skewed train matrix of ~1.0 M / ~20 M entries, 20 % as
many test rows, and popularity-skewed lists of distinct unrated items drawn on the device.  CUDA events around `--iters`
calls after `--warmup`; prints one JSON line per shape and k, with the card, its power limit and SM clock.

    python tools/eval_metrics_bench.py [--iters 50] [--warmup 5] [--out results/eval_metrics_bench.json]
"""
import argparse
import json
import os
from types import SimpleNamespace

import numpy as np
import scipy.sparse as sp
import torch

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.evaluation import metric_tables, position_tables

SHAPES = {"C1": (6040, 3706, 1_000_000), "ML-20M": (138493, 26744, 20_000_000)}


def synth(n_users, n_items, nnz, seed=0):
    g = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, n_items + 1) ** 0.9
    p /= p.sum()
    def csr(n):
        m = sp.csr_matrix((np.ones(n, np.float32), (g.integers(0, n_users, n), g.choice(n_items, n, p=p))),
                          shape=(n_users, n_items))
        m.sum_duplicates(); m.data[:] = 1
        return m
    train, test = csr(nnz), csr(nnz // 5)
    test = test - test.multiply(train)                               # test rows the user has not rated
    test.eliminate_zeros(); test.sort_indices()
    return train, test, np.log(p)


def lists(train, logp, k, dev, chunk=4096):
    """Top-k of log pop + Gumbel noise over the unrated items: popularity-skewed lists of distinct items."""
    n_users, n_items = train.shape
    lp = torch.from_numpy(logp).to(dev)
    out = torch.empty(n_users, k, dtype=torch.int32, device=dev)
    gen = torch.Generator(device=dev).manual_seed(1)
    for a in range(0, n_users, chunk):
        b = min(n_users, a + chunk)
        s = lp[None, :] - torch.log(-torch.log(torch.rand(b - a, n_items, device=dev, generator=gen, dtype=torch.float64)))
        m = train[a:b].tocoo()
        s[torch.from_numpy(m.row).to(dev).long(), torch.from_numpy(m.col).to(dev).long()] = -float("inf")
        out[a:b] = torch.topk(s, k, dim=1).indices.int()
    return out


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


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
    ref = np.load(os.path.join(bl.ROOT, "tests", "golden", "metrics_c1.npz"))
    rows = []
    for shape, (n_users, n_items, nnz) in SHAPES.items():
        train, test, logp = synth(n_users, n_items, nnz)
        cs = (test.indptr.astype(np.int64), test.indices.astype(np.int64), np.ones(test.nnz))
        tab = metric_tables(SimpleNamespace(sp_i_train=train, transactions=train.nnz), cs, np.diff(test.indptr) > 0)
        t = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x)).to(dev, dt)
        for k in (10, 100):
            idx = lists(train, logp, k, dev)
            disc, tail, inv = position_tables(k)
            base = (t(cs[0], torch.int64), t(cs[1], torch.int32))
            four = base + (t(cs[2], torch.float64), t(np.zeros(n_users), torch.float64), t(disc, torch.float64))
            nineteen = base + (t(tab.user_info, torch.int32), t(tab.pop, torch.int32), t(tab.long_tail, torch.uint8),
                               t(tab.nov, torch.float64), t(disc, torch.float64), t(tail, torch.float64), t(inv, torch.float64))
            ms4 = timed(lambda: ops.eval_topk(idx, k, *four), a.iters, a.warmup)
            ms19 = timed(lambda: ops.eval_topk_metrics(idx, k, *nineteen), a.iters, a.warmup)
            s1, _ = ops.eval_topk_metrics(idx, k, *nineteen)
            s2, _ = ops.eval_topk_metrics(idx, k, *nineteen)
            row = {"shape": shape, "users": n_users, "items": n_items, "train_nnz": int(train.nnz), "k": k,
                   "four_metric_ms": round(ms4, 4), "nineteen_metric_ms": round(ms19, 4), "ratio": round(ms19 / ms4, 2),
                   "rerun_bit_identical": bool(torch.equal(s1, s2)), "gpu": gpu}
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
