"""Time the AUC / GAUC rank pass (ops.score_rank: every relevant item's rank in the whole catalogue) against the top-10
scorer of the same tables (ops.score_topk, k = 10), at the C1 shape (synth_c1's 6 040 x 3 706 file) and the ML-20M shape
(benchlib's seeded 138 493 x 26 744 matrix), fp32 and fp64, d = 64.  80 % of each user's ratings are the train mask,
the other 20 % the relevant items.  Random N(0, 0.1) tables.  Per call: the median of benchlib.repeat over `--iters`
runs after one warm-up run.  Prints one JSON line per shape and precision, with the card, its power limit and clocks.

    python tools/auc_bench.py [--iters 10] [--out results/auc_bench.json]
"""
import argparse
import json
import os

import numpy as np
import torch

import benchlib as bl
from elliot_b200 import ops

D = 64


def split(u, i, n_users, seed=0):
    """(train mask CSR, item-sorted relevant CSR) on the device: a seeded 80 / 20 split of the ratings."""
    g = np.random.default_rng(seed)
    test = g.random(u.size) < 0.2
    rel_u, rel_i = u[test], i[test]
    indptr = np.zeros(n_users + 1, np.int64)
    np.cumsum(np.bincount(rel_u, minlength=n_users), out=indptr[1:])
    rel = bl.upload(indptr, bl.DEV, torch.int64), bl.upload(rel_i[np.lexsort((rel_i, rel_u))], bl.DEV, torch.int32)
    return bl.train_mask(u[~test], i[~test], n_users), rel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = bl.card()
    lines = []
    for shape, make in (("C1", bl.c1_matrix), ("ML-20M", bl.ml20m_matrix)):
        u, i, _, n_users, n_items = make()
        (mp, mi), (rp, ri) = split(u, i, n_users)
        g = torch.Generator(device=bl.DEV).manual_seed(0)
        for dtype in (torch.float32, torch.float64):
            U = torch.randn(n_users, D, generator=g, device=bl.DEV, dtype=dtype) * 0.1
            V = torch.randn(n_items, D, generator=g, device=bl.DEV, dtype=dtype) * 0.1
            b = torch.zeros(n_items, device=bl.DEV, dtype=dtype)
            t = bl.repeat(lambda mark: (ops.score_rank(U, V, b, D, rp, ri, mp, mi), mark("rank"),
                                        ops.score_topk(U, V, b, D, 10, mp, mi), mark("topk10")), args.iters)
            n_pos, _ = ops.score_rank(U, V, b, D, rp, ri, mp, mi)
            rec = {"shape": shape, "users": n_users, "items": n_items, "dtype": str(dtype).split(".")[-1], "d": D,
                   "relevant": int(ri.numel()), "ranked": int(n_pos.sum().item()), "rank_ms": round(t["rank"], 3),
                   "score_topk_k10_ms": round(t["topk10"], 3), "iters": args.iters, **card}
            print(json.dumps(rec), flush=True)
            lines.append(rec)
            del U, V, b
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
