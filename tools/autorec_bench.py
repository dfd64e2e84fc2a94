"""Time UserAutoRec and ItemAutoRec through the model's own code (recommender/autorec.py's AutoRecModel) at the C1 shape
(synth_c1's 6 040 x 3 706 file) and the ML-20M shape (benchlib's seeded 138 493 x 26 744 matrix), hidden_neuron 500.
UserAutoRec's rows are users, ItemAutoRec's items (the transpose).

Per shape, model and batch size (512 and the reference's default, every row in one batch): one epoch's phases — the
encoder (sparse product + sigmoid), the decoder kernel, dW1 + db1, Adam — each the median of benchlib.repeat over
`--iters` epochs after a warm-up, then top-10 of every user.  Beside the decoder's time:
  - its algorithmic bytes: per observed entry the W2 row read and the dW2 row reduction (2 x 4 H), per batch row the h
    read and the dpre1 write (2 x 4 H), and the achieved rate over the data sheet's 3.35 TB/s;
  - the data-sheet lower bound of the reference's dense formulation (three products of 2 B n_out H flops per step at the
    989 TFLOP/s dense bf16 peak), a computed bound, not a measurement.
Prints one JSON line per shape, model and batch size, with the card, its power limit and clocks.

    python tools/autorec_bench.py [--iters 3] [--out results/autorec_bench.json]
"""
import argparse
import json
import os

import numpy as np
import scipy.sparse as sp
import torch

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.recommender.autorec import LINEAR, SIGMOID, AutoRecModel

H = 500
HBM_PEAK = 3.35e12
BF16_PEAK = 989e12


def csr(m):
    m = sp.csr_matrix(m, dtype=np.float32); m.sort_indices()
    return (torch.from_numpy(m.indptr.astype(np.int64)).to(bl.DEV), torch.from_numpy(m.indices.astype(np.int32)).to(bl.DEV),
            torch.from_numpy(m.data.astype(np.float32)).to(bl.DEV))


def epoch(m, order, B):
    def run(mark):
        n = order.numel()
        for s in range(0, n, B):
            rows = order[s:s + B]
            m._loss.zero_()
            h = m.encode(rows)
            mark("encoder")
            dpre1 = torch.empty_like(h)
            ops.autorec_decoder_f32(*m.csr, rows, h, m.P[2], m.P[3], m.act, m._loss, m.G[2], m.G[3], dpre1)
            mark("decoder")
            ops.dmf_sparse_bwd(m.G[0], *m.csr, rows, dpre1)
            ops.colsum(dpre1, m.G[1])
            mark("dW1_db1")
            m.adam()
            mark("adam")
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = bl.card()
    lines = []
    for shape, make in (("C1", bl.c1_matrix), ("ML-20M", bl.ml20m_matrix)):
        u, i, _, n_users, n_items = make()
        X = sp.csr_matrix((np.ones(len(u), np.float32), (u, i)), shape=(n_users, n_items))
        X.sum_duplicates(); X.data[:] = 1.0
        T = int(X.nnz)
        mask = bl.train_mask(u, i, n_users)
        for name, act, M in (("UserAutoRec", LINEAR, X), ("ItemAutoRec", SIGMOID, X.T)):
            c = csr(M)
            n_rows, n_out = M.shape
            for B in (512, T):
                m = AutoRecModel(n_out, n_out, H, 1e-4, act, 42, bl.DEV, c)
                order = torch.randperm(n_rows, generator=torch.Generator().manual_seed(42)).to(torch.int32).to(bl.DEV)
                Bs = min(B, n_rows)
                rec = {"model": name, "shape": shape, "users": n_users, "items": n_items, "train": T, "hidden_neuron": H,
                       "batch": B, "rows_per_epoch": n_rows, "steps_per_epoch": -(-n_rows // Bs)}
                t = bl.repeat(epoch(m, order, Bs), args.iters)
                rec.update({f"{k}_ms": round(v, 3) for k, v in t.items()})
                rec["epoch_ms"] = round(sum(t.values()), 2)
                dec_bytes = 8 * H * T + 8 * H * n_rows
                rec.update({"decoder_bytes": dec_bytes, "decoder_TBps": round(dec_bytes / (t["decoder"] * 1e-3) / 1e12, 3),
                            "decoder_share_of_hbm_peak": round(dec_bytes / (t["decoder"] * 1e-3) / HBM_PEAK, 3),
                            "dense_formulation_bound_ms": round(3 * 2 * n_rows * n_out * H / BF16_PEAK * 1e3, 3),
                            "dense_formulation_bound_note": "computed: three 2 B n_out H products per epoch at 989 TFLOP/s "
                                                            "(data sheet, dense bf16); not a measurement"})
                if act == LINEAR:
                    rec.update({f"{k}_ms": round(v, 3) for k, v in bl.repeat(
                        lambda mark: (setattr(m, "_h_step", None), m.topk(10, *mask), mark("recommend_k10")), args.iters).items()})
                else:
                    perm = torch.randperm(n_rows, generator=torch.Generator().manual_seed(7)).tolist()
                    rec.update({f"{k}_ms": round(v, 3) for k, v in bl.repeat(
                        lambda mark: (m.item_topk(perm, 10, *mask), mark("recommend_k10")), args.iters).items()})
                rec.update({"reference": "not timed (TensorFlow is not installed)", "iters": args.iters, **card})
                print(json.dumps(rec), flush=True)
                lines.append(rec)
                del m
                torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
