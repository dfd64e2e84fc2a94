"""Time DMF through the model's own code (recommender/dmf.py's DMFModel, the sampler ops.MtPointwiseRatioSampler) at the C1
shape (synth_c1's 6 040 x 3 706 file) and the ML-20M shape (benchlib's seeded 138 493 x 26 744 matrix), with the
reference's defaults: user_mlp = item_mlp = (64, 32), neg_ratio 5, cosine.  An epoch is transactions x 6 samples.

Per shape and batch size (512 and the reference's default, the whole epoch in one batch): the epoch's phases — the
sampler, the two towers' forward and backward, the head, Adam — each the median of benchlib.repeat over `--iters` runs
after a warm-up, and top-10 of every user.  At batch 512 only the first `--steps` steps of the epoch are timed and the
epoch is their time scaled by steps per epoch (`epoch_est_ms`); the sampler is timed on the samples those steps use.
A batch whose towers do not fit in the device's free memory is reported with its estimated need instead of a time.
Prints one JSON line per shape and batch size, with the card, its power limit and clocks.

    python tools/dmf_bench.py [--iters 3] [--steps 2000] [--out results/dmf_bench.json]
"""
import argparse
import json
import os

import numpy as np
import scipy.sparse as sp
import torch

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.recommender.dmf import DMFModel

MLP, NEG = [64, 32], 5


def csrs(u, i, r, n_users, n_items):
    R = sp.csr_matrix((np.asarray(r, np.float32), (u, i)), shape=(n_users, n_items))
    R.sum_duplicates(); R.sort_indices()
    C = R.T.tocsr(); C.sort_indices()
    up = lambda M: (torch.from_numpy(M.indptr.astype(np.int64)).to(bl.DEV), torch.from_numpy(M.indices.astype(np.int32)).to(bl.DEV),
                    torch.from_numpy(M.data.astype(np.float32)).to(bl.DEV))
    return up(R), up(C)


def epoch(m, sampler, n, B):
    def run(mark):
        sampler.epoch()
        u, i, r = sampler.step(n)
        mark("sampler")
        for s in range(0, n, B):
            e = min(s + B, n)
            Uo, Vo = m.user.forward(u[s:e]), m.item.forward(i[s:e])
            mark("towers_fwd")
            dU, dV = torch.empty_like(Uo), torch.empty_like(Vo)
            ops.dmf_head_f32(Uo, Vo, m.F, r[s:e], m.max_ratings, m.cosine, m._loss, dU, dV)
            mark("head")
            m.user.backward(dU, m._grads_of(m.user)); m.item.backward(dV, m._grads_of(m.item))
            mark("towers_bwd")
            m.adam()
            mark("adam")
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = bl.card()
    lines = []
    for shape, make in (("C1", bl.c1_matrix), ("ML-20M", bl.ml20m_matrix)):
        u, i, r, n_users, n_items = make()
        ucsr, icsr = csrs(u, i, r, n_users, n_items)
        T = int(ucsr[1].numel())
        E = T * (1 + NEG)
        srt = ucsr[1]
        sampler = ops.MtPointwiseRatioSampler(n_users, n_items, ucsr[0], srt, ucsr[2], srt, NEG, seed=42)  # sorted rows as the set order: timing only
        for B in (512, E):
            m = DMFModel(n_users, n_items, MLP, MLP, "cosine", float(ucsr[2].max().item()), 1e-4, 42, bl.DEV, ucsr, icsr,
                         min(B, n_users))
            rec = {"model": "DMF", "shape": shape, "users": n_users, "items": n_items, "train": T, "samples_per_epoch": E,
                   "user_mlp": MLP, "item_mlp": MLP, "neg_ratio": NEG, "batch": B, "steps_per_epoch": -(-E // B)}
            need = B * (16 * 2 * sum(MLP) + 64) + E * 12
            if need > torch.cuda.mem_get_info()[0]:
                rec["not_run"] = f"one batch needs ~{need / 2**30:.0f} GiB of tower activations and gradients"
            else:
                steps = min(args.steps, -(-E // B))
                n = min(E, steps * B)
                t = bl.repeat(epoch(m, sampler, n, B), args.iters)
                rec.update({"timed_steps": steps, **{f"{k}_ms": round(v, 2) for k, v in t.items()},
                            "epoch_est_ms": round(sum(t.values()) * (-(-E // B)) / steps, 1)})
                rec.update({f"{k}_ms": round(v, 3)
                            for k, v in bl.repeat(lambda mark: (m.topk(10, ucsr[0], srt), mark("recommend_k10")), args.iters).items()})
                # users of the first score block the tensor-core scorer hands to the exact kernel (ties at the k-th score)
                Uh, Vh, _ = ops.dmf_score_operands_f32(*m.tower_outputs(), m.F, m.block, m.cosine)
                n0 = min(m.block, n_users)
                st = ops.score_topk_tc(Uh, Vh, None, m.F, 10, ucsr[0], srt, user_begin=0, n_sel=n0, stats=True)[2]
                rec.update({"first_block_users": n0, "first_block_rechecked": st["rechecked"]})
            rec.update({"reference": "not timed (TensorFlow is not installed)", "iters": args.iters, **card})
            print(json.dumps(rec), flush=True)
            lines.append(rec)
            del m
            torch.cuda.empty_cache()
        del sampler
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
