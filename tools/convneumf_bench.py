"""Time ConvNeuMF through the model's own code (recommender/convneumf.py's ConvNeuMFModel) at the reference's defaults
(embedding_size 100, cnn_channels (1, 32, 32), kernels and strides 2): the C1 shape (synth_c1's 6 040 x 3 706 file) and
the ML-20M shape (benchlib's seeded 138 493 x 26 744 matrix), every rating a train transaction.

- Training, batch 512: `--steps` steps split into their phases (the sampler's draw of the epoch, the gradient pass, the
  Keras Adam pass), the median of benchlib.repeat over `--iters` runs after one warm-up, and the epoch extrapolated from
  them (steps per epoch x the per-step time, plus one sampler call): an extrapolation, labelled as one.
- Scoring at C1: the fused scorer over every user and item, top-10 of every user (scoring + dense top-k) and the AUC / GAUC
  rank pass (scoring + dense rank) over 20 % of each user's items as the relevant set.
- Scoring at ML-20M: the fused scorer over a slice of `--ml20m-users` users, and the whole evaluation extrapolated from it.

Beside the measurements each line carries the computed bounds (not measured): per pair, 2 R_1 c_1 level-1 FMAs on the
CUDA cores at the data sheet's 67 TFLOP/s fp32 and sum_l R_l 4 c_(l-1) c_l MACs on the tensor cores at its 989 TFLOP/s
bf16 dense, times the pairs of a full evaluation; and the materialised alternative's traffic (level 1 written once to HBM
in bf16, at 3.35 TB/s).  The reference's TensorFlow arm is not timed: TensorFlow is not installed where this runs.
Prints one JSON line per shape, with the card, its power limit and clocks.

    python tools/convneumf_bench.py [--iters 3] [--steps 50] [--ml20m-users 2048] [--out results/convneumf_bench.json]
"""
import argparse
import json
import os

import numpy as np
import torch

import benchlib as bl
from elliot_b200 import ops
from elliot_b200.recommender.convneumf import ConvNeuMFModel

F, WIDTHS, B = 100, [32, 32], 512
FP32_FMA_PER_S = 67e12 / 2
BF16_MAC_PER_S = 989e12 / 2
HBM_BYTES_PER_S = 3.35e12


def bounds(m, pairs):
    """Computed per-pair work and the least time of `pairs` pairs at the data sheet's rates (not measured)."""
    fma1 = 2 * m.R[1] * m.c[1]
    macs = sum(m.R[l] * 4 * m.c[l - 1] * m.c[l] for l in range(2, m.L + 1))
    l1_ns, tc_ns = fma1 / FP32_FMA_PER_S * 1e9, macs / BF16_MAC_PER_S * 1e9
    hbm = 2 * m.R[1] * m.c[1] * pairs
    return {"level1_values_per_pair": m.R[1] * m.c[1], "level1_fma_per_pair": fma1, "tc_macs_per_pair": macs,
            "bound_level1_ns_per_pair": round(l1_ns, 2), "bound_tc_ns_per_pair": round(tc_ns, 2),
            "bound_eval_s": round(max(l1_ns, tc_ns) * pairs * 1e-9, 3),
            "materialised_level1_bytes": hbm, "materialised_level1_s_at_hbm_peak": round(hbm / HBM_BYTES_PER_S, 2),
            "bounds_note": "computed from the data sheet's rates, not measured"}


def train_phases(m, sampler, T, steps):
    def run(mark):
        tu, ti, tj = sampler.step(T)
        mark("sampler")
        for s in range(0, steps * B, B):
            m.grads(tu[s:s + B], ti[s:s + B], tj[s:s + B])
            mark("grads")
            m.adam()
            mark("adam")
    return run


def rel_sets(indptr, srt, n_users):
    """20 % of each user's train items as the relevant set (the rank pass's work depends on their number only)."""
    ip, ix = indptr.cpu().numpy(), srt.cpu().numpy()
    rows = [ix[ip[u]:ip[u + 1]][::5] for u in range(n_users)]
    rp = np.zeros(n_users + 1, np.int64); rp[1:] = np.cumsum([len(r) for r in rows])
    return torch.from_numpy(rp).to(bl.DEV), torch.from_numpy(np.concatenate(rows).astype(np.int32)).to(bl.DEV)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--ml20m-users", type=int, default=2048)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = bl.card()
    lines = []
    for shape, make in (("C1", bl.c1_matrix), ("ML-20M", bl.ml20m_matrix)):
        u, i, _, n_users, n_items = make()
        indptr, srt = bl.train_mask(u, i, n_users)
        T = int(srt.numel())
        m = ConvNeuMFModel(n_users, n_items, F, 1e-3, WIDTHS, 0.0, 0.005, 0.0005, 42, bl.DEV)
        sampler = ops.MtSampler(n_users, n_items, indptr, srt, srt, seed=42)       # sorted rows as the set order: timing only
        steps = min(args.steps, T // B)
        t = bl.repeat(train_phases(m, sampler, T, steps), args.iters)
        per_step = (t["grads"] + t["adam"]) / steps
        n_steps = -(-T // B)
        rec = {"model": "ConvNeuMF", "shape": shape, "users": n_users, "items": n_items, "train": T, "embedding_size": F,
               "cnn_channels": [1] + WIDTHS, "batch": B, "timed_steps": steps,
               "step_grads_ms": round(t["grads"] / steps, 3), "step_adam_ms": round(t["adam"] / steps, 3),
               "sampler_epoch_ms": round(t["sampler"], 2),
               "epoch_ms_extrapolated": round(t["sampler"] + per_step * n_steps, 1),
               "epoch_note": f"{steps} timed steps x {n_steps} steps per epoch + one sampler call: an extrapolation"}
        if shape == "C1":
            pairs = n_users * n_items
            rp, ri = rel_sets(indptr, srt, n_users)
            sc = bl.repeat(lambda mark: ([m.scores(u0, u1) for u0, u1 in m._blocks()], mark("score_all")), args.iters)
            tk = bl.repeat(lambda mark: (m.topk(10, indptr, srt), mark("recommend_k10")), args.iters)
            rk = bl.repeat(lambda mark: (m.rank(rp, ri, indptr, srt), mark("rank_pass")), args.iters)
            s1 = m.scores(0, min(n_users, 256)); s2 = m.scores(0, min(n_users, 256))
            rec.update({"score_all_ms": round(sc["score_all"], 2), "recommend_k10_ms": round(tk["recommend_k10"], 2),
                        "rank_pass_ms": round(rk["rank_pass"], 2), "scorer_ns_per_pair": round(sc["score_all"] * 1e6 / pairs, 3),
                        "scorer_rerun_bit_identical": bool(torch.equal(s1, s2))})
        else:
            nu = min(args.ml20m_users, n_users)
            pairs = n_users * n_items
            sc = bl.repeat(lambda mark: (m.scores(0, nu), mark("score_slice")), args.iters)
            rec.update({"score_users": nu, "score_slice_ms": round(sc["score_slice"], 2),
                        "scorer_ns_per_pair": round(sc["score_slice"] * 1e6 / (nu * n_items), 3),
                        "score_all_s_extrapolated": round(sc["score_slice"] * 1e-3 * n_users / nu, 2),
                        "score_all_note": f"{nu} users timed, scaled to {n_users}: an extrapolation"})
        rec.update(bounds(m, pairs))
        rec.update({"reference": "not timed (TensorFlow is not installed)", "iters": args.iters, **card})
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del m, sampler
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()
