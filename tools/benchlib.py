"""What the model benchmarks under tools/ share: the card they ran on, the two data sets, a data shim with the DataSet
fields the device models read, the train mask, and a phase timer driven by the models' own `mark(phase)` hooks."""
import os
import subprocess
import sys

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from elliot_b200 import synth_c1  # noqa: E402
from elliot_b200.recommender._device import upload  # noqa: E402

DEV = "cuda:0"


def card():
    """The GPU's name, power limit and SM clocks (read-only nvidia-smi queries): a number measured on it needs them."""
    out = {"gpu": torch.cuda.get_device_properties(0).name}
    for key, q in (("power_limit_w", "power.limit"), ("sm_clock_mhz", "clocks.sm"), ("sm_clock_max_mhz", "clocks.max.sm")):
        try:
            out[key] = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                                      capture_output=True, text=True).stdout.strip()
        except OSError:
            out[key] = "not read"
    return out


def c1_matrix():
    """Every rating of elliot_b200/synth_c1.py's file: (users, items, ratings 1-5, 6 040, 3 706), ~1.0 M ratings."""
    u, i, r = synth_c1.rows()
    return u - 1, i - 1, r.astype(np.float32), synth_c1.N_USERS, synth_c1.N_ITEMS


def ml20m_matrix(seed=20):
    """138 493 x 26 744 with ~18.4 M distinct half-star ratings (20 M draws before duplicate (user, item) pairs are
    dropped; popularity capped at ML-20M's largest item count, 67 310), generated from a seed."""
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


class Data:
    """The DataSet fields the device models read, from distinct (user, item, rating) triples; public ids are private
    ids.  `_tr` holds the triples grouped by user, the form dict_order_csr takes."""

    def __init__(self, u, i, r, U, I):
        self.sp_i_train_ratings = sp.csr_matrix((r, (u, i)), shape=(U, I), dtype=np.float32)
        self.sp_i_train = sp.csr_matrix((np.ones(len(u), np.float32), (u, i)), shape=(U, I), dtype=np.float32)
        self.users, self.items = range(U), range(I)
        self.num_users, self.num_items = U, I
        o = np.argsort(u, kind="stable")
        self._tr = (u[o].astype(np.int64), i[o].astype(np.int64), r[o].astype(np.float64))


def train_mask(u, i, U):
    """The train items of every user as a CSR on the device, (indptr int64, indices int32) with each row sorted."""
    indptr = np.zeros(U + 1, np.int64)
    np.cumsum(np.bincount(u, minlength=U), out=indptr[1:])
    return upload(indptr, DEV, torch.int64), upload(i[np.lexsort((i, u))], DEV, torch.int32)


def reference_seconds(golden):
    """The reference's C1 run time stored in tests/golden/<golden> when it was minted (not measured in this run)."""
    g = np.load(os.path.join(ROOT, "tests", "golden", golden))
    return {"value": float(g["reference_seconds"]),
            "note": "whole reference run_experiment on one host core, minted with the golden, not this run"}


def repeat(fn, n, seconds=False):
    """Runs fn(mark) once to warm up, then n times, and returns each phase's median over the n runs, in milliseconds
    (seconds if `seconds`).  Each run starts on an idle device; `mark(phase)` records a CUDA event, the interval since the
    previous event is charged to `phase`, and a phase marked more than once in a run adds up."""
    def once():
        marks = []

        def mark(phase):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            marks.append((phase, e))
        torch.cuda.synchronize()
        mark(None)
        fn(mark)
        torch.cuda.synchronize()
        t = {}
        for (_, a), (phase, b) in zip(marks, marks[1:]):
            t[phase] = t.get(phase, 0.0) + a.elapsed_time(b)
        return t
    once()
    runs = [once() for _ in range(n)]
    scale = 1e-3 if seconds else 1.0
    return {k: float(np.median([r[k] for r in runs])) * scale for k in runs[0]}
