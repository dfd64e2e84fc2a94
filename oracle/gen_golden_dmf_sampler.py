"""Goldens of the pointwise ratio sampler (DMF's; dataset/samplers/pointwise_pos_neg_ratio_ratings_sampler.py), made by
running the reference's own `Sampler`, imported by file path (it is pure NumPy):

- tests/golden/dmf_sampler_cases.npz: small seeded rating dicts, explicit (1..5) and binarised ratings, neg_ratio 0, 1
  and 5, two epochs each, drawn through step() at batch sizes that do not divide the epoch.  Per case the rows in the
  order the sampler iterates them (its `_ui_dict`), their ratings, and both epochs' (u, i, r) streams.
- tests/golden/dmf_sampler_c1.npz: the synthetic C1 file (elliot_b200/synth_c1.py) as the dict
  {user - 1: {item - 1: rating}} in file order, neg_ratio 5, two epochs of transactions * 6 samples: per epoch the crc32
  of the u, i and r streams and three windows of 2 000 samples (start, middle, end).

    python oracle/gen_golden_dmf_sampler.py        # $ELLIOT_REFERENCE or ../reference beside the repository
"""
import os
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_golden import OUT, _load  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

SAMPLER = "elliot/dataset/samplers/pointwise_pos_neg_ratio_ratings_sampler.py"
WIN = 2000


def small_dict(seed, n_users, n_items, binary):
    g = np.random.default_rng(seed)
    d = {}
    for u in range(n_users):
        c = int(g.integers(1, n_items // 2))
        its = g.choice(n_items, size=c, replace=False)
        d[u] = {int(i): (1.0 if binary else float(g.integers(1, 6))) for i in its}
    d[0][n_items - 1] = 1.0 if binary else 5.0                        # every item id is some user's
    return d


def run(d, neg_ratio, epochs, batch):
    mod = _load("ref_pw_sampler", SAMPLER)
    s = mod.Sampler(d, None, neg_ratio)
    T = sum(len(v) for v in d.values())
    events = T * (1 + neg_ratio)
    streams = []
    for _ in range(epochs):
        parts = list(s.step(events, batch))
        assert all(len(p[0]) == batch for p in parts[:-1])
        streams.append(tuple(np.concatenate([p[k] for p in parts]) for k in range(3)))
    rows = [list(s._ui_dict[u]) for u in range(len(d))]
    return s, rows, events, streams


def crc(a, dt):
    return zlib.crc32(np.ascontiguousarray(a, dt).tobytes())


def c1_dict():
    u, i, r = synth_c1.rows()
    d = {}
    for a, b, c in zip(u.tolist(), i.tolist(), r.tolist()):
        d.setdefault(a - 1, {})[b - 1] = float(c)
    return {k: d[k] for k in range(len(d))}


def main():
    out = {}
    cases = [("explicit_r0", 1, 0, False, 7), ("explicit_r1", 2, 1, False, 13), ("explicit_r5", 3, 5, False, 50),
             ("binary_r5", 4, 5, True, 33), ("binary_r1", 5, 1, True, 1)]
    names = []
    for name, seed, neg, binary, batch in cases:
        d = small_dict(seed, 40, 60, binary)
        s, rows, events, streams = run(d, neg, 2, batch)
        names.append(name)
        out[f"{name}_meta"] = np.array([len(d), s._nitems, neg, events, batch], np.int64)
        out[f"{name}_indptr"] = np.r_[0, np.cumsum([len(r) for r in rows])].astype(np.int64)
        out[f"{name}_rows"] = np.concatenate(rows).astype(np.int32)
        out[f"{name}_ratings"] = np.array([d[u][i] for u, r in enumerate(rows) for i in r], np.float32)
        for e, (su, si, sr) in enumerate(streams):
            out[f"{name}_e{e}_u"], out[f"{name}_e{e}_i"] = su.astype(np.int32), si.astype(np.int32)
            out[f"{name}_e{e}_r"] = sr.astype(np.float32)
    out["names"] = np.array(names)
    np.savez_compressed(os.path.join(OUT, "dmf_sampler_cases.npz"), **out)

    u, i, r = synth_c1.rows()
    d = c1_dict()
    _, _, events, streams = run(d, 5, 2, 1 << 20)
    c1 = {"checksum": np.int64(synth_c1.checksum(u, i, r)), "events": np.int64(events), "neg_ratio": np.int64(5),
          "starts": np.array([0, events // 2, events - WIN], np.int64)}
    for e, (su, si, sr) in enumerate(streams):
        c1[f"e{e}_crc"] = np.array([crc(su, np.int32), crc(si, np.int32), crc(sr, np.float32)], np.int64)
        for k, s0 in enumerate(c1["starts"]):
            c1[f"e{e}_w{k}"] = np.stack([su[s0:s0 + WIN], si[s0:s0 + WIN], sr[s0:s0 + WIN]]).astype(np.float64)
    np.savez_compressed(os.path.join(OUT, "dmf_sampler_c1.npz"), **c1)
    print("wrote", sorted(out)[:3], "...", events)


if __name__ == "__main__":
    main()
