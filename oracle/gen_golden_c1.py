#!/usr/bin/env python
"""Mint the C1-scale golden (BASELINE.json configs[0]: BPRMF d=64 on an ML-1M-shaped matrix, reference CPU path via
run_experiment, config_files/sample_hello_world.yml:2-10 shape) by running the UNMODIFIED reference end to end:

    elliot.run.run_experiment(<yaml>)   with a `BPRMF:` block (factors 64, 10 epochs, the reference's default
                                        hyper-parameters, seed 42), `strategy: dataset`, `random_subsampling 0.2`

on the synthetic 6 040 x 3 706 / ~1.0 M-rating matrix of elliot_b200/synth_c1.py (MovieLens-1M itself is not shipped and
there is no network).  tensorflow/hyperopt are stubbed for import only (oracle/ref_stubs.py); BPRMF is pure NumPy.
Captured (tests/golden/bprmf_c1.npz): the reference Evaluator's test metrics after EVERY epoch (a pass-through wrapper
around Evaluator.eval records them — the reference only logs them), the recommendation lists the reference stored
(`save_recs`), the dataset checksum.  Build container only (~6 min of CPU); the GPU tests read the .npz.

    python oracle/gen_golden_c1.py [--epochs 10]
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_stubs  # noqa: E402
from elliot_b200 import synth_c1  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden", "bprmf_c1.npz")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--factors", type=int, default=64)
    args = ap.parse_args()
    per_epoch, recs, checksum, dt = ref_stubs.run_c1(
        lambda tsv, d, extra: synth_c1.yaml_text(tsv, d, "BPRMF", args.epochs, args.factors, extra=extra))
    assert recs, "the reference stored no recommendation file"
    name, rec = list(recs.items())[-1]
    kept = ref_stubs.first_users(rec)                               # lists of the first 400 users (by public id)
    np.savez_compressed(OUT, metrics=np.array(ref_stubs.METRICS), per_epoch=np.array(per_epoch), epochs=args.epochs,
                        factors=args.factors, rec_file=name, checksum=np.uint64(checksum), reference_seconds=dt, **kept)
    print(f"wrote {OUT}: {len(per_epoch)} epochs, {len(kept['rec_users'])} rec rows, reference run {dt:.0f} s")


if __name__ == "__main__":
    main()
