"""BASELINE.json configs[0] / north_star "nDCG@10 within 1e-4 of the reference on the same seed", at C1 scale, through
the YAML path (VERDICT r1 #2): the golden tests/golden/bprmf_c1.npz was minted by the UNMODIFIED reference's own
`elliot.run.run_experiment` (oracle/gen_golden_c1.py) on the ML-1M-shaped synthetic file of elliot_b200/synth_c1.py
(6 040 x 3 706, ~1.0 M ratings, `random_subsampling 0.2`, BPRMF d=64, 10 epochs, seed 42).

  exact mode      : every epoch's nDCG/HR/Precision/Recall equals the reference's (asserted <= 1e-4 as the north_star
                    states; the observed difference is ~1e-12), the stored recommendation lists are item-for-item equal.
  throughput mode : (Hogwild, Philox stream — a different but equally distributed triple sequence) nDCG@10 after the
                    same number of epochs, mean over 3 seeds, within HOGWILD_TOL of the reference's; the tolerance is
                    the measured run-to-run spread of the mode, stated here and in DESIGN.md §5.
With EB_C1_PARITY_JSON=<file> the measured numbers are also written to that file.
"""
import json
import os

import numpy as np
import pytest

from elliot_b200 import synth_c1

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bprmf_c1.npz")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOGWILD_TOL = 0.005          # |mean_seeds nDCG@10(hogwild) - nDCG@10(reference)|, absolute (H100: 0.0006; single seeds <= 0.0031)
OUT = {}


@pytest.fixture(scope="module")
def c1(tmp_path_factory):
    g = dict(np.load(GOLDEN))
    d = tmp_path_factory.mktemp("c1")
    tsv = str(d / "dataset.tsv")
    assert synth_c1.write_tsv(tsv) == int(g["checksum"]), "this numpy draws a different synthetic file than the golden's"
    return g, d, tsv


def _run(d, tsv, g, tag, model_extra="", seed=42):
    from elliot_b200 import run_experiment
    out = d / tag
    os.makedirs(out, exist_ok=True)
    cfg = out / "cfg.yml"
    cfg.write_text(synth_c1.yaml_text(tsv, str(out), "BPRMF", int(g["epochs"]), int(g["factors"]), model_extra=model_extra, seed=seed))
    return run_experiment(str(cfg))[0], out


def _dump():
    path = os.environ.get("EB_C1_PARITY_JSON")           # optional record of the measured numbers; the tree stays untouched
    if path:
        with open(path, "w") as fh:
            json.dump(OUT, fh, indent=1)


def test_c1_exact_mode_reproduces_the_reference_run(c1):
    g, d, tsv = c1
    res, out = _run(d, tsv, g, "exact")
    names = g["metrics"].tolist()
    hist = res["history"]
    assert len(hist) == int(g["epochs"]) == g["per_epoch"].shape[0]
    worst = 0.0
    for ep, row in enumerate(hist):
        for m, want in zip(names, g["per_epoch"][ep]):
            worst = max(worst, abs(row[10][m] - float(want)))
    OUT["exact"] = {"max_abs_metric_diff_over_epochs": worst, "ndcg_per_epoch": [r[10]["nDCG"] for r in hist],
                    "reference_ndcg_per_epoch": g["per_epoch"][:, 0].tolist()}
    _dump()
    assert worst <= 1e-4, worst                                  # north_star tolerance
    assert worst <= 1e-9, worst                                  # what exact mode actually delivers
    # the recommendation file of the same epoch as the golden's, item for item
    suffix = str(g["rec_file"]).rsplit("_it=", 1)[1]
    mine = [f for f in os.listdir(out / "recs") if f.endswith("_it=" + suffix)]
    assert len(mine) == 1 and mine[0] == str(g["rec_file"]), (mine, str(g["rec_file"]))   # same model `name` as the reference's
    rec = np.loadtxt(out / "recs" / mine[0], delimiter="\t")
    sel = np.isin(rec[:, 0].astype(np.int64), np.unique(g["rec_users"]))
    assert np.array_equal(rec[sel, 0].astype(np.int64), g["rec_users"]) and np.array_equal(rec[sel, 1].astype(np.int64), g["rec_items"])
    assert np.abs(rec[sel, 2] - g["rec_scores"]).max() < 1e-9


def test_c1_throughput_mode_reaches_the_reference_ndcg(c1):
    g, d, tsv = c1
    ref = float(g["per_epoch"][-1, 0])
    finals, curves = [], []
    for seed in (42, 43, 44):
        res, _ = _run(d, tsv, g, f"hog{seed}", model_extra="      b200_mode: hogwild\n      b200_batch: 65536\n", seed=seed)
        curves.append([r[10]["nDCG"] for r in res["history"]]); finals.append(curves[-1][-1])
    OUT["hogwild"] = {"reference_final_ndcg": ref, "final_ndcg_per_seed": finals, "mean": float(np.mean(finals)),
                      "abs_diff_of_mean": abs(float(np.mean(finals)) - ref), "curves": curves, "tolerance": HOGWILD_TOL,
                      "b200_batch": 65536}
    _dump()
    assert abs(float(np.mean(finals)) - ref) <= HOGWILD_TOL, (finals, ref)
