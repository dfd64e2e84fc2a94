"""What the device-model tests share: uploads, W and score readbacks, and the C1 end-to-end harness (the synthetic file
checked against a golden's checksum, one run_experiment per evaluation path, and the checks every such run makes)."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from elliot_b200 import ops, synth_c1

DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def to_dev(a, dt=None):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)


def dev_csr(M, sort=True):
    """M as a float32 CSR on the device; `sort=False` keeps the stored column order."""
    M = sp.csr_matrix(M, dtype=np.float32)
    if sort:
        M.sort_indices()
    return to_dev(M.indptr, torch.int64), to_dev(M.indices, torch.int32), to_dev(M.data, torch.float32)


def w_host(W, n):
    p, i, v = (a.cpu().numpy() for a in W)
    return sp.csr_matrix((v, i, p), shape=(n, n))


def all_scores(A, W, n):
    """Every column's score of every row of A . W, read back from a top-n call without a mask."""
    idx, val = ops.rp3_score_topk(A, W, n, n)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    P = np.zeros((idx.shape[0], n), np.float32)
    np.put_along_axis(P, idx.astype(np.int64), val, 1)
    assert np.all(np.sort(idx, 1) == np.arange(n)[None, :])
    return P


# ---------------------------------------------------------------- run_experiment at C1 scale
def c1_fixture(golden):
    """A module fixture giving (the arrays of tests/golden/`golden`, a fresh directory, the C1 file written in it); the
    file must have the checksum the golden was minted on."""
    @pytest.fixture(scope="module")
    def c1(tmp_path_factory):
        g = dict(np.load(os.path.join(GOLD, golden)))
        d = tmp_path_factory.mktemp(golden.split(".")[0])
        tsv = str(d / "dataset.tsv")
        assert synth_c1.write_tsv(tsv) == int(g["checksum"]), "this numpy draws a different synthetic file than the golden's"
        return g, d, tsv
    return c1


def run(out, text, device_eval=False):
    """run_experiment on the YAML `text` (its output paths under `out`), written to out/cfg.yml; returns its first
    result.  Device evaluation computes the metrics straight from the top-k tensor, without rec dicts, so it runs with
    save_recs off."""
    from elliot_b200 import run_experiment
    os.makedirs(out, exist_ok=True)
    if device_eval:
        text = text.replace("save_recs: True", "save_recs: False")
    (out / "cfg.yml").write_text(text)
    return run_experiment(str(out / "cfg.yml"))[0]


def assert_no_rec_files(out):
    assert not os.path.exists(out / "recs") or not os.listdir(out / "recs")


def assert_metrics(res, names, want, *what):
    """Every metric within 1e-4 of the reference's: `want` holds one value per name for the final test results, or one
    such row per epoch for res["history"]."""
    want = np.asarray(want, dtype=np.float64)
    got = [res["test_results"]] if want.ndim == 1 else res["history"]
    rows = want.reshape(-1, len(names))
    assert len(got) == len(rows), (*what, len(got), len(rows))
    for e, (r, w) in enumerate(zip(got, rows)):
        for m, v in zip(names, w):
            assert abs(r[10][m] - v) <= 1e-4, (*what, e, m, r[10][m], v)
