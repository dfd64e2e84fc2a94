"""The clustered fairness metrics on the GPU: ops.eval_fairness against the host mirror (fairness.host_fairness_sums) on
the goldens and on random lists (users= subsets, ld > k, zero rows, every user skipped), per-user nDCG bits against
eb_eval_topk_f64, bit-identical reruns, Evaluator.eval_tensors against the reference's values, the C1 MostPop
run_experiment against the reference's performance table under both evaluation paths (and unchanged other metrics and
rec files), and BPRMF exact mode giving the same fairness values through the dict and the device paths."""
import os
import shutil

import numpy as np
import pandas as pd
import pytest
import torch

import c1_harness as c1h
from c1_harness import DEV, to_dev
from elliot_b200 import fairness, ops, synth_c1
from elliot_b200.evaluation import ideal_dcg
from fairness_cases import CASES, GOLD, assert_matches, case_evaluator, fairness_part, write_file

pytestmark = pytest.mark.gpu


def device_pass(ev, which, k, key, idx, scores=None, users=None):
    ucl, nu, icl, ni = ev._clusterings(key)
    has_rows, u_d, i_d = ev._fair_device(which, key, idx.device)
    c, s = ops.eval_fairness(idx, k, *ev._device_set(which, k, idx.device), has_rows, u_d, nu, i_d, ni,
                             scores=scores, users=users)
    return c.cpu().numpy(), s.cpu().numpy()


def host_pass(ev, which, k, key, idx, scores, priv):
    ucl, nu, icl, ni = ev._clusterings(key)
    cs = ev._sets[which]
    return fairness.host_fairness_sums(priv, idx, scores, k, cs, ideal_dcg(cs, k), ev._has_rows(which), ucl, nu, icl, ni)


def assert_same(dev, host, what):
    np.testing.assert_array_equal(dev[0], host[0], err_msg=str(what))
    d, h = dev[1], host[1]
    np.testing.assert_array_equal(np.isnan(d), np.isnan(h), err_msg=str(what))
    ok = ~np.isnan(h)
    np.testing.assert_allclose(d[ok], h[ok], rtol=1e-12, atol=1e-15, err_msg=str(what))


@pytest.mark.parametrize("case", sorted(CASES))
def test_device_pass_equals_host_mirror_on_goldens(case, tmp_path):
    g, data, ev = case_evaluator(case, tmp_path)
    idx_h, sc_h = g["rec_idx"], g["rec_scores"]
    idx, sc = to_dev(idx_h, torch.int32), to_dev(sc_h, torch.float32)   # fp32 scores are cast once, exactly
    for which in ("val", "test"):
        for k in g["cutoffs"].tolist():
            for key in {e.launch for e in ev._complex}:
                dev = device_pass(ev, which, k, key, idx, sc)
                host = host_pass(ev, which, k, key, idx_h, sc_h.astype(np.float32), np.arange(data.num_users))
                assert_same(dev, host, (case, which, k, key))
                again = device_pass(ev, which, k, key, idx, sc)
                assert np.array_equal(dev[0], again[0]) and dev[1].tobytes() == again[1].tobytes()   # bit-identical


def test_random_lists_subsets_wide_rows_zero_rows_and_skipped_users(tmp_path):
    g, data, ev = case_evaluator("d", tmp_path)                      # 300 item clusters: global histograms
    rng = np.random.default_rng(5)
    n_users, n_items = data.num_users, data.num_items
    for k, ld in ((7, 7), (20, 33), (40, 40)):
        idx_h = rng.integers(0, n_items, size=(n_users, ld)).astype(np.int64)
        cut = rng.integers(0, ld + 1, size=n_users)
        idx_h[np.arange(ld)[None, :] >= cut[:, None]] = -1
        sc_h = rng.normal(size=(n_users, ld))
        users = rng.permutation(n_users)[: n_users // 3]
        idx = to_dev(idx_h, torch.int32)
        for key in {e.launch for e in ev._complex}:
            assert_same(device_pass(ev, "test", min(k, ld), key, idx, to_dev(sc_h)),
                        host_pass(ev, "test", min(k, ld), key, idx_h, sc_h, np.arange(n_users)), ("all", k, ld))
            sub = to_dev(idx_h[users], torch.int32)
            assert_same(device_pass(ev, "test", min(k, ld), key, sub, to_dev(sc_h[users]),
                                    users=to_dev(users, torch.int32)),
                        host_pass(ev, "test", min(k, ld), key, idx_h[users], sc_h[users], users), ("users", k, ld))
    key = ev._complex[-1].launch
    empty = torch.empty((0, 10), dtype=torch.int32, device=DEV)
    c, s = device_pass(ev, "test", 10, key, empty)
    assert not c.any() and not s.any()
    ev._fair_dev[("test", key, str(torch.device(DEV)))] = (torch.zeros(n_users, dtype=torch.uint8, device=DEV),
                                                           *ev._fair_device("test", key, DEV)[1:])
    c, s = device_pass(ev, "test", 10, key, to_dev(g["rec_idx"], torch.int32), to_dev(g["rec_scores"]))
    assert not c.any() and not s.any()                               # no user with test rows: nothing counted


def test_per_user_ndcg_has_the_bits_of_eval_topk(tmp_path):
    g, data, ev = case_evaluator("a", tmp_path)
    n_users = data.num_users
    idx = to_dev(g["rec_idx"], torch.int32)
    own = to_dev(np.arange(n_users), torch.int32)                    # one cluster per user: its sum is its nDCG
    none = torch.full((data.num_items,), -1, dtype=torch.int32, device=DEV)
    has_rows = to_dev(ev._has_rows("test"), torch.uint8)
    for k in (1, 5, 10, 20):
        ds = ev._device_set("test", k, DEV)
        c, s = ops.eval_fairness(idx, k, *ds, has_rows, own, n_users, none, 1)
        _, pu = ops.eval_topk(idx, k, *ds, per_user=True)
        want = pu[:, 0].cpu().numpy()
        counted = c.cpu().numpy()[:n_users] == 1
        assert counted.any() and np.array_equal(counted, ~np.isnan(want) & ev._has_rows("test"))
        assert s.cpu().numpy()[:n_users][counted].tobytes() == want[counted].tobytes(), k


@pytest.mark.parametrize("case", sorted(CASES))
def test_eval_tensors_equals_the_reference(case, tmp_path):
    g, data, ev = case_evaluator(case, tmp_path)
    idx = to_dev(g["rec_idx"], torch.int32)
    if ev.needs_scores:
        with pytest.raises(Exception, match="MADrating"):
            ev.eval_tensors(idx)
    res = ev.eval_tensors(idx, vals=to_dev(g["rec_scores"]))
    for c, k in enumerate(g["cutoffs"].tolist()):
        for s, split in enumerate(("val_results", "test_results")):
            assert_matches(fairness_part(res[k][split]), g["keys"], g["values"][c, s], (case, k, split))


# ---------------------------------------------------------------- run_experiment at C1 scale
c1 = c1h.c1_fixture("fairness_c1.npz")


def c1_dirs(g, d, name):
    """d/name/cfg for the config, with the clustering files in d/name/data/movielens_1m and d/name/data/c1_synth."""
    root = d / name
    for sub in ("movielens_1m", "c1_synth"):
        os.makedirs(root / "data" / sub, exist_ok=True)
        write_file(str(root / "data" / sub / "u_happy.tsv"), g["u_happy"][:, 0], g["u_happy"][:, 1])
        write_file(str(root / "data" / sub / "i_pop.tsv"), g["i_pop"][:, 0], g["i_pop"][:, 1])
    return root / "cfg"


@pytest.mark.parametrize("ev", ["host", "device"])
def test_c1_mostpop_run_gives_the_reference_table(c1, ev):
    from oracle.gen_golden_fairness import RUN_CUTOFFS, run_yaml
    g, d, tsv = c1
    out = c1_dirs(g, d, f"run_{ev}")
    text = run_yaml(tsv, str(out)).replace("      meta:\n", f"      b200_eval: {ev}\n      meta:\n", 1)
    c1h.run(out, text, device_eval=ev == "device")
    for k in RUN_CUTOFFS:
        got = pd.read_csv(out / "performance" / f"rec_cutoff_{k}.tsv", sep="\t")
        assert list(got.columns) == g[f"run_columns_{k}"].tolist()
        assert got.iloc[:, 0].astype(str).tolist() == g[f"run_models_{k}"].tolist()
        # a MAD is a difference of cluster averages, so the summation order of the device's sums (not the reference's
        # dict order) shows up to ~1e-12 relative in it at C1
        assert_matches(dict(zip(got.columns[1:], got.iloc[0, 1:].to_numpy(np.float64))), got.columns[1:],
                       g[f"run_values_{k}"][0], ("c1 run", ev, k), rtol=1e-11)
    if ev == "host":                                                 # the complex entries change nothing else
        plain = d / "plain" / "cfg"
        text = synth_c1.experiment_yaml(tsv, str(plain), "MostPop", "", metrics=("nDCG", "HR"), cutoffs=RUN_CUTOFFS)
        c1h.run(plain, text)
        for k in RUN_CUTOFFS:
            want = pd.read_csv(plain / "performance" / f"rec_cutoff_{k}.tsv", sep="\t")
            got = pd.read_csv(out / "performance" / f"rec_cutoff_{k}.tsv", sep="\t")
            assert got[["nDCG", "HR"]].equals(want[["nDCG", "HR"]])
        assert (plain / "recs" / "MostPop.tsv").read_bytes() == (out / "recs" / "MostPop.tsv").read_bytes()


def test_c1_bprmf_exact_same_fairness_through_dict_and_device(c1):
    g, d, tsv = c1
    from oracle.gen_golden_fairness import run_entries
    vals = {}
    for ev in ("host", "device"):
        out = c1_dirs(g, d, f"bpr_{ev}")
        text = synth_c1.experiment_yaml(tsv, str(out), "BPRMF", "      epochs: 1\n      factors: 16\n      seed: 42\n",
                                        meta=("save_recs: False", "verbose: False"), metrics=("nDCG",), cutoffs=(5, 10),
                                        complex_metrics=run_entries(), model_extra=f"      b200_eval: {ev}\n")
        vals[ev] = c1h.run(out, text)["test_results"]
    for k in (5, 10):
        keys = list(vals["host"][k])
        assert len(keys) == 39                                       # nDCG and the nine metrics' 38 keys
        # the MADs are differences of cluster averages summed in different orders on the two paths (see the MostPop run)
        assert_matches(vals["device"][k], keys, [vals["host"][k][m] for m in keys], ("bprmf", k), rtol=1e-10)
    shutil.rmtree(d / "bpr_host", ignore_errors=True)
