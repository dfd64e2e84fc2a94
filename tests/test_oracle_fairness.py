"""CPU tests of the clustered fairness metrics (elliot_b200/fairness.py): the host mirror through Evaluator.eval against
what the unmodified reference Evaluator computed on the same lists (tests/golden/fairness_*.npz), the complex_metrics
block through build_base_config, and the entries refused at construction."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

from elliot_b200.dataset import DataSet
from fairness_cases import (CASES, GOLD, as_recs, assert_matches, case_evaluator, config, fairness_part, frame,
                            write_file)


@pytest.mark.parametrize("case", sorted(CASES))
def test_host_mirror_equals_reference_evaluator(case, tmp_path):
    g, data, ev = case_evaluator(case, tmp_path)
    recs = as_recs(data, g["rec_idx"], g["rec_scores"])
    res = ev.eval((recs, recs))
    for c, k in enumerate(g["cutoffs"].tolist()):
        for s, split in enumerate(("val_results", "test_results")):
            assert list(res[k][split])[0] == "nDCG"                       # simple metrics first
            assert_matches(fairness_part(res[k][split]), g["keys"], g["values"][c, s], (case, k, split))


def test_oracle_equals_reference_evaluator(tmp_path):
    from oracle import fairness as oracle
    for case in sorted(CASES):
        (tmp_path / case).mkdir()
        g, data, ev = case_evaluator(case, tmp_path / case)
        recs = as_recs(data, g["rec_idx"], g["rec_scores"])
        for c, k in enumerate(g["cutoffs"].tolist()):
            want = g["values"][c, 1]
            got = oracle.evaluate(data, recs, data.test_dict, k, data.config.evaluation.complex_metrics)
            assert_matches(got, g["keys"], want, (case, k))


def test_host_mirror_equals_reference_at_c1(tmp_path):
    from elliot_b200 import synth_c1
    from elliot_b200.evaluation import Evaluator
    from elliot_b200.run import _read, split_random_subsampling
    from oracle.gen_golden_fairness import c1_lists, crc
    import json
    g = np.load(os.path.join(GOLD, "fairness_c1.npz"))
    tsv = str(tmp_path / "dataset.tsv")
    assert synth_c1.write_tsv(tsv) == int(g["checksum"])
    (train, test), = split_random_subsampling(_read(tsv, False), 0.2, 42)
    uf = write_file(str(tmp_path / "u_happy.tsv"), g["u_happy"][:, 0], g["u_happy"][:, 1])
    itf = write_file(str(tmp_path / "i_pop.tsv"), g["i_pop"][:, 0], g["i_pop"][:, 1])
    entries = json.loads(str(g["entries"]).replace("{ufile}", uf).replace("{ifile}", itf))
    data = DataSet(config(int(g["top_k"]), g["cutoffs"].tolist(), 0, entries), (train, test))
    assert data.users == g["users"].tolist() and data.items == g["items"].tolist()
    ev = Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))
    recs, rec_idx, rec_scores = c1_lists(data, int(g["top_k"]))      # the golden's lists, redrawn from the dataset
    assert crc(rec_idx) == int(g["rec_idx_crc"]) and crc(rec_scores) == int(g["rec_scores_crc"])
    res = ev.eval((recs, recs))
    for c, k in enumerate(g["cutoffs"].tolist()):
        assert_matches(fairness_part(res[k]["test_results"]), g["keys"], g["values"][c], ("c1", k))


def test_build_base_config_resolves_paths_as_the_reference(tmp_path):
    from elliot_b200.run import build_base_config
    cfg_dir = tmp_path / "cfg"
    cfg_dir.mkdir()
    cfg = cfg_dir / "exp.yml"
    cfg.write_text(f"""experiment:
  dataset: ml
  data_config:
    strategy: dataset
    dataset_path: ../data/{{0}}/dataset.tsv
  top_k: 10
  evaluation:
    simple_metrics: [nDCG]
    complex_metrics:
    - metric: UserMADrating
      clustering_name: Happiness
      clustering_file: ../data/{{0}}/u_happy.tsv
    - metric: REO
      clustering_name: i_pop.tsv
      clustering_file: {tmp_path}/x/../i_pop.tsv
      other: ./here
      plain: name
      number: 3
      digit_first: 1a.b
  path_output_rec_result: {tmp_path}/out/recs
  path_output_rec_weight: {tmp_path}/out/weights
  path_output_rec_performance: {tmp_path}/out/performance
  models: {{}}
""")
    base, _ = build_base_config(str(cfg))
    a, b = base.evaluation.complex_metrics
    assert a == {"metric": "UserMADrating", "clustering_name": "Happiness",
                 "clustering_file": str(tmp_path / "data" / "ml" / "u_happy.tsv")}
    assert b == {"metric": "REO", "clustering_name": str(cfg_dir / "i_pop.tsv"),      # looks like a file name
                 "clustering_file": str(tmp_path / "i_pop.tsv"), "other": str(cfg_dir / "here"), "plain": "name",
                 "number": 3, "digit_first": "1a.b"}
    cfg.write_text(cfg.read_text().replace("    complex_metrics:", "    unused:"))
    assert build_base_config(str(cfg))[0].evaluation.complex_metrics == []


@pytest.mark.parametrize("name", ["DSC", "ExtendedF1", "ExtendedEPC", "ExtendedPopREO", "SRecall", "NoSuchMetric"])
def test_unsupported_complex_names_raise(name, tmp_path):
    g = CASES["a"]
    with pytest.raises(Exception, match=f"metric {name} is not available"):
        DataSet_and_eval(g, [{"metric": name}])


def DataSet_and_eval(g, entries, simple=("nDCG",)):
    from elliot_b200.evaluation import Evaluator
    data = DataSet(config(int(g["top_k"]), g["cutoffs"].tolist(), float(g["thr"]), entries, simple),
                   (frame(g["train"]), frame(g["val"]), frame(g["test"])))
    return Evaluator(data, SimpleNamespace(meta=SimpleNamespace()))


@pytest.mark.parametrize("labels", [[0, 2, 2], [1, 2, 1], [-1, 0, 1], [0.0, 1.5, 1.0]])
def test_labels_outside_0_to_n_minus_1_raise(labels, tmp_path):
    g = CASES["a"]
    path = write_file(str(tmp_path / "c.tsv"), [7, 10, 13], labels)
    with pytest.raises(Exception, match="labels must be the integers"):
        DataSet_and_eval(g, [{"metric": "UserMADranking", "clustering_name": "x", "clustering_file": path}])


def test_duplicate_ids_raise(tmp_path):
    g = CASES["a"]
    path = write_file(str(tmp_path / "d.tsv"), [1000, 1005, 1000], [0, 1, 1])
    with pytest.raises(Exception, match="listed more than once"):
        DataSet_and_eval(g, [{"metric": "REO", "clustering_name": "x", "clustering_file": path}])


def test_without_complex_metrics_results_are_unchanged(tmp_path):
    g, data, ev = case_evaluator("a", tmp_path, simple=("nDCG", "HR", "MAP", "Gini"))
    plain = DataSet_and_eval(g, [], simple=("nDCG", "HR", "MAP", "Gini"))
    recs = as_recs(data, g["rec_idx"], g["rec_scores"])
    a, b = ev.eval((recs, recs)), plain.eval((recs, recs))
    for k in a:
        for split in ("val_results", "test_results"):
            assert {m: a[k][split][m] for m in b[k][split]} == b[k][split]
            assert list(a[k][split])[:4] == ["nDCG", "HR", "MAP", "Gini"]
