"""Synthetic data generator (no model arithmetic): the MovieLens-1M-SHAPED interaction file used for BASELINE.json configs[0]
(sample_hello_world.yml:2-10 names data/movielens_1m/dataset.tsv, which is not shipped and cannot be downloaded here).

6 040 users x 3 706 items, ~1.0 M ratings: per-user counts from a clipped log-normal (min 20 like ML-1M's filter), items
drawn without replacement from a Zipf-like popularity, ratings 1..5, rows shuffled, `user\\titem\\trating\\ttimestamp`
like the reference's loader expects (dataset.py:75-80).  Deterministic for a given numpy; the checksum of the rows is
stored in the golden so that a different numpy stream fails loudly instead of silently changing the data.
"""
import zlib

import numpy as np

N_USERS, N_ITEMS, SEED = 6040, 3706, 20240924


def rows(seed=SEED):
    g = np.random.default_rng(seed)
    pop = 1.0 / np.arange(1, N_ITEMS + 1) ** 0.9
    pop /= pop.sum()
    counts = np.clip(g.lognormal(np.log(110.0), 0.95, N_USERS), 20, 2300).astype(np.int64)
    us, its = [], []
    for u in range(N_USERS):
        c = int(counts[u])
        it = g.choice(N_ITEMS, size=c, replace=False, p=pop)
        us.append(np.full(c, u + 1, np.int64)); its.append(it.astype(np.int64) + 1)
    u = np.concatenate(us); i = np.concatenate(its)
    r = g.integers(1, 6, size=u.size).astype(np.int64)
    perm = g.permutation(u.size)
    return u[perm], i[perm], r[perm]


def checksum(u, i, r):
    return zlib.crc32(np.stack([u, i, r], 1).astype(np.int64).tobytes())


def write_tsv(path, seed=SEED):
    u, i, r = rows(seed)
    with open(path, "w") as fh:
        fh.write("".join(f"{a}\t{b}\t{float(c)}\t{t}\n" for t, (a, b, c) in enumerate(zip(u.tolist(), i.tolist(), r.tolist()))))
    return checksum(u, i, r)


def experiment_yaml(tsv, out_dir, model_key, block, meta=("save_recs: True",), extra="", model_extra="",
                    metrics=("nDCG", "HR", "Precision", "Recall")):
    """The reference's YAML layout (sample_hello_world.yml:1-19) over the C1 file above: one `model_key` block with the
    given `meta` lines (without indentation) and parameter lines (`block`, indented, newline-ended), evaluated with
    `metrics`.  `extra` goes into the experiment section, `model_extra` after the model's parameters."""
    meta = "".join(f"        {m}\n" for m in meta)
    return f"""experiment:
  dataset: c1_synth
  data_config:
    strategy: dataset
    dataset_path: {tsv}
  splitting:
    test_splitting:
      strategy: random_subsampling
      test_ratio: 0.2
  top_k: 10
  evaluation:
    simple_metrics: [{', '.join(metrics)}]
  path_output_rec_result: {out_dir}/recs
  path_output_rec_weight: {out_dir}/weights
  path_output_rec_performance: {out_dir}/performance
  path_log_folder: {out_dir}/log
{extra}  models:
    {model_key}:
      meta:
{meta}{block}{model_extra}"""


def hello_world_yaml(tsv, out_dir, extra="", model_extra=""):
    """config_files/sample_hello_world.yml's ItemKNN block (neighbors 50, cosine, save_recs)."""
    return experiment_yaml(tsv, out_dir, "ItemKNN", "      neighbors: 50\n      similarity: cosine\n", extra=extra,
                           model_extra=model_extra)


def als_yaml(tsv, out_dir, model_key, epochs, block, extra="", model_extra=""):
    """An iALS or WRMF block (`block`: its parameter lines, e.g. factors / alpha / reg) with save_recs."""
    return experiment_yaml(tsv, out_dir, model_key, f"      epochs: {epochs}\n{block}", extra=extra,
                           model_extra=model_extra)


def ease_yaml(tsv, out_dir, extra="", model_extra=""):
    """An EASER block with the reference's defaults (neighborhood -1, l2_norm 1e3) and save_recs."""
    return experiment_yaml(tsv, out_dir, "EASER", "", extra=extra, model_extra=model_extra)


def rp3beta_yaml(tsv, out_dir, extra="", model_extra=""):
    """config_files/recsys_config.yml's RP3beta block (neighborhood 546, alpha 1.0807, beta 0.7029, normalize_similarity
    True) with save_recs."""
    return experiment_yaml(tsv, out_dir, "RP3beta", "      neighborhood: 546\n      alpha: 1.0807\n      beta: 0.7029\n"
                           "      normalize_similarity: True\n", extra=extra, model_extra=model_extra)


def slim_yaml(tsv, out_dir, extra="", model_extra=""):
    """config_files/recsys_config.yml's Slim block (l1_ratio 0.0000119, alpha 0.0788, neighborhood 544) with
    save_recs."""
    return experiment_yaml(tsv, out_dir, "Slim", "      l1_ratio: 0.0000119\n      alpha: 0.0788\n      neighborhood: 544\n",
                           extra=extra, model_extra=model_extra)


def pure_svd_yaml(tsv, out_dir, extra="", model_extra=""):
    """The PureSVD block of the reference's docstring (factors 10, seed 42) with save_recs."""
    return experiment_yaml(tsv, out_dir, "PureSVD", "      factors: 10\n      seed: 42\n", extra=extra,
                           model_extra=model_extra)


def slope_one_yaml(tsv, out_dir, extra="", model_extra=""):
    """The SlopeOne block of the reference's docstring (no parameters) with save_recs."""
    return experiment_yaml(tsv, out_dir, "SlopeOne", "", extra=extra, model_extra=model_extra)


def nonneg_mf_yaml(tsv, out_dir, extra="", model_extra=""):
    """The NonNegMF block of the reference's docstring (epochs 10, batch_size 512, factors 10, lr 0.001, reg 0.1) with
    save_recs."""
    return experiment_yaml(tsv, out_dir, "NonNegMF", "      epochs: 10\n      batch_size: 512\n      factors: 10\n"
                           "      lr: 0.001\n      reg: 0.1\n", extra=extra, model_extra=model_extra)


def yaml_text(tsv, out_dir, model_key, epochs, factors, extra="", model_extra="", seed=42, save_recs=True,
              metrics=("nDCG", "HR", "Precision", "Recall")):
    """A `BPRMF:` block with BPRMF.py:43-56 keys, the reference's default hyper-parameters, save_recs (unless
    save_recs=False) and verbose off, evaluated with `metrics`."""
    return experiment_yaml(tsv, out_dir, model_key, f"""      epochs: {epochs}
      factors: {factors}
      lr: 0.05
      bias_regularization: 0
      user_regularization: 0.0025
      positive_item_regularization: 0.0025
      negative_item_regularization: 0.00025
      seed: {seed}
""", meta=(f"save_recs: {save_recs}", "verbose: False"), extra=extra, model_extra=model_extra, metrics=metrics)
