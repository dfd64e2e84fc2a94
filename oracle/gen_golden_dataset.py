#!/usr/bin/env python
"""Mint tests/golden/dataset_views.npz from the ORIGINAL project's own DataSet and BPRMF (needs a checkout of it, see REF in
oracle/ref_stubs.py; tensorflow / hyperopt are import stubs, nothing of the reference is modified).

On a small seeded (train, test) frame it records what the reference's `elliot.dataset.dataset.DataSet` exposes — the user /
item id orders and the train / test CSR views the kernels read (`train_csr_of`, `eval_csr_of`) — and the model `name` the
reference's BPRMF builds for a fixed parameter set.  tests/test_dataset_golden.py compares elliot_b200's mirror with them.

    python oracle/gen_golden_dataset.py
"""
import logging
import os
import sys
import tempfile
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_stubs  # noqa: E402

PARAMS = dict(epochs=2, factors=8, lr=0.05, seed=42, batch_size=512, user_regularization=0.0025)
PARAMS_LIST = [("_factors", "factors", "f", 10, int, None), ("_learning_rate", "lr", "lr", 0.05, None, None),
               ("_bias_regularization", "bias_regularization", "bias_reg", 0, None, None),
               ("_user_regularization", "user_regularization", "u_reg", 0.0025, None, None),
               ("_positive_item_regularization", "positive_item_regularization", "pos_i_reg", 0.0025, None, None),
               ("_negative_item_regularization", "negative_item_regularization", "neg_i_reg", 0.00025, None, None),
               ("_update_negative_item_factors", "update_negative_item_factors", "up_neg_i_f", True, None, None),
               ("_update_users", "update_users", "up_u", True, None, None), ("_update_items", "update_items", "up_i", True, None, None),
               ("_update_bias", "update_bias", "up_b", True, None, None)]


def frames():
    import pandas as pd
    g = np.random.default_rng(3)
    rows = sorted({(int(10 + 3 * g.integers(60)), int(100 + 7 * g.integers(40))) for _ in range(900)})
    g.shuffle(rows)
    tr = pd.DataFrame({"userId": [r[0] for r in rows[:700]], "itemId": [r[1] for r in rows[:700]], "rating": 1.0})
    keep = set(tr.userId)
    te_rows = [r for r in rows[700:] if r[0] in keep]
    te = pd.DataFrame({"userId": [r[0] for r in te_rows], "itemId": [r[1] for r in te_rows], "rating": 1.0})
    return tr, te


def config():
    tmp = tempfile.mkdtemp()
    return SimpleNamespace(config_test=True, align_side_with_train=False, top_k=10, path_output_rec_weight=tmp,
                           path_output_rec_result=tmp, path_output_rec_performance=tmp,
                           evaluation=SimpleNamespace(simple_metrics=["nDCG", "HR"], relevance_threshold=0, paired_ttest=False,
                                                      wilcoxon_test=False, cutoffs=[10]))


def params():
    return SimpleNamespace(meta=SimpleNamespace(save_recs=False, verbose=False), **PARAMS)


def main():
    ref_stubs.install()
    logging.disable(logging.CRITICAL)
    import elliot.dataset.dataset as ref_ds
    from elliot.recommender.base_recommender_model import BaseRecommenderModel as RefBase
    from elliot.recommender.latent_factor_models.BPRMF.BPRMF import BPRMF as RefBPRMF
    from elliot_b200.dataset import eval_csr_of, train_csr_of
    cfg = config()
    data = ref_ds.DataSet(cfg, frames(), SimpleNamespace())
    ip, ix = (np.asarray(x) for x in train_csr_of(data, "cpu")[:2])
    eip, eix = (np.asarray(x) for x in eval_csr_of(data, "test")[:2])

    class Probe(RefBPRMF):
        def __init__(self):
            pass
    p = Probe()
    RefBase.__init__(p, data, cfg, params())
    p.logger = logging.getLogger("probe")
    p._params_list = PARAMS_LIST
    p.autoset_params()
    out = os.path.join(ROOT, "tests", "golden", "dataset_views.npz")
    np.savez_compressed(out, users=np.array(data.users, np.int64), items=np.array(data.items, np.int64),
                        train_indptr=ip.astype(np.int64), train_indices=ix.astype(np.int32),
                        test_indptr=eip.astype(np.int64), test_indices=eix.astype(np.int32), name=np.array(p.name))
    print("wrote", out, p.name)


if __name__ == "__main__":
    main()
