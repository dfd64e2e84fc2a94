"""The DataSet mirror and the model name against the ORIGINAL project's own DataSet and BPRMF, through data they produced
(tests/golden/dataset_views.npz, minted by oracle/gen_golden_dataset.py on a small seeded frame): user / item id orders,
the train CSR in the reference's set order, the test CSR, and the BPRMF `name` for a fixed parameter set."""
import logging
import os

import numpy as np

from oracle.gen_golden_dataset import PARAMS_LIST, config, frames, params

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dataset_views.npz")


def test_dataset_views_equal_the_reference_dataset():
    from elliot_b200.dataset import DataSet, eval_csr_of, train_csr_of
    g = np.load(GOLDEN)
    mirror = DataSet(config(), frames())
    assert list(mirror.users) == g["users"].tolist() and list(mirror.items) == g["items"].tolist()
    ip, ix = (np.asarray(x) for x in train_csr_of(mirror, "cpu")[:2])
    assert np.array_equal(ip, g["train_indptr"]) and np.array_equal(ix, g["train_indices"])
    eip, eix = (np.asarray(x) for x in eval_csr_of(mirror, "test")[:2])
    assert np.array_equal(eip, g["test_indptr"]) and np.array_equal(eix, g["test_indices"])


def test_bprmf_name_equals_the_reference_name():
    from elliot_b200.dataset import DataSet
    from elliot_b200.recommender._bases import BaseRecommenderModel
    from elliot_b200.recommender.bprmf import BPRMF
    g = np.load(GOLDEN)
    cfg = config()
    data = DataSet(cfg, frames())

    class Probe(BPRMF):
        def __init__(self):
            pass
    p = Probe()
    BaseRecommenderModel.__init__(p, data, cfg, params())
    p.logger = logging.getLogger("probe")
    p._params_list = PARAMS_LIST
    p.autoset_params()
    assert p.name == str(g["name"])
