"""TEST INFRASTRUCTURE (build container only): make the unmodified reference package importable where its third-party
dependencies tensorflow==2.3.2 and hyperopt are absent.

`elliot/recommender/__init__.py:12-25` imports every model eagerly and `elliot/run.py:15` imports hyperopt, so without
them nothing of the reference — not even the pure-NumPy BPRMF — can be driven through `elliot.run.run_experiment`.
`install()` puts a meta-path finder in front that serves permissive stub modules for exactly those packages (any
attribute is a subclassable, callable dummy) and puts the original project (REF) on sys.path.  Nothing of the reference is stubbed
or modified; code paths that would really call TensorFlow/hyperopt (the TF models, hyper-parameter search) stay out of
reach and are never used by the generators/tests that call this.

`run_c1()` runs the reference's `run_experiment` on the C1 synthetic file and returns what the goldens record.

Also provides a logging config equivalent to elliot/config/logger_config.yml without its `queue: cfg://objects.queue`
handler, which Python >= 3.12's logging.config rejects (the reference targets Python 3.6-3.8); the reference reads it
through its own `path_logger_config` key.
"""
import abc
import glob
import importlib.abc
import importlib.machinery
import importlib.util
import os
import shutil
import sys
import tempfile
import time
import types

import numpy as np

# a checkout of the original Elliot project: $ELLIOT_REFERENCE, or a directory named `reference` beside this repository
REF = os.environ.get("ELLIOT_REFERENCE") or os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "reference")
STUBBED = ("tensorflow", "hyperopt", "tensorflow_probability")


class _Meta(abc.ABCMeta):
    def __getattr__(cls, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return cls


class Stub(metaclass=_Meta):
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return self

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return Stub


class _StubModule(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return Stub


class _Finder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path, target=None):
        if fullname.split(".")[0] in STUBBED:
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _StubModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


def available():
    return os.path.isdir(REF)


def install():
    if not any(isinstance(f, _Finder) for f in sys.meta_path):
        sys.meta_path.insert(0, _Finder())
    if REF not in sys.path:
        sys.path.insert(0, REF)


LOGGER_NAMES = ["recommender", "DataSet", "DataSetLoader", "Evaluator", "namespace", "ModelCoordinator", "prefiltering",
                "splitter", "result_handler", "EarlyStopping", "__main__"]


def write_logger_config(path):
    body = ("version: 1\nformatters:\n  simple:\n    format: '%(time_filter)-15s: %(levelname)-.1s %(message)s'\n"
            "filters:\n  time_filter:\n    (): elliot.utils.logging.TimeFilter\n"
            "handlers:\n  console:\n    class: logging.StreamHandler\n    level: FATAL\n    formatter: simple\n"
            "    stream: ext://sys.stdout\n    filters: [time_filter]\n"
            "  file:\n    class: logging.FileHandler\n    level: FATAL\n    filename: !CUSTOM ${log_path_exp}\n"
            "    formatter: simple\n    filters: [time_filter]\n"
            "loggers:\n" + "".join(f"  '{n}':\n    level: FATAL\n    handlers: [console, file]\n    propagate: false\n"
                                    for n in LOGGER_NAMES)
            + "root:\n  level: FATAL\n  handlers: [console]\n")
    with open(path, "w") as fh:
        fh.write(body)
    return path


METRICS = ["nDCG", "HR", "Precision", "Recall"]


def load(path, name):
    """Import one reference file by its path, as module `name`."""
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_c1(make_yaml):
    """elliot.run.run_experiment on `make_yaml(tsv, out_dir, extra=...)` over the C1 synthetic file of
    elliot_b200/synth_c1.py, in a temporary directory.  Returns (the test METRICS of every evaluation in order, {rec file
    name: its rows} sorted by name, the file's checksum, the wall time of the run).  A pass-through wrapper around
    Evaluator.eval records the metrics, which the reference only logs."""
    from elliot_b200 import synth_c1
    install()
    tmp = tempfile.mkdtemp(prefix="c1_golden_")
    try:
        tsv = os.path.join(tmp, "dataset.tsv")
        checksum = synth_c1.write_tsv(tsv)
        logcfg = write_logger_config(os.path.join(tmp, "logger_config.yml"))
        cfg = os.path.join(tmp, "cfg.yml")
        with open(cfg, "w") as fh:
            fh.write(make_yaml(tsv, tmp, extra=f"  path_logger_config: {logcfg}\n"))
        from elliot.evaluation.evaluator import Evaluator
        from elliot.run import run_experiment
        evals = []
        orig_eval = Evaluator.eval

        def recording_eval(self, recommendations):       # pass-through: records what the reference computed
            res = orig_eval(self, recommendations)
            k = list(res.keys())[0]
            evals.append([float(res[k]["test_results"][m]) for m in METRICS])
            print(f"evaluation {len(evals)}: " + " ".join(f"{m}={v:.6f}" for m, v in zip(METRICS, evals[-1])), flush=True)
            return res
        Evaluator.eval = recording_eval
        try:
            t0 = time.time()
            run_experiment(cfg)
            dt = time.time() - t0
        finally:
            Evaluator.eval = orig_eval
        recs = {os.path.basename(f): np.loadtxt(f, delimiter="\t")
                for f in sorted(glob.glob(os.path.join(tmp, "recs", "*.tsv")))}
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return evals, recs, checksum, dt


def first_users(rec, keep=400):
    """The rows of the first `keep` users (by public id) of a rec file: rec_users, rec_items, rec_scores, and
    n_rec_users, the number of users in the file."""
    users = np.unique(rec[:, 0].astype(np.int64))
    sel = np.isin(rec[:, 0].astype(np.int64), users[:keep])
    return {"rec_users": rec[sel, 0].astype(np.int64), "rec_items": rec[sel, 1].astype(np.int64),
            "rec_scores": rec[sel, 2], "n_rec_users": len(users)}
