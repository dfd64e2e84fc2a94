"""TEST INFRASTRUCTURE (build container only): make the unmodified reference package importable where its third-party
dependencies tensorflow==2.3.2 and hyperopt are absent.

`elliot/recommender/__init__.py:12-25` imports every model eagerly and `elliot/run.py:15` imports hyperopt, so without
them nothing of the reference — not even the pure-NumPy BPRMF — can be driven through `elliot.run.run_experiment`.
`install()` puts a meta-path finder in front that serves permissive stub modules for exactly those packages (any
attribute is a subclassable, callable dummy) and puts the original project (REF) on sys.path.  Nothing of the reference is stubbed
or modified; code paths that would really call TensorFlow/hyperopt (the TF models, hyper-parameter search) stay out of
reach and are never used by the generators/tests that call this.

Also provides a logging config equivalent to elliot/config/logger_config.yml without its `queue: cfg://objects.queue`
handler, which Python >= 3.12's logging.config rejects (the reference targets Python 3.6-3.8); the reference reads it
through its own `path_logger_config` key.
"""
import abc
import importlib.abc
import importlib.machinery
import os
import sys
import types

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
