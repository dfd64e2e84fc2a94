"""elliot_b200 — H100 (sm_90a) core for Elliot's embedding-training hot path.

    from elliot_b200 import run_experiment            # mirrors elliot.run.run_experiment
    from elliot_b200.recommender import BPRMF         # mirrors elliot.recommender.BPRMF

The arithmetic lives in elliot_b200/csrc/*.cu behind the C ABI in include/elliot_b200.h
(loaded with ctypes, see _lib.py); there is no CPU fallback.
"""
__version__ = "0.1.0"


def run_experiment(config_path: str = ""):
    from .run import run_experiment as _run
    return _run(config_path)
