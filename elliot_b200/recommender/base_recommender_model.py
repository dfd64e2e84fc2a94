"""Host-side mirror of the reference's model boundary
(elliot/recommender/base_recommender_model.py:27-163): same constructor contract
`Model(data=, config=, params=)`, same meta/base keys and defaults, same `_params_list`
6-tuples + `autoset_params()`, same `@init_charger` side effects (seeding order, evaluator,
name, weight folder).  When the reference package itself is importable (a real Elliot
install) elliot_b200.recommender binds to ITS base classes instead — see _bases.py."""
import inspect
import logging
import os
import random
from abc import ABC, abstractmethod
from functools import wraps
from types import SimpleNamespace

import numpy as np

from .early_stopping import EarlyStopping


def _logger(name, level=logging.INFO):
    lg = logging.getLogger(f"elliot_b200.{name}")
    lg.setLevel(level)
    return lg


class BaseRecommenderModel(ABC):
    def __init__(self, data, config, params, *args, **kwargs):
        self._data, self._config, self._params = data, config, params
        self._negative_sampling = hasattr(data.config, "negative_sampling")
        meta = getattr(params, "meta", SimpleNamespace())
        self._restore = getattr(meta, "restore", False)
        ev = data.config.evaluation
        cut = getattr(ev, "cutoffs", [data.config.top_k])
        cut = cut if isinstance(cut, list) else [cut]
        first = ev.simple_metrics[0] if ev.simple_metrics else ""
        vm = getattr(meta, "validation_metric", f"{first}@{cut[0]}").split("@")
        if vm[0].lower() not in [m.lower() for m in ev.simple_metrics]:
            raise Exception("Validation metric must be in the list of simple metrics")
        self._validation_k = int(vm[1]) if len(vm) > 1 else cut[0]
        if self._validation_k not in cut:
            raise Exception("Validation cutoff must be in general cutoff values")
        self._validation_metric = vm[0]
        self._save_weights = getattr(meta, "save_weights", False)
        self._save_recs = getattr(meta, "save_recs", False)
        self._verbose = getattr(meta, "verbose", None)
        self._validation_rate = getattr(meta, "validation_rate", 1)
        self._optimize_internal_loss = getattr(meta, "optimize_internal_loss", False)
        self._epochs = int(getattr(params, "epochs", 2))
        self._seed = getattr(params, "seed", 42)
        self._early_stopping = EarlyStopping(SimpleNamespace(**getattr(params, "early_stopping", {})),
                                             self._validation_metric, self._validation_k, cut, ev.simple_metrics)
        self._iteration = 0
        if self._epochs < self._validation_rate:
            raise Exception(f"The first validation epoch ({self._validation_rate}) "
                            f"is later than the overall number of epochs ({self._epochs}).")
        self._batch_size = getattr(params, "batch_size", -1)
        self.best_metric_value = 0
        self._losses, self._results, self._params_list = [], [], []

    def get_base_params_shortcut(self):
        return "_".join(f"{k}={str(v).replace('.', '$')}" for k, v in
                        (("seed", self._seed), ("e", self._epochs), ("bs", self._batch_size)))

    def get_params_shortcut(self):
        return "_".join(f"{p[2]}={str(p[5](getattr(self, p[0])) if p[5] else getattr(self, p[0])).replace('.', '$')}"
                        for p in self._params_list)

    def autoset_params(self):
        """(attribute, yaml key, shortcut, default, reader, printer) tuples -> attributes."""
        for attr, key, _, default, reader, _ in self._params_list:
            raw = getattr(self._params, key, default)
            setattr(self, attr, raw if reader is None else reader(raw))
            self.logger.info(f"Parameter {key} set to {getattr(self, attr)}")

    @abstractmethod
    def train(self): ...

    @abstractmethod
    def get_recommendations(self, *args): ...

    @abstractmethod
    def get_loss(self): ...

    @abstractmethod
    def get_params(self): ...

    @abstractmethod
    def get_results(self): ...


def init_charger(init):
    """Constructor wrapper with the reference's order of side effects
    (base_recommender_model.py:142-163): base init -> logger -> seed numpy and random with the
    model seed -> model init -> evaluator -> name -> weight folder."""
    @wraps(init)
    def new_init(self, *args, **kwargs):
        BaseRecommenderModel.__init__(self, *args, **kwargs)
        pkg = inspect.getmodule(self).__package__ or ""
        rec_name = f"external.{self.__class__.__name__}" if "external" in pkg else self.__class__.__name__
        self.logger = _logger(rec_name, logging.CRITICAL if getattr(self._config, "config_test", False) else logging.INFO)
        np.random.seed(self._seed)
        random.seed(self._seed)
        self._nprandom, self._random = np.random, random
        self._num_items, self._num_users = self._data.num_items, self._data.num_users
        from ..evaluation import RANK, Evaluator
        asked = [m for m in self._data.config.evaluation.simple_metrics if m.upper() in RANK]
        if asked and not hasattr(self, "get_rank_tensors"):
            raise Exception(f"{self.__class__.__name__} cannot evaluate {'/'.join(asked)}: these rank every relevant "
                            f"item in the whole catalogue, and only the factor models that list with score_topk have "
                            f"that rank pass; this model's scores come from a different scorer, which would need its own")
        init(self, *args, **kwargs)
        # AUC / GAUC come from this model's rank pass (checked above); other configs build the evaluator as before
        self.evaluator = Evaluator(self._data, self._params, rank_pass=True) if asked else Evaluator(self._data, self._params)
        self._params.name = self.name
        wdir = os.path.abspath(os.sep.join([self._config.path_output_rec_weight, self.name]))
        os.makedirs(wdir, exist_ok=True)
        self._saving_filepath = os.path.join(wdir, f"best-weights-{self.name}")
    return new_init
