"""RecMixin mirror (elliot/recommender/recommender_utils_mixin.py:9-136): evaluate /
best-epoch bookkeeping / protocol + mask choice / result getters, same semantics."""
import os

import numpy as np


def store_recommendation(recommendations, path=""):
    """user\\titem\\tscore TSV (elliot/utils/write.py:35-44)."""
    with open(path, "w") as out:
        for u, recs in recommendations.items():
            for i, value in recs:
                out.write(f"{u}\t{i}\t{value}\n")


class RecMixin:
    def evaluate(self, it=None, loss=0):
        if it is not None and (it + 1) % self._validation_rate:
            return
        on_device = (getattr(self._params, "b200_eval", "host") == "device" and hasattr(self, "get_recommendations_tensors")
                     and hasattr(self.evaluator, "eval_tensors") and not self._save_recs and not self._negative_sampling)
        self._losses.append(loss)
        counts = None
        if self.evaluator.needs_rank:
            # AUC / GAUC: every relevant item's rank in the whole catalogue, from the model's rank pass once per split;
            # the lists stay top_k
            counts = {w: tuple(t.cpu().numpy() for t in self.get_rank_tensors(*rel))
                      for w, rel in self.evaluator.rank_sets(self._device).items()}
        if on_device:
            # extension: the (users x k) index tensor goes from the scoring kernel straight into the metric
            # kernel; no {user: [(item, score)]} dicts are built (recommender_utils_mixin.py:84-88 / evaluator.py:117-147)
            idx, _ = self.get_recommendations_tensors(self.evaluator.get_needed_recommendations())
            recs = None
            self._results.append(self.evaluator.eval_tensors(idx, rank_counts=counts))
        else:
            recs = self.get_recommendations(self.evaluator.get_needed_recommendations())
            self._results.append(self.evaluator.eval(recs, rank_counts=counts))
        if it is not None:
            self.logger.info(f"Epoch {it + 1}/{self._epochs} loss {loss / (it + 1):.5f}")
        else:
            self.logger.info("Finished")
        if self._save_recs:
            name = f"{self.name}_it={it + 1}.tsv" if it is not None else f"{self.name}.tsv"
            os.makedirs(self._config.path_output_rec_result, exist_ok=True)
            store_recommendation(recs[1], os.path.abspath(os.sep.join([self._config.path_output_rec_result, name])))
        if (len(self._results) - 1) == self.get_best_arg():
            if it is not None:
                self._params.best_iteration = it + 1
            self.best_metric_value = self._results[-1][self._validation_k]["val_results"][self._validation_metric]
            if self._save_weights:
                if hasattr(self, "_model"):
                    self._model.save_weights(self._saving_filepath)
                else:
                    self.logger.warning("Saving weights FAILED. No model to save.")

    def process_protocol(self, k, *args):
        if not self._negative_sampling:
            recs = self.get_single_recommendation(self.get_candidate_mask(), k, *args)
            return recs, recs
        val = self.get_single_recommendation(self.get_candidate_mask(validation=True), k, *args) \
            if hasattr(self._data, "val_dict") else {}
        return val, self.get_single_recommendation(self.get_candidate_mask(), k, *args)

    def get_candidate_mask(self, validation=False):
        if self._negative_sampling:
            return self._data.val_mask if validation else self._data.test_mask
        return self._data.allunrated_mask

    def restore_weights(self):
        try:
            self._model.load_weights(self._saving_filepath)
            self.evaluate()
            return True
        except Exception as ex:
            raise Exception(f"Error in model restoring operation! {ex}")

    def get_loss(self):
        if self._optimize_internal_loss:
            return min(self._losses)
        return -max(r[self._validation_k]["val_results"][self._validation_metric] for r in self._results)

    def get_params(self):
        return self._params.__dict__

    def get_results(self):
        return self._results[self.get_best_arg()]

    def get_best_arg(self):
        if self._optimize_internal_loss:
            return int(np.argmin(self._losses))
        return int(np.argmax([r[self._validation_k]["val_results"][self._validation_metric] for r in self._results]))

    def iterate(self, epochs):
        for iteration in range(epochs):
            if self._early_stopping.stop(self._losses[:], self._results):
                self.logger.info(f"Met Early Stopping conditions: {self._early_stopping}")
                break
            yield iteration
