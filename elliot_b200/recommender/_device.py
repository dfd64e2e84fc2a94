"""Host glue every device model shares: the device choice, the top-k tensors turned into the reference's
recommendation dicts, the recommendation methods, and the uploads and memory check of the item models."""
import numpy as np
import torch


def cuda_device(params, who, default="cuda:0"):
    """The model's device: the YAML key `b200_device`, else `default`.  Refuses to run without CUDA."""
    if not torch.cuda.is_available():
        raise RuntimeError(f"elliot_b200.{who} needs a CUDA device (there is no CPU fallback)")
    return torch.device(getattr(params, "b200_device", default))


def recs_dict(data, idx, val, first=0, out=None):
    """{public user: [(public item, score), ...]} from top-k tensors whose row r is private user first + r; -1 slots
    are skipped and scores become Python floats of their float64 value.  Adds to `out` when it is given."""
    out = {} if out is None else out
    idx, val = idx.cpu().numpy(), val.cpu().numpy().astype(np.float64)
    items = np.array(data.items, dtype=object)
    for r, u in enumerate(data.users[first:first + idx.shape[0]]):
        ok = idx[r] >= 0
        out[u] = list(zip(items[idx[r][ok]].tolist(), val[r][ok].tolist()))
    return out


class TopKRecs:
    """The recommendation methods of a model whose `_model.topk(k, mask_indptr, mask_indices)` ranks every user.
    Listed before RecMixin in the bases, so that these methods win over the host framework's own."""

    def get_recommendations(self, k: int = 10):
        recs_val, recs_test = self.process_protocol(k)
        return dict(recs_val), dict(recs_test)

    def get_recommendations_tensors(self, k: int = 10):
        """(idx, val) device tensors, rows = private users, -1 padded."""
        return self._model.topk(k, self._indptr, self._sorted_idx)

    def get_single_recommendation(self, mask, k, *args):
        if self._negative_sampling:
            raise NotImplementedError("evaluation-time negative sampling masks are outside this build's hot-path scope")
        return recs_dict(self._data, *self.get_recommendations_tensors(k))


class RankRecs:
    """The AUC / GAUC rank pass of a model whose `_model.rank(rel_indptr, rel_items, mask_indptr, mask_indices)` ranks
    every relevant item in the full lists its `_model.topk` takes the top k of (ops.score_rank on the same tables)."""

    def get_rank_tensors(self, rel_indptr, rel_items):
        """(n_pos, sum_c) int64 device tensors, rows = private users."""
        return self._model.rank(rel_indptr, rel_items, self._indptr, self._sorted_idx)


class PairScoreRecs:
    """The MAE / MSE / RMSE pair pass of a model whose `_model.pair_scores(rel_indptr, rel_items, mask_indptr,
    mask_indices)` scores every relevant item as the full lists its `_model.topk` takes the top k of would (ops.score_pairs_f32
    on the same tables; -inf for a train item)."""

    def get_pair_score_tensors(self, rel_indptr, rel_items):
        """float32 device tensor, one score per entry of the relevant-item CSR."""
        return self._model.pair_scores(rel_indptr, rel_items, self._indptr, self._sorted_idx)


def upload(a, device, dtype):
    """A numpy array on the device as a contiguous tensor of `dtype`, in its stored order."""
    return torch.from_numpy(np.ascontiguousarray(a)).to(device, dtype)


def upload_csr(indptr, indices, data, device):
    """A CSR's parts on the device as (indptr int64, indices int32, data float32), in their stored order."""
    return upload(indptr, device, torch.int64), upload(indices, device, torch.int32), upload(data, device, torch.float32)


def check_free(who, device, need, what):
    """Refuses a model whose peak working set (`need` bytes, described by `what`) exceeds the device's free memory."""
    free = torch.cuda.mem_get_info(device)[0]
    if need > free:
        raise MemoryError(f"{who} needs {need / 2**30:.1f} GiB on {device} at its peak ({what}) and "
                          f"{free / 2**30:.1f} GiB are free")
