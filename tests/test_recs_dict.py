"""recs_dict: the top-k tensors of the device models turned into the reference's {public user: [(public item, score)]}
recommendation dicts, on CPU tensors."""
import numpy as np
import torch

from elliot_b200.recommender._device import recs_dict


class _Data:
    users = ["u7", "u3", "u9", "u1"]           # private user r is users[r]
    items = [40, 10, 30]                       # private item j is items[j]


IDX = torch.tensor([[2, 0, -1], [-1, -1, -1], [1, 2, 0], [0, -1, -1]], dtype=torch.int32)
VAL = torch.tensor([[0.1, -2.5, float("-inf")], [float("-inf")] * 3, [3.0, 1e-3, 0.0], [7.25, float("-inf"), float("-inf")]],
                   dtype=torch.float32)


def test_public_ids_padding_and_float64_scores():
    out = recs_dict(_Data, IDX, VAL)
    f = lambda x: float(np.float32(x))
    assert out == {"u7": [(30, f(0.1)), (40, -2.5)], "u3": [], "u9": [(10, 3.0), (30, f(1e-3)), (40, 0.0)],
                   "u1": [(40, 7.25)]}
    assert all(type(s) is float and type(i) is int for recs in out.values() for i, s in recs)
    assert out["u7"][0][1] != 0.1                # the float64 value of the float32 score, not a rounded decimal


def test_blocks_with_a_first_row_add_to_one_dict():
    out = recs_dict(_Data, IDX[:2], VAL[:2])
    again = recs_dict(_Data, IDX[2:], VAL[2:], first=2, out=out)
    assert again is out
    assert out == recs_dict(_Data, IDX, VAL)
    assert list(out) == ["u7", "u3", "u9", "u1"]


def test_float64_scores_pass_unchanged():
    val = VAL.double() + 1e-12
    out = recs_dict(_Data, IDX, val)
    assert out["u9"][1] == (30, float(val[2, 1]))
