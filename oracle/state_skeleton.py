"""The structure of an optimizer's or a learning-rate scheduler's state_dict without its numbers, shared by
oracle/make_golden_optim.py and the tests that read its fixture: tensors become "tensor <dtype> <shape>", floats
(Python or numpy) "float", other leaves keep their value; dict keys become strings (JSON)."""
from __future__ import annotations

import numbers

import torch


def skeleton(obj):
    if isinstance(obj, torch.Tensor):
        return f"tensor {str(obj.dtype).removeprefix('torch.')} {list(obj.shape)}"
    if isinstance(obj, dict):
        return {str(k): skeleton(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return [skeleton(v) for v in obj]
    if isinstance(obj, bool) or obj is None or isinstance(obj, str):
        return obj
    if isinstance(obj, numbers.Integral):
        return int(obj)
    if isinstance(obj, numbers.Real):
        return "float"
    return type(obj).__name__
