"""Sorted key/value helpers: parallel sort and ordered key matching.

Capability parity with the reference's (unused) ``include/ps/internal/parallel_sort.h:23-55``,
``parallel_kv_match.h:29-120`` and ``assign_op.h:12-68``: sort a key array, and for two ascending key lists
combine the values of the keys present in both (``dst[k] op= src[k]``). The reference forks threads recursively;
here both are data-parallel tensor programs that run on whichever device the tensors live on (a GPU sorts
and matches keys far faster than hand-threaded host code).
"""
from __future__ import annotations

from typing import Callable, Dict, Tuple

import torch

ASSIGN, PLUS, MINUS, TIMES, DIVIDE, AND, OR, XOR = range(8)

_OPS: Dict[int, Callable[[torch.Tensor, torch.Tensor], torch.Tensor]] = {
    ASSIGN: lambda d, s: s,
    PLUS: lambda d, s: d + s,
    MINUS: lambda d, s: d - s,
    TIMES: lambda d, s: d * s,
    DIVIDE: lambda d, s: d / s,
    AND: lambda d, s: d & s,
    OR: lambda d, s: d | s,
    XOR: lambda d, s: d ^ s,
}


def parallel_sort(keys: torch.Tensor, descending: bool = False) -> torch.Tensor:
    """In-place sort of a 1-D tensor (radix sort on CUDA tensors); returns the tensor."""
    keys.copy_(torch.sort(keys, descending=descending).values)
    return keys


def sort_by_key(keys: torch.Tensor, vals: torch.Tensor, k: int = 1) -> Tuple[torch.Tensor, torch.Tensor]:
    """Sorts (keys, vals) by key; ``vals`` holds ``k`` values per key."""
    order = torch.argsort(keys, stable=True)
    return keys[order], vals.view(-1, k)[order].reshape(-1)


def parallel_ordered_match(src_keys: torch.Tensor, src_vals: torch.Tensor, dst_keys: torch.Tensor,
                           dst_vals: torch.Tensor, k: int = 1, op: int = ASSIGN) -> int:
    """For every key present in both ascending, duplicate-free key lists: ``dst_vals[key] op= src_vals[key]``
    (``k`` values per key). Returns the number of matched values (matched keys * k), like the reference."""
    if src_keys.numel() == 0 or dst_keys.numel() == 0:
        return 0
    assert src_vals.numel() == src_keys.numel() * k and dst_vals.numel() == dst_keys.numel() * k
    pos = torch.searchsorted(dst_keys, src_keys)
    pos_c = pos.clamp(max=dst_keys.numel() - 1)
    hit = dst_keys[pos_c] == src_keys
    di = pos_c[hit]
    d = dst_vals.view(-1, k)
    s = src_vals.view(-1, k)[hit]
    d[di] = _OPS[op](d[di], s)
    return int(hit.sum()) * k
