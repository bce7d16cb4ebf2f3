"""Module parameters and buffers as views of one flat vector.

Every kernel of this package reads and writes flat fp32 / int32 vectors (parameters, Adam moments, RunningNorm and
EMANorm statistics), while the reference-facing modules stay ordinary `nn.Module`s: their tensors are views of those
vectors, so `state_dict()` shows what the kernels wrote, `load_state_dict()` writes into the memory they read, a torch
optimiser steps the same storage, and a captured CUDA graph stays valid as long as the vectors keep their addresses.
"""
import math
from typing import List, Optional, Sequence, Tuple

import torch as th
from torch import nn


def contiguous_view(tensors: Sequence[th.Tensor], dtype: th.dtype, device: th.device) -> Optional[th.Tensor]:
    """The flat vector `tensors` already form, if every one has `dtype`, sits on `device`, is contiguous, shares the
    first tensor's storage and follows the previous one back to back; else None."""
    t0 = tensors[0]
    total = 0
    for t in tensors:
        if (t.dtype != dtype or t.device != device or not t.is_contiguous()
                or t.untyped_storage().data_ptr() != t0.untyped_storage().data_ptr()
                or t.data_ptr() != t0.data_ptr() + t0.element_size() * total):
            return None
        total += t.numel()
    return t0.detach().as_strided((total,), (1,), t0.storage_offset())


def views(flat: th.Tensor, shapes: Sequence[Sequence[int]]) -> List[th.Tensor]:
    """Consecutive slices of `flat`, reshaped to `shapes`."""
    out, off = [], 0
    for s in shapes:
        k = math.prod(s)
        out.append(flat[off:off + k].view(s))
        off += k
    return out


class FlatAlias:
    """Keeps an ordered list of slots (a module and the name of one of its parameters or buffers) views of one flat
    vector.  A parameter is re-pointed through `.data`, so the `Parameter` object, and any optimiser holding it,
    survives; a buffer is replaced in the module's buffer table."""

    def __init__(self, slots: Sequence[Tuple[nn.Module, str]]):
        self._slots = [(m._parameters if name in m._parameters else m._buffers, name) for m, name in slots]
        self._key: Optional[tuple] = None
        self._flat: Optional[th.Tensor] = None

    def tensors(self) -> List[th.Tensor]:
        return [table[name] for table, name in self._slots]

    def _signature(self, dtype: th.dtype, device: th.device) -> tuple:
        return (dtype, device, *[table[name].data_ptr() for table, name in self._slots])

    def get(self, dtype: th.dtype, device: th.device) -> th.Tensor:
        """The flat `dtype` vector on `device` that the slots view.  When no slot was re-pointed since the last call
        this returns the same tensor; otherwise it adopts the vector the slots already form, or copies their values
        into a new one and re-points every slot to its slice.  `device` is a concrete device (`cuda:0`, not `cuda`)."""
        if self._signature(dtype, device) == self._key:
            return self._flat
        ts = self.tensors()
        flat = contiguous_view(ts, dtype, device)
        if flat is None:
            flat = th.cat([t.detach().reshape(-1).to(device=device, dtype=dtype) for t in ts])
            for (table, name), p, v in zip(self._slots, ts, views(flat, [t.shape for t in ts])):
                if isinstance(p, nn.Parameter):
                    p.data = v
                else:
                    table[name] = v
        self._flat = flat
        self._key = self._signature(dtype, device)
        return flat
