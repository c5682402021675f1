"""Outputs the quantizer modules make: on the input's device."""
from __future__ import annotations

import torch


def empty_like_rows(x: torch.Tensor, shape, dtype) -> torch.Tensor:
    """An output on x's device (pinned when x is pinned, so the library streams both the same way)."""
    if x.is_cuda:
        return torch.empty(shape, dtype=dtype, device=x.device)
    return torch.empty(shape, dtype=dtype, pin_memory=x.is_pinned())
