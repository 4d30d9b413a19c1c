"""The library's seeded Gaussian draws as tensors (``ddnm_noise_fill``).

One value is a pure function of ``(seed, tag, draw, global image row, element index)`` (include/ddnm_b200.h, "Seeded noise"),
so ``randn(seed, (8, ...), tag)[4:]`` equals ``randn(seed, (4, ...), tag, row_offset=4)``.  This is how a caller of the seeded
samplers gets ``x_T`` (``TAG_XT``) and the measurement noise of ``--add_noise`` (``TAG_Y``); the samplers' own per-pair draws
(``TAG_LOOP``, draw = pair index) are produced inside the step kernels and only materialised here for comparisons.
"""
import ctypes as C

import torch

from . import _lib

TAG_LOOP, TAG_XT, TAG_Y, TAG_HQ, TAG_DEQUANT = 0, 1, 2, 3, 4


def randn(seed, shape, tag, draw=0, row_offset=0, device="cuda"):
    """float32 CUDA tensor of ``shape`` = (rows, ...): row b holds the draws of global image row ``row_offset + b``."""
    shape = tuple(int(d) for d in shape)
    if len(shape) < 2 or min(shape) < 1:
        raise ValueError("shape must be (rows, ...) with every extent >= 1")
    out = torch.empty(shape, device=device, dtype=torch.float32)
    ns = _lib.noise_seed(seed, row_offset)
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().ddnm_noise_fill(C.byref(ns), int(tag), int(draw), _lib.ptr(out), shape[0], out[0].numel(),
                                              _lib.cur_stream()))
    return out
