"""Two-stage sampling: a base sample at the low resolution, then the super-resolution denoiser (``model.SuperResModel``,
guided_diffusion/unet.py:667-681) conditioned on it.

    x_low, x_high = sample_then_upsample(x_T, model, betas, eta, A_funcs, y, sr_model, x_T_sr, config=cfg, cls_fn=cond_fn, seed=7)

Stage 1 is ``ddnm_diffusion`` (``ddnm_plus_diffusion`` when ``sigma_y > 0``) with the base denoiser, optionally classifier-guided.
Stage 2 runs the same DDNM loop with the super-resolution denoiser, ``low_res = x_low`` passed to every step, and the
``SuperResolution(ratio)`` average-pooling operator whose measurement is ``x_low`` itself: the null-space projection keeps the
ratio x ratio average pool of the result equal to the first stage's image, and the denoiser fills in the detail.  Both loops,
the denoisers and the bilinear conditioning run in libddnm_b200.so.
"""
import torch

from .model import SuperResModel
from .operators import SuperResolution
from .sampler import sample_device


def _nearest_up(x, ratio):
    """an image whose ratio x ratio average pool is exactly x"""
    return x.repeat_interleave(ratio, dim=2).repeat_interleave(ratio, dim=3)


def sample_then_upsample(x_T, model, b, eta, A_funcs, y, sr_model, x_T_sr, config=None, sr_config=None, sigma_y=0.0, cls_fn=None,
                         sr_cls_fn=None, sr_eta=None, seed=None, row_offset=0):
    """Returns (x_low, x_high) as CUDA tensors in model space ([-1, 1]).

    x_T, model, b, eta, A_funcs, y, config, sigma_y, cls_fn: the first stage, as for ``ddnm_diffusion`` / ``ddnm_plus_diffusion``.
    sr_model: a ``SuperResModel`` with ``small_size`` = the base model's resolution; x_T_sr: its starting noise [B, 3, R, R].
    sr_config / sr_eta / sr_cls_fn: the second stage's schedule, eta and guidance (default: the first stage's config and eta,
    no guidance; a class-conditional super-resolution model needs a guidance function, as any class-conditional denoiser does
    in these samplers).  seed: library-drawn noise for both stages (the second stage uses seed + 1)."""
    if not isinstance(sr_model, SuperResModel):
        raise TypeError("the second stage needs a ddnm_b200.model.SuperResModel")
    small, large = model.resolution, sr_model.resolution
    if sr_model.small_size != small or large % small:
        raise ValueError(f"super-resolution model maps {sr_model.small_size} -> {large}, the base model samples {small}")
    plus = sigma_y > 0
    x_low, _ = sample_device(x_T, model, b, eta, A_funcs, y, sigma_y, plus, config, cls_fn=cls_fn, seed=seed, row_offset=row_offset)
    ratio = large // small
    op = SuperResolution(3, large, ratio, x_low.device)
    with torch.no_grad():
        y_sr = op.A(_nearest_up(x_low, ratio))
    x_high, _ = sample_device(x_T_sr, sr_model, b, eta if sr_eta is None else sr_eta, op, y_sr, 0.0, False,
                              config if sr_config is None else sr_config, cls_fn=sr_cls_fn,
                              seed=None if seed is None else int(seed) + 1, row_offset=row_offset, low_res=x_low)
    return x_low, x_high
