"""The runner's per-batch body either side of the sampling loop (guided_diffusion/diffusion.py:533-603), on the device.

``data_transform`` / ``inverse_data_transform`` keep the signatures of datasets/__init__.py:201-227; ``restore_batch`` is the
body of ``Diffusion.svd_based_ddnm_plus``'s loop: transform -> y = A(x) (+ noise) -> A^+ y previews -> x_T -> DDNM / DDNM+ ->
inverse transform, PNG bytes and PSNR.  The restored batch never visits the host as fp32: one fused pass
(``ddnm_finish_images``) produces the uint8 HWC bytes a PNG encoder wants plus the per-image PSNRs, so the D2H traffic is
196 KB + 4 B per image instead of the reference's 786 KB x 2 (``x`` and ``x0_pred``) + one blocking copy back per image
for the PSNR (diffusion.py:600).  Everything numeric runs in libddnm_b200.so; there is no CPU fallback.
"""
import os
import struct
import zlib

import numpy as np
import torch

from . import _lib
from .noise import TAG_XT, TAG_Y, randn
from .sampler import sample_device


def _flags(config):
    if hasattr(config, "image_mean"):
        raise NotImplementedError("config.image_mean is set by no shipped config and is not supported")
    return int(bool(config.data.rescaled)), int(bool(config.data.logit_transform))


def _cuda_f32(X):
    assert X.is_cuda, "ddnm_b200.runner works on CUDA tensors"
    return X.float().contiguous()


def data_transform(config, X, uniform_noise=None, gauss_noise=None):
    """datasets/__init__.py:201-213.  The dequantisation draws come from the current CUDA generator in the reference's
    order (rand_like, then randn_like) unless passed in."""
    X = _cuda_f32(X)
    rescaled, logit = _flags(config)
    if config.data.uniform_dequantization and uniform_noise is None:
        uniform_noise = torch.rand_like(X)
    if config.data.gaussian_dequantization and gauss_noise is None:
        gauss_noise = torch.randn_like(X)
    un = _cuda_f32(uniform_noise) if uniform_noise is not None else None
    gn = _cuda_f32(gauss_noise) if gauss_noise is not None else None
    out = torch.empty_like(X)
    _lib.check(_lib.lib().ddnm_data_transform(_lib.ptr(X), X.numel(), _lib.ptr(un), _lib.ptr(gn), rescaled, logit, _lib.ptr(out),
                                             _lib.cur_stream()))
    return out


def inverse_data_transform(config, X):
    """datasets/__init__.py:216-227."""
    X = _cuda_f32(X)
    rescaled, logit = _flags(config)
    out = torch.empty_like(X)
    _lib.check(_lib.lib().ddnm_inverse_data_transform(_lib.ptr(X), X.numel(), rescaled, logit, _lib.ptr(out), _lib.cur_stream()))
    return out


def get_gaussian_noisy_img(img, noise_level):
    """guided_diffusion/diffusion.py:21-22."""
    return img + torch.randn_like(img) * noise_level


def finish_images(config, x, x_orig=None, want_float=False):
    """One fused pass over model-space images ``x`` (B,C,H,W): returns ``(u8, psnr, x01)`` —
    u8 (B,H,W,C) uint8 CUDA = the bytes ``tvu.save_image`` would encode for each image (diffusion.py:596-598),
    psnr (B,) fp32 CUDA against ``inverse_data_transform(x_orig)`` (:599-601) or None, x01 the [0,1] images or None."""
    x = _cuda_f32(x)
    assert x.dim() == 4
    B, Cc, H, W = x.shape
    rescaled, logit = _flags(config)
    orig = _cuda_f32(x_orig) if x_orig is not None else None
    if orig is not None:
        assert orig.shape == x.shape
    u8 = torch.empty((B, H, W, Cc), dtype=torch.uint8, device=x.device)
    psnr = torch.empty((B,), dtype=torch.float32, device=x.device) if orig is not None else None
    x01 = torch.empty_like(x) if want_float else None
    _lib.check(_lib.lib().ddnm_finish_images(_lib.ptr(x), _lib.ptr(orig), B, Cc, H, W, rescaled, logit, _lib.ptr(x01), _lib.ptr(u8),
                                            _lib.ptr(psnr), _lib.cur_stream()))
    return u8, psnr, x01


# ------------------------------------------------------------------------------------------------------------------
# PNG container (host): zlib-deflated, filter 0 rows.  Decodes to exactly the uint8 array handed in, i.e. the same pixels
# the reference's PIL-written files hold.
# ------------------------------------------------------------------------------------------------------------------
def _chunk(tag, data):
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)


def encode_png(img_u8, level=6):
    a = np.ascontiguousarray(img_u8)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] in (1, 3), "expected (H, W, 1|3) uint8"
    h, w, c = a.shape
    raw = np.concatenate([np.zeros((h, 1), np.uint8), a.reshape(h, w * c)], axis=1).tobytes()
    ihdr = struct.pack(">IIBBBBB", w, h, 8, 0 if c == 1 else 2, 0, 0, 0)
    return b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", ihdr) + _chunk(b"IDAT", zlib.compress(raw, level)) + _chunk(b"IEND", b"")


def decode_png(blob):
    """Inverse of ``encode_png`` for its own files (8-bit gray / RGB, filter 0) — used by the tests."""
    assert blob[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, w = 8, b"", None
    while pos < len(blob):
        n, tag = struct.unpack(">I", blob[pos:pos + 4])[0], blob[pos + 4:pos + 8]
        data = blob[pos + 8:pos + 8 + n]
        if tag == b"IHDR":
            w, h, depth, ctype = struct.unpack(">IIBB", data[:10])
            assert depth == 8 and ctype in (0, 2)
            c = 1 if ctype == 0 else 3
        elif tag == b"IDAT":
            idat += data
        pos += 12 + n
    rows = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + w * c)
    assert not rows[:, 0].any(), "only filter 0 rows are produced by encode_png"
    return rows[:, 1:].reshape(h, w, c).copy()


def save_png(path, img_u8):
    with open(path, "wb") as f:
        f.write(encode_png(img_u8))


def _save_all(folder, pattern, u8_cuda, idx0):
    host = u8_cuda.cpu().numpy()
    for i in range(host.shape[0]):
        save_png(os.path.join(folder, pattern.format(idx0 + i)), host[i])
    return host


def restore_batch(config, model, A_funcs, deg, x_orig, betas, eta, sigma_y=0.0, add_noise=False, image_folder=None, idx_so_far=0,
                  x_T=None, noise=None, cls_fn=None, seed=None):
    """Body of the reference's evaluation loop for one batch (guided_diffusion/diffusion.py:533-603).

    x_orig: (B,C,H,W) in [0,1] (what the DataLoader yields), host or CUDA.  ``sigma_y`` is the level the reference passes on,
    i.e. already doubled (diffusion.py:524).  Returns a dict with ``psnr`` (B,) CPU, ``images`` (B,H,W,C) uint8 numpy,
    ``Apy`` / ``orig`` previews (uint8 numpy) and ``y``; PNGs are written under ``image_folder`` with the reference's names
    when it is given.

    ``seed``: x_T, the ``add_noise`` term and the loop's draws come from the library's seeded generator with
    ``row_offset = idx_so_far``, so image i of a dataset gets the same draws whatever ``sampling.batch_size`` is (the
    dequantisation draws of ``data_transform``, off in every shipped config, stay torch's); with ``model.batch_invariant``
    it restores bit-identically, otherwise to fp32 reassociation.
    """
    dev = torch.device("cuda")
    C_, R = config.data.channels, config.data.image_size
    with torch.no_grad():
        x_orig = data_transform(config, x_orig.to(dev, non_blocking=True))                # :534-535
        y = A_funcs.A(x_orig)                                                             # :537
        b, hwc = y.shape
        if add_noise and seed is not None:
            y = y + randn(seed, y.shape, TAG_Y, row_offset=idx_so_far, device=dev) * sigma_y
        elif add_noise:                                                                   # :550-551 (same draw count and order)
            y = get_gaussian_noisy_img(y, sigma_y)
        Apy = A_funcs.A_pinv(y).view(b, C_, R, R)                                         # :555
        if deg[:6] == "deblur":                                                           # :558-560
            Apy = y.view(b, C_, R, R)
        elif deg == "colorization":                                                       # :561-562
            Apy = y.view(b, 1, R, R).repeat(1, 3, 1, 1)
        elif deg == "inpainting":                                                         # :563-564
            Apy = Apy + (A_funcs.A_pinv(A_funcs.A(torch.ones_like(Apy))).reshape(*Apy.shape) - 1)
        apy_u8, _, _ = finish_images(config, Apy)
        orig_u8, _, _ = finish_images(config, x_orig)
        if x_T is None and seed is not None:
            x_T = randn(seed, (b, C_, R, R), TAG_XT, row_offset=idx_so_far, device=dev)
        elif x_T is None:
            x_T = torch.randn(b, C_, R, R, device=dev)                                    # :578-584
        plus = sigma_y != 0.0                                                             # :587-590
        x0, _ = sample_device(x_T, model, betas, eta, A_funcs, y, sigma_y if plus else 0.0, plus, config, noise=noise,
                              cls_fn=cls_fn, seed=seed,                                # cls_fn: diffusion.py:181-189 (class-conditional configs)
                              row_offset=idx_so_far if seed is not None else 0)
        img_u8, psnr, _ = finish_images(config, x0, x_orig)                               # :592-601
        out = dict(psnr=psnr.cpu(), y=y)
        if image_folder is not None:
            os.makedirs(os.path.join(image_folder, "Apy"), exist_ok=True)
            out["Apy"] = _save_all(image_folder, "Apy/Apy_{}.png", apy_u8, idx_so_far)
            out["orig"] = _save_all(image_folder, "Apy/orig_{}.png", orig_u8, idx_so_far)
            out["images"] = _save_all(image_folder, "{}_0.png", img_u8, idx_so_far)
        else:
            out["Apy"], out["orig"], out["images"] = apy_u8.cpu().numpy(), orig_u8.cpu().numpy(), img_u8.cpu().numpy()
    return out
