"""Drop-in for hq_demo's arbitrary-size DDNM restoration (the "mask-shift trick"): what
``hq_demo/main.py`` + ``SpacedDiffusion.p_sample_loop`` (hq_demo/guided_diffusion/gaussian_diffusion.py:578-750) do for one input
image — 256 x 256 windows every 128 pixels over an (H, W) canvas, each window a DDNM schedule with RePaint-style time travel
(scheduler.py get_schedule_jump), the already-restored part of every window pinned from the canvas (:344-384).

    out = restore(model, y_img, classes, deg="sr_averagepooling", scale=4, sigma_y=0.0, resize_y=True,
                  timestep_respacing=100, schedule_jump_params=dict(t_T=100, n_sample=1, jump_length=10, jump_n_sample=3))

``model`` is a learn_sigma 256x256 ``ddnm_b200.model.UNetModel``: the class-conditional imagenet network of
hq_demo/confs/inet256.yml (``classes``: the ImageNet label(s), main.py ``--class``) or the unconditional face network of
hq_demo/confs/face256.yml (called without labels, main.py:98-100; ``classes`` may be None).  ``cond_fn`` is the optional
classifier gradient callable ``cond_fn(x, t, y)`` (main.py:65-76).  ``conf_name`` selects the reference's ``conf.name`` gating:
under ``"face256"`` the input must be 256 pixels high (:586-588) and the masked degradations ``inpainting`` / ``mask_color_sr``
are available, with ``gt_keep_mask`` the (B,3,256,256) keep mask as the RePaint loader yields it (:601-621):

    out = restore(model, gt, None, deg="inpainting", conf_name="face256", gt_keep_mask=mask, timestep_respacing=250,
                  schedule_jump_params=dict(t_T=250, n_sample=1, jump_length=10, jump_n_sample=3))

The loops are host code exactly as in the reference; every tensor operation of a step (x0_t, clipping, Eq. 17 / 19, the
mask-shift overwrite, the posterior mean, the re-noising, the time-travel step) runs inside libddnm_b200.so, the denoiser as its
CUDA graph.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib
from .model import SuperResModel, UNetModel, _EngineModel
from .noise import TAG_HQ, randn


def get_schedule_jump(t_T, n_sample, jump_length, jump_n_sample, jump2_length=1, jump2_n_sample=1, jump3_length=1, jump3_n_sample=1,
                      start_resampling=100000000):
    """hq_demo/guided_diffusion/scheduler.py:70-148 (integers only)."""
    def table(length, n):
        return {j: n - 1 for j in range(0, t_T - length, length)}
    jumps, jumps2, jumps3 = table(jump_length, jump_n_sample), table(jump2_length, jump2_n_sample), table(jump3_length, jump3_n_sample)
    t, ts = t_T, []
    while t >= 1:
        t -= 1
        ts.append(t)
        if t + 1 < t_T - 1 and t <= start_resampling:
            for _ in range(n_sample - 1):
                t += 1
                ts.append(t)
                if t >= 0:
                    t -= 1
                    ts.append(t)
        if jumps3.get(t, 0) > 0 and t <= start_resampling - jump3_length:
            jumps3[t] -= 1
            for _ in range(jump3_length):
                t += 1
                ts.append(t)
        if jumps2.get(t, 0) > 0 and t <= start_resampling - jump2_length:
            jumps2[t] -= 1
            for _ in range(jump2_length):
                t += 1
                ts.append(t)
            jumps3 = table(jump3_length, jump3_n_sample)
        if jumps.get(t, 0) > 0 and t <= start_resampling - jump_length:
            jumps[t] -= 1
            for _ in range(jump_length):
                t += 1
                ts.append(t)
            jumps2 = table(jump2_length, jump2_n_sample)
            jumps3 = table(jump3_length, jump3_n_sample)
    ts.append(-1)
    assert ts[0] > ts[1] and all(abs(a - b) == 1 for a, b in zip(ts[:-1], ts[1:]))        # _check_times (:46-66)
    return ts


def space_timesteps(num_timesteps, section_counts):
    """respace.py:24-86 (comma-separated sections; the ddimN form is not used by the shipped configs)."""
    if isinstance(section_counts, str):
        section_counts = [int(x) for x in section_counts.split(",")]
    if isinstance(section_counts, int):
        section_counts = [section_counts]
    size_per, extra = divmod(num_timesteps, len(section_counts))
    start, steps = 0, []
    for i, count in enumerate(section_counts):
        size = size_per + (1 if i < extra else 0)
        if size < count:
            raise ValueError(f"cannot divide section of {size} steps into {count}")
        stride = 1 if count <= 1 else (size - 1) / (count - 1)
        cur = 0.0
        for _ in range(count):
            steps.append(start + round(cur))
            cur += stride
        start += size
    return set(steps)


class SpacedTables:
    """float64 constant tables of the respaced process (gaussian_diffusion.py:165-206, respace.py:89-107)."""

    def __init__(self, diffusion_steps, timestep_respacing):
        scale = 1000 / diffusion_steps
        betas = np.linspace(scale * 0.0001, scale * 0.02, diffusion_steps, dtype=np.float64)
        ac = np.cumprod(1.0 - betas, axis=0)
        use = space_timesteps(diffusion_steps, timestep_respacing)
        nb, self.timestep_map, last = [], [], 1.0
        for i, a in enumerate(ac):
            if i in use:
                nb.append(1 - a / last)
                last = a
                self.timestep_map.append(i)
        b = np.array(nb, dtype=np.float64)
        alphas = 1.0 - b
        acp = np.cumprod(alphas, axis=0)
        prev = np.append(1.0, acp[:-1])
        self.betas = b
        self.sqrt_recip = np.sqrt(1.0 / acp)
        self.sqrt_recipm1 = np.sqrt(1.0 / acp - 1)
        self.posterior_variance = b * (1.0 - prev) / (1.0 - acp)
        self.coef1 = b * np.sqrt(prev) / (1.0 - acp)
        self.coef2 = (1.0 - prev) * np.sqrt(alphas) / (1.0 - acp)


def _shift_rects(sh, sw, sh_total, sw_total, H, W):
    """The mask-shift overwrites of gaussian_diffusion.py:344-384 as up to two rectangles
    (dst_y, dst_x, h, w, src_y, src_x): x0_hat[dst] = canvas[src], applied in order."""
    none = (0, 0, 0, 0, 0, 0)
    if sw == 0 and sh == 0:
        return none, none
    last_h = sh == sh_total - 1 and H % 128 != 0
    last_w = sw == sw_total - 1 and W % 128 != 0
    if sw == 0:
        h_l = 128 * sh
        if last_h:
            return (0, 0, 256 - H % 128, 256, h_l - 128 + H % 128, 0), none
        return (0, 0, 128, 256, h_l, 0), none
    w_l, h_l = 128 * sw, 128 * sh
    if last_w:
        w_l = w_l - 128 + W % 128
        first = (0, 0, 256, 256 - W % 128, (h_l - 128 + H % 128) if last_h else h_l, w_l)
    else:
        first = (0, 0, 256, 128, (h_l - 128 + H % 128) if last_h else h_l, w_l)
    second = none
    if sh != 0:
        if last_h:
            second = (0, 0, 256 - H % 128, 256, h_l - 128 + H % 128, w_l)
        else:
            second = (0, 0, 128, 256, h_l, w_l)
    return first, second


def restore(model, gt, classes=None, deg="sr_averagepooling", scale=4, sigma_y=0.0, resize_y=False, timestep_respacing=100,
            schedule_jump_params=None, diffusion_steps=1000, clip_denoised=True, cond_fn=None, noise=None, seed=None,
            gt_keep_mask=None, conf_name="inet256"):
    """gt: the degraded input image(s) (B,3,h,w) in [-1,1] on the GPU (main.py:103-110); returns the restored canvas as a CPU
    tensor (B,3,H,W) — H, W = gt's size (x scale with ``resize_y``).  ``noise``: optional (n_draws,B,3,256,256) tape in the
    reference's draw order (initial x, then one per p_sample / undo call); by default the draws come from torch's generator in
    that order.  ``seed``: the library draws them instead (stream tag 3, draw index = position in that order, row = image), inside
    the step kernels; reproducible against itself, not against torch's generator.  The row is the image's index within this
    call (there is no row_offset), so with ``model.batch_invariant`` an image restores bit-identically in any call where it has
    the same index, e.g. alone and as row 0 of a batch.
    ``conf_name``: "inet256" or "face256" (the reference's conf.name).  ``gt_keep_mask``: the keep mask of ``inpainting`` /
    ``mask_color_sr`` (face256 only), fp32 in [0, 1] and broadcastable to (B,3,256,256); it multiplies, so fractional edge
    values weigh the pixel.  The masked degradations restore one 256 x 256 window per image: ``resize_y`` with a scale above 1
    would make gt larger than the mask, which the reference cannot multiply either.  hq_demo itself runs one image per call; with
    B > 1 every degradation here works image by image (the reference's color2gray would fold the batch into channels)."""
    if seed is not None and noise is not None:
        raise ValueError("seed= and noise= are two sources for the same draws: give one")
    if conf_name not in ("inet256", "face256"):
        raise ValueError(f"conf_name must be 'inet256' or 'face256', not {conf_name!r}")
    if not isinstance(model, _EngineModel):
        model = getattr(model, "module", model)
    if not isinstance(model, UNetModel) or isinstance(model, SuperResModel) or model.out_ch != 6 or model.resolution != 256:
        raise TypeError("hq.restore needs a learn_sigma 256x256 ddnm_b200 UNetModel (class-conditional or unconditional)")
    if model.num_classes is not None and classes is None:
        raise ValueError("the class-conditional model needs classes")
    if 256 % scale != 0:
        raise ValueError("Please set a SR scale divisible by 256")
    if conf_name == "face256" and gt.shape[2] != 256:             # :586-588, before resize_y
        raise ValueError("Only support output size 256x256 for face images")
    table = {"sr_averagepooling": (0, scale), "colorization": (1, 1), "sr_color": (1, scale)}
    if conf_name == "face256":                                  # :601-622
        table.update(inpainting=(0, 1), mask_color_sr=(1, scale))
    if deg not in table:
        raise NotImplementedError("degradation type not supported")
    use_gray, sc = table[deg]
    masked = deg in ("inpainting", "mask_color_sr")
    if masked:
        if gt_keep_mask is None:
            raise ValueError(f"{deg} needs gt_keep_mask")
        if resize_y and scale != 1:
            raise ValueError(f"{deg} with resize_y: gt would be {256 * scale} pixels high, the keep mask is 256 x 256")
        if gt.shape[3] != 256:
            raise ValueError(f"{deg} needs a 256 x 256 gt (the keep mask's size)")
    L = _lib.lib()
    jump = schedule_jump_params or dict(t_T=int(timestep_respacing), n_sample=1, jump_length=10, jump_n_sample=3)
    K = SpacedTables(diffusion_steps, timestep_respacing)
    with torch.no_grad():
        dev = torch.device("cuda", torch.cuda.current_device())
        gt = gt.to(dev).float().contiguous()
        B = gt.shape[0]
        if resize_y:                                            # MeanUpsample(gt, scale) (:593-595): pure replication
            gt = gt.repeat_interleave(scale, 2).repeat_interleave(scale, 3).contiguous()
        H, W = gt.shape[2], gt.shape[3]
        if H % sc or W % sc:
            raise ValueError("image size must be a multiple of the SR scale")
        if H < 256 or W < 256:
            raise ValueError("Please set a larger SR scale")
        d = _lib.SimpleDeg()
        d.use_mask, d.use_gray, d.scale, d.img_dim, d.channels, d.mask = 0, use_gray, sc, 256, 3, None
        apy_canvas = torch.empty_like(gt)
        scratch = torch.empty(3 * B * 3 * 256 * 256, device=dev)
        if masked:
            try:
                mask = torch.broadcast_to(gt_keep_mask.to(dev).float(), (B, 3, 256, 256)).contiguous()
            except RuntimeError as e:
                raise ValueError(f"gt_keep_mask of shape {tuple(gt_keep_mask.shape)} does not broadcast to {(B, 3, 256, 256)}") from e
            d.image_mask = mask.data_ptr()
            _lib.check(L.ddnm_hq_canvas_masked(C.byref(d), _lib.ptr(gt), B, _lib.ptr(apy_canvas), _lib.ptr(scratch), _lib.cur_stream()))
        else:
            _lib.check(L.ddnm_hq_canvas(_lib.ptr(gt), B, H, W, sc, use_gray, _lib.ptr(apy_canvas), _lib.cur_stream()))
        final = torch.zeros_like(gt)
        sh_total, sw_total = math.ceil(H / 128) - 1, math.ceil(W / 128) - 1
        labels = None if classes is None else torch.as_tensor(classes).to(dev).long().reshape(-1)
        model_labels = labels if model.num_classes is not None else None     # face256: model(x, t, None) (main.py:98-100)
        tape = None if noise is None else noise.to(dev).float().contiguous()
        ns = None if seed is None else _lib.noise_seed(seed)
        draws = [0]

        def draw():
            """The next draw: a tensor (torch / tape modes), or its index (seeded mode: the kernels generate the values)."""
            k = draws[0]
            draws[0] += 1
            if ns is not None:
                return k
            return torch.randn(B, 3, 256, 256, device=dev) if tape is None else tape[k]
        if ns is None:
            x = draw().clone()                                  # th.randn(*shape) (:574); carried over from window to window
        else:
            x = randn(seed, (B, 3, 256, 256), TAG_HQ, draw=draw(), device=dev)
        x_next, x0_hat = torch.empty_like(x), torch.empty_like(x)
        times = get_schedule_jump(**jump)
        for sh in range(sh_total):
            for sw in range(sw_total):
                h_l = H - 256 if (sh == sh_total - 1 and H % 128 != 0) else 128 * sh
                w_l = W - 256 if (sw == sw_total - 1 and W % 128 != 0) else 128 * sw
                apy = apy_canvas[:, :, h_l:h_l + 256, w_l:w_l + 256].contiguous()
                r0, r1 = _shift_rects(sh, sw, sh_total, sw_total, H, W)
                rects = (C.c_int * 12)(*r0, *r1)
                for t_last, t_cur in zip(times[:-1], times[1:]):
                    if t_cur < t_last:
                        t = t_last
                        t_model = torch.full((B,), float(K.timestep_map[t]), device=dev)
                        mo = model(x, t_model, model_labels)
                        s = _lib.HqScalars()
                        f = np.float32
                        post_var = f(K.posterior_variance[t])
                        sigma_t, a_t = np.sqrt(post_var, dtype=np.float32), f(K.coef1[t])
                        if sigma_t >= a_t * f(sigma_y):                     # Eq. 19 (:330-336), float32 like the 0-dim tensors
                            lam, gam = f(1.0), post_var - (a_t * f(1.0) * f(sigma_y)) ** 2
                        else:
                            lam, gam = sigma_t / a_t * f(sigma_y), f(0.0)
                        s.c_recip, s.c_recipm1 = float(f(K.sqrt_recip[t])), float(f(K.sqrt_recipm1[t]))
                        s.coef1, s.coef2 = float(a_t), float(f(K.coef2[t]))
                        s.lambda_t, s.gamma_t, s.nonzero, s.clip = float(lam), float(gam), 0.0 if t == 0 else 1.0, 1 if clip_denoised else 0
                        grad = None
                        if cond_fn is not None:                             # condition_mean (:414-430)
                            with torch.enable_grad():
                                grad = cond_fn(x, torch.full((B,), K.timestep_map[t], device=dev, dtype=torch.long), labels)
                            grad = grad.float().contiguous()
                        z = draw()
                        if ns is None:
                            _lib.check(L.ddnm_hq_step(C.byref(d), _lib.ptr(x), _lib.ptr(mo), 6, _lib.ptr(apy), _lib.ptr(final), H, W, rects,
                                                      _lib.ptr(grad), _lib.ptr(z), C.byref(s), B, _lib.ptr(x0_hat), _lib.ptr(x_next),
                                                      _lib.ptr(scratch), _lib.cur_stream()))
                        else:
                            _lib.check(L.ddnm_hq_step_seeded(C.byref(d), _lib.ptr(x), _lib.ptr(mo), 6, _lib.ptr(apy), _lib.ptr(final), H, W,
                                                             rects, _lib.ptr(grad), C.byref(ns), z, C.byref(s), B, _lib.ptr(x0_hat),
                                                             _lib.ptr(x_next), _lib.ptr(scratch), _lib.cur_stream()))
                        x, x_next = x_next, x
                    else:
                        beta = np.float32(K.betas[t_last + 1])              # inpa_inj_time_shift = 1 (:727-733)
                        z = draw()
                        a, bb = float(np.sqrt(np.float32(1.0) - beta, dtype=np.float32)), float(np.sqrt(beta, dtype=np.float32))
                        if ns is None:
                            _lib.check(L.ddnm_hq_undo(_lib.ptr(x), _lib.ptr(z), a, bb, x.numel(), _lib.cur_stream()))
                        else:
                            _lib.check(L.ddnm_hq_undo_seeded(_lib.ptr(x), C.byref(ns), z, a, bb, B, x[0].numel(), _lib.cur_stream()))
                final[:, :, h_l:h_l + 256, w_l:w_l + 256] = x0_hat           # :737-747
        return final.to("cpu")
