"""Oracle: hq_demo's face256 configuration, on top of oracle/hq.py.

Restates what /root/reference/hq_demo adds for ``confs/face256.yml``:
  * the unconditional learn_sigma denoiser, called as ``model(x, t, None)`` (main.py:98-100),
  * the ``conf.name == 'face256'`` gating of ``p_sample_loop_progressive`` (gaussian_diffusion.py:586-588, :601-621): the input must
    be 256 pixels high (checked before ``resize_y``); ``inpainting`` and ``mask_color_sr`` exist only there,
  * the keep-mask degradations (:601-622) with ``gt_keep_mask`` (B,3,256,256), A_temp = A:
      inpainting     A(z) = z*mask,                         Ap = A
      mask_color_sr  A(z) = pool(color2gray(z*mask)),        Ap(v) = gray2color(MeanUpsample(v))*mask
hq_demo runs one image per call (main.py builds gt with ``unsqueeze(0)``).  Its color2gray returns ``(B,H,W).repeat(1,3,1,1)``,
which is (1,3B,H,W) for B > 1, so gray2color would then read image 0 for every row; this oracle converts each image on its own,
which is what a B = 1 call computes for every row.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import torch

from oracle import hq as HQO


def color2gray(x):
    """color2gray of each image: (B,3,H,W) -> (B,3,H,W), rounded as :54-57"""
    coef = 1 / 3
    g = x[:, 0, :, :] * coef + x[:, 1, :, :] * coef + x[:, 2, :, :] * coef
    return g[:, None].repeat(1, 3, 1, 1)


def masked_degradation(deg, scale, mask):
    """(A, Ap) of :601-622; A_temp = A"""
    if deg == "inpainting":
        A = lambda z: z * mask      # noqa: E731
        return A, A
    if deg == "mask_color_sr":
        pool = torch.nn.AdaptiveAvgPool2d((256 // scale, 256 // scale))
        return (lambda z: pool(color2gray(z * mask))), (lambda z: HQO.gray2color(HQO.mean_upsample(z, scale)) * mask)
    raise NotImplementedError("degradation type not supported")


def restore(model, gt, classes, noise, *, deg="sr_averagepooling", scale=4, sigma_y=0.0, resize_y=False, diffusion_steps=1000,
            respacing=100, jump=None, clip_denoised=True, cond_fn=None, gt_keep_mask=None, conf_name="face256", trace=None):
    """oracle.hq.restore with the face256 rules and degradations; ``model(x, t_original, classes)`` (classes may be None for the
    unconditional denoiser).  The keep-mask degradations restore the single 256 x 256 window of a 256 x 256 gt."""
    if 256 % scale != 0:
        raise ValueError("Please set a SR scale divisible by 256")
    if conf_name == "face256" and gt.shape[2] != 256:
        raise ValueError("Only support output size 256x256 for face images")
    if deg not in ("inpainting", "mask_color_sr"):
        return HQO.restore(model, gt, classes, noise, deg=deg, scale=scale, sigma_y=sigma_y, resize_y=resize_y,
                           diffusion_steps=diffusion_steps, respacing=respacing, jump=jump, clip_denoised=clip_denoised,
                           cond_fn=cond_fn, trace=trace)
    if conf_name != "face256":
        raise NotImplementedError("degradation type not supported")
    if resize_y:
        gt = HQO.mean_upsample(gt, scale)
    assert gt.shape[2:] == (256, 256) and gt_keep_mask is not None
    K = HQO.SpacedConstants(diffusion_steps, respacing)
    jump = jump or dict(t_T=respacing, n_sample=1, jump_length=10, jump_n_sample=3)
    noise = list(noise)
    A, Ap = masked_degradation(deg, scale, gt_keep_mask)
    Apy = Ap(A(gt))                                                  # :645-646
    B = gt.shape[0]
    x = noise.pop(0)
    tmap = torch.tensor(K.timestep_map)
    f32 = HQO.f32
    x0_hat = None
    times = HQO.get_schedule_jump(**jump)
    for t_last, t_cur in zip(times[:-1], times[1:]):                 # one window: no mask-shift overwrite
        if t_cur < t_last:
            t = t_last
            tt = torch.full((B,), t, dtype=torch.long)
            eps = model(x, tmap[tt], classes)[:, :3]
            x0_t = f32(K.sqrt_recip_alphas_cumprod, t) * x - f32(K.sqrt_recipm1_alphas_cumprod, t) * eps
            if clip_denoised:
                x0_t = x0_t.clamp(-1, 1)
            sigma_t = torch.sqrt(f32(K.posterior_variance, t))
            a_t = f32(K.posterior_mean_coef1, t)
            if sigma_t >= a_t * sigma_y:
                lambda_t = 1
                gamma_t = f32(K.posterior_variance, t) - (a_t * lambda_t * sigma_y) ** 2
            else:
                lambda_t = sigma_t / a_t * sigma_y
                gamma_t = 0.
            x0_hat = lambda_t * Apy + x0_t - lambda_t * Ap(A(x0_t))
            mean = f32(K.posterior_mean_coef1, t) * x0_hat + f32(K.posterior_mean_coef2, t) * x
            if cond_fn is not None:
                mean = mean.float() + gamma_t * cond_fn(x, tmap[tt], classes).float()
            nonzero = 0.0 if t == 0 else 1.0
            x = mean + nonzero * torch.sqrt(torch.ones(1) * gamma_t) * noise.pop(0)
            if trace is not None:
                trace.append(dict(t=t, x0_hat=x0_hat.clone(), x=x.clone()))
        else:
            beta = f32(K.betas, t_last + 1)
            x = torch.sqrt(1 - beta) * x + torch.sqrt(beta) * noise.pop(0)
    return x0_hat.clone()
