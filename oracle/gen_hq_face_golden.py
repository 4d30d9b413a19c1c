"""Fixtures of hq_demo's face256 configuration, from the reference's own code: tests/golden/hq_face.npz (+ .part files).

hq_demo's create_model_and_diffusion + SpacedDiffusion.p_sample_loop_progressive (gaussian_diffusion.py:548-756) on a face256-
shaped conf: an unconditional learn_sigma UNetModel of reduced width (64 base channels, one res block per level, attention at
32/16/8 with 64-wide heads, random weights), 6 respaced steps with a jump schedule that travels back, B = 2 images with two
different keep masks (hq_demo's mask_mouth.png through the RePaint loader's transform, and a synthetic mask with fractional
edges whose third channel differs), torch-drawn noise tapes.  Cases: inpainting, mask_color_sr at scale 2 and 4 (the second
with sigma_y = 0.1), sr_averagepooling at scale 4 on the 256 x 256 face input, and sr_averagepooling with resize_y over two
windows of a 256 x 320 canvas (inet256 gating, same unconditional model).

p_sample_loop (:495-546) forwards to p_sample_loop_progressive and then iterates over the keys of the dict that returns, so the
canvas is taken from that dict's "sample".  hq_demo restores one image per call (main.py builds gt with unsqueeze(0)); its
color2gray turns (B,H,W) into (1,3B,H,W) through repeat(1,3,1,1), which for B > 1 makes gray2color read image 0 for every row.
The mask_color_sr cases therefore run the reference once per image (B = 1, the image's rows of the tape) and stack the results.

    python -m oracle.gen_hq_face_golden        (a process of its own: hq_demo's guided_diffusion shadows the main reference's)

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import os
import sys

import numpy as np
import torch

from oracle.gen_golden import GOLD, REF, close, save_split
from oracle import hq as HQO
from oracle import hq_face as HQF
from oracle import unet_openai as UO
from oracle.ref_shim import cpu_shim

HQ = os.path.join(REF, "hq_demo")
JUMP = dict(t_T=6, n_sample=1, jump_length=2, jump_n_sample=2)
# key, deg, scale, sigma_y, resize_y, input (h, w), conf name
CASES = [("inpaint", "inpainting", 1, 0.0, False, (256, 256), "face256"),
         ("mcsr2", "mask_color_sr", 2, 0.0, False, (256, 256), "face256"),
         ("mcsr4_noisy", "mask_color_sr", 4, 0.1, False, (256, 256), "face256"),
         ("sr4", "sr_averagepooling", 4, 0.0, False, (256, 256), "face256"),
         ("sr4_w320", "sr_averagepooling", 4, 0.0, True, (64, 80), "inet256")]


def unet_cfg():
    return UO.OpenAIUNetConfig(image_size=256, model_channels=64, num_res_blocks=1, channel_mult=(1, 1, 2, 2, 4, 4),
                               attention_resolutions=(32, 16, 8), num_head_channels=64, out_channels=6, num_classes=None)


def synthetic_mask():
    """(3,256,256) keep mask with 8-pixel linear edges, quantised like a PNG / 255; channel 2's hole is shifted by 6 pixels"""
    yy, xx = np.mgrid[0:256, 0:256].astype(np.float64)
    chans = []
    for c in range(3):
        dy = 6 if c == 2 else 0
        d = np.maximum(np.abs(yy - 150 - dy) - 40, np.abs(xx - 128) - 70)
        chans.append(np.round(np.clip(d / 8 + 0.5, 0, 1) * 255) / 255)
    return np.stack(chans).astype(np.float32)


def mouth_mask():
    """hq_demo/data/datasets/gt_keep_masks/face/mask_mouth.png as image_datasets.py:163-188 hands it over: RGB, / 255, CHW (the
    PNG is 256 x 256 already, so center_crop_arr resizes it to its own size and crops nothing)"""
    from PIL import Image
    pil = Image.open(os.path.join(HQ, "data/datasets/gt_keep_masks/face/mask_mouth.png"))
    pil.load()
    arr = np.asarray(pil.convert("RGB"))
    assert arr.shape == (256, 256, 3)
    return np.transpose(arr.astype(np.float32) / 255.0, [2, 0, 1])


def main():
    assert "guided_diffusion" not in sys.modules, "run `python -m oracle.gen_hq_face_golden` in a process of its own"
    sys.path.insert(0, HQ)
    import guided_diffusion.gaussian_diffusion as GD
    from guided_diffusion.script_util import create_model_and_diffusion, model_and_diffusion_defaults, select_args
    import conf_mgt
    assert os.path.abspath(GD.__file__).startswith(HQ)
    GD.save_image = lambda img, save_dir, idx: None          # progress PNGs (:49-52)
    GD.os.makedirs = lambda *a, **k: None
    conf = conf_mgt.conf_base.Default_Conf()
    base = dict(attention_resolutions="32,16,8", class_cond=False, diffusion_steps=1000, learn_sigma=True, noise_schedule="linear",
                num_channels=64, num_head_channels=64, num_heads=4, num_res_blocks=1, resblock_updown=True, use_fp16=False,
                use_scale_shift_norm=True, timestep_respacing="6", use_kl=False, predict_xstart=False, rescale_timesteps=False,
                rescale_learned_sigmas=False, num_heads_upsample=-1, channel_mult="", dropout=0.0, use_checkpoint=False,
                use_new_attention_order=False, image_size=256, name="face256", schedule_jump_params=JUMP)
    conf.update(base)
    torch.manual_seed(4321)
    model, diffusion = create_model_and_diffusion(**select_args(conf, model_and_diffusion_defaults().keys()), conf=conf)
    model.eval()
    cfg = unet_cfg()
    sd = UO.init_state_dict(cfg, 4321)
    rsd = model.state_dict()
    assert set(sd) == set(rsd), sorted(set(sd) ^ set(rsd))[:8]
    for k in sd:
        if not torch.equal(sd[k], rsd[k]):
            assert rsd[k].abs().sum() == 0, f"{k}: differs from the reference but is not a zero-initialised tensor"
    model.load_state_dict(sd)
    times = HQO.get_schedule_jump(**JUMP)
    assert any(b > a for a, b in zip(times[:-1], times[1:])), "the schedule must travel back at least once"

    def model_fn(x, t, y=None, gt=None, **kwargs):            # main.py:98-100 with class_cond: false
        return model(x, t, None)
    masks = torch.from_numpy(np.stack([mouth_mask(), synthetic_mask()]))
    m = masks.numpy()
    assert set(np.unique(m[0])) == {0.0, 1.0} and ((m[1] > 0) & (m[1] < 1)).any() and not np.array_equal(m[1, 0], m[1, 2])
    out = {"masks": m}
    for i, (key, deg, scale, sy, resize_y, (h, w), name) in enumerate(CASES):
        conf.update(dict(base, name=name))
        seed = 900 + i
        g = torch.Generator().manual_seed(seed)
        gt = torch.rand(2, 3, h, w, generator=g) * 2 - 1
        H, W = (h * scale, w * scale) if resize_y else (h, w)
        tape = [torch.randn(2, 3, 256, 256, generator=g) for _ in range(HQO.count_draws(H, W, JUMP))]
        rows = [slice(0, 2)] if deg != "mask_color_sr" else [slice(0, 1), slice(1, 2)]
        ref = []
        for r in rows:
            kw = dict(gt=gt[r].clone(), scale=scale, deg=deg, resize_y=resize_y, sigma_y=sy, save_path="unused",
                      y=torch.zeros(r.stop - r.start, dtype=torch.long))
            if deg in ("inpainting", "mask_color_sr"):
                kw["gt_keep_mask"] = masks[r].clone()
            rt = [z[r] for z in tape[1:]]
            with torch.no_grad(), cpu_shim(rt) as shim:
                res = diffusion.p_sample_loop_progressive(model_fn, (r.stop - r.start, 3, 256, 256), noise=tape[0][r], clip_denoised=True,
                                                          model_kwargs=kw, cond_fn=None, device="cpu", progress=False, conf=conf)
            assert len(shim.tape) == 0, f"{key}: the reference consumed a different number of draws ({len(shim.tape)} left)"
            ref.append(res["sample"])
        ref = torch.cat(ref)
        with torch.no_grad():       # the oracle at the reference's batch size
            o = torch.cat([HQF.restore(lambda a, b, c: UO.forward(sd, a, b.float(), cfg), gt[r], None, [z[r] for z in tape], deg=deg,
                                       scale=scale, sigma_y=sy, resize_y=resize_y, respacing=6, jump=JUMP, gt_keep_mask=masks[r],
                                       conf_name=name) for r in rows])
        d = close(o, ref, 2e-3, f"hq_face {key}")
        assert ref.shape == (2, 3, H, W)
        out[key + "_seed"] = np.array([seed])
        out[key + "_out_s2"] = ref[:, :, ::2, ::2].contiguous().numpy()
        out[key + "_sums"] = np.array([ref.double().sum().item(), ref.double().abs().sum().item()])
        print(f"hq_face {key}: canvas {tuple(ref.shape)}, {len(tape)} draws, ok (oracle-ref {d:.2e})")
    save_split(os.path.join(GOLD, "hq_face"), out)


if __name__ == "__main__":
    main()
