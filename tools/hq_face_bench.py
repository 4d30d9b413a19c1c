"""Time one hq_demo face256 restoration on the GPU and print one JSON line with the GPU's name and power limit.

The model is face256.yml's unconditional UNetModel (256 channels, 2 res blocks, attention at 32/16/8, 64-wide heads, learn_sigma)
with random weights; the schedule is 250 respaced steps with jump 10 / 3 (face256.yml:33, 61-65).  For B = 1 and B = 4 it reports

  restore_s       wall time of hq.restore(deg="inpainting") with the hq_demo mouth-shaped keep mask, seeded draws
  pairs           (t_last, t_cur) pairs of the schedule: forward + fused step, or one time-travel step
  fwd_ms          the denoiser forward (CUDA graph), median of --iters
  step_ms         one fused ddnm_hq_step with the per-image mask (inpainting and mask_color_sr x4), median of --iters

  python tools/hq_face_bench.py [--iters 50]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from classifier_bench import smi, timed   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    from ddnm_b200 import _lib
    from ddnm_b200 import hq as HQ
    from ddnm_b200.model import create_model
    from ddnm_b200.weights import random_state_dict_openai

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = _lib.lib()
    m = create_model(image_size=256, num_channels=256, num_res_blocks=2, learn_sigma=True, class_cond=False,
                     attention_resolutions="32,16,8", num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True,
                     use_fp16=False)
    m.load_state_dict(random_state_dict_openai(m, seed=7))
    jump = dict(t_T=250, n_sample=1, jump_length=10, jump_n_sample=3)
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"),
           "pairs": len(HQ.get_schedule_jump(**jump)) - 1}
    g = torch.Generator().manual_seed(0)
    mask = torch.ones(1, 3, 256, 256)
    mask[:, :, 150:210, 80:176] = 0                       # a mouth-region hole
    for B in (1, 4):
        gt = (torch.rand(B, 3, 256, 256, generator=g) * 2 - 1).to(dev)
        masks = mask.expand(B, -1, -1, -1).contiguous().to(dev)
        x = torch.randn(B, 3, 256, 256, generator=g).to(dev)
        t = torch.full((B,), 500.0, device=dev)
        with torch.no_grad():
            fwd = timed(lambda: m(x, t, None), args.iters)[0]
        mo = m(x, t, None)
        s = _lib.HqScalars()
        s.c_recip, s.c_recipm1, s.coef1, s.coef2, s.lambda_t, s.gamma_t, s.nonzero, s.clip = 1.5, 1.1, 0.5, 0.5, 1.0, 0.01, 1.0, 1
        rects = (C.c_int * 12)(*([0] * 12))
        z = torch.randn_like(x)
        x0h, xn, scratch = torch.empty_like(x), torch.empty_like(x), torch.empty(3 * x.numel(), device=dev)
        steps = {}
        for name, gray, sc in (("inpainting", 0, 1), ("mask_color_sr4", 1, 4)):
            d = _lib.SimpleDeg()
            d.use_mask, d.use_gray, d.scale, d.img_dim, d.channels, d.mask = 0, gray, sc, 256, 3, None
            d.image_mask = masks.data_ptr()

            def step():
                _lib.check(L.ddnm_hq_step(C.byref(d), _lib.ptr(x), _lib.ptr(mo), 6, _lib.ptr(gt), _lib.ptr(gt), 256, 256, rects, None,
                                          _lib.ptr(z), C.byref(s), B, _lib.ptr(x0h), _lib.ptr(xn), _lib.ptr(scratch), _lib.cur_stream()))
            steps[name] = round(timed(step, args.iters)[0], 4)
        HQ.restore(m, gt, None, deg="inpainting", timestep_respacing=10, schedule_jump_params=dict(t_T=10, n_sample=1, jump_length=10,
                   jump_n_sample=1), seed=1, gt_keep_mask=masks, conf_name="face256")                 # warm-up (engine build)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        HQ.restore(m, gt, None, deg="inpainting", timestep_respacing=250, schedule_jump_params=jump, seed=1, gt_keep_mask=masks,
                   conf_name="face256")
        torch.cuda.synchronize()
        res[f"B{B}"] = {"restore_s": round(time.perf_counter() - t0, 3), "fwd_ms": round(fwd, 3), "step_ms": steps}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
