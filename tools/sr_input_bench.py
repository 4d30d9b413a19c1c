"""Input stage of the super-resolution UNet at its output size: the fused stem (bilinear upsample + channel concat inside the
3x3 convolution, ``ddnm_conv_stem_sr`` with low_res) against the composition it replaces (``F.interpolate`` + ``torch.cat`` in
PyTorch, then the same convolution on the concatenated tensor), and one whole denoising forward of a SuperResModel for scale.

    python tools/sr_input_bench.py [--batch 16] [--size 256] [--small 64] [--cout 192] [--iters 200] [--rounds 3] [--forward-batch 8] [--out FILE]

Per arm: kernel / op time from CUDA events over --iters back-to-back launches (arms alternated --rounds times), and the peak of
torch's allocator during one input stage above what the inputs and the output already hold.  Prints one JSON line with the GPU's
name, power limit and maximum SM clock read in the same run.  Random inputs and weights; needs an H100."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ddnm_b200 import _lib  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in q.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # noqa: BLE001 — reported, not fatal
        return dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=str(e))


def stem(x, low, w, b, out, iters, fused):
    N, C_, H, W = x.shape
    ms = C.c_float(0.0)
    _lib.check(_lib.lib().ddnm_conv_stem_sr(_lib.ptr(x), _lib.ptr(low) if fused else None, N, 3, H, W, low.shape[2], low.shape[3],
                                            _lib.ptr(w), _lib.ptr(b), w.shape[0], _lib.ptr(out), iters, C.byref(ms), _lib.cur_stream()))
    return ms.value


def events(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def compose(x, low):
    return torch.cat([x, F.interpolate(low, x.shape[2:], mode="bilinear", align_corners=False)], dim=1)


def peak_extra(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del r
    return peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--small", type=int, default=64)
    ap.add_argument("--cout", type=int, default=192)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--forward-batch", type=int, default=8)
    ap.add_argument("--forward-iters", type=int, default=10)
    ap.add_argument("--out", default="", help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(1)
    B, R, s, Co = a.batch, a.size, a.small, a.cout
    x = torch.randn(B, 3, R, R, device=dev, generator=g)
    low = torch.rand(B, 3, s, s, device=dev, generator=g) * 2 - 1
    w = torch.randn(Co, 6, 3, 3, device=dev, generator=g) * 0.2
    b = torch.randn(Co, device=dev, generator=g) * 0.1
    out = torch.empty(B, R, R, Co, device=dev)
    out2 = torch.empty_like(out)
    cat = compose(x, low)
    # warm-up of every shape, and the two forms agree
    stem(x, low, w, b, out, 3, True)
    stem(cat, low, w, b, out2, 3, False)
    agree = (out - out2).abs().max().item()

    res = dict(fused_ms=[], composed_torch_ms=[], composed_conv_ms=[], composed_ms=[])
    for _ in range(a.rounds):
        res["fused_ms"].append(stem(x, low, w, b, out, a.iters, True))
        t_torch = events(lambda: compose(x, low), a.iters)
        t_conv = stem(cat, low, w, b, out2, a.iters, False)
        res["composed_torch_ms"].append(t_torch)
        res["composed_conv_ms"].append(t_conv)
        res["composed_ms"].append(t_torch + t_conv)
    del cat
    peak_fused = peak_extra(lambda: stem(x, low, w, b, out, 0, True))

    def composed_stage():
        c = compose(x, low)
        stem(c, low, w, b, out2, 0, False)
        return c
    peak_comp = peak_extra(composed_stage)

    # one whole forward of the 64 -> 256 upsampler's network shape (sr_create_model defaults of the guided-diffusion release)
    from ddnm_b200.model import sr_create_model
    from ddnm_b200.weights import random_state_dict_openai
    m = sr_create_model(R, s, Co, 2, learn_sigma=True, class_cond=False, use_checkpoint=False, attention_resolutions="32,16,8",
                        num_heads=4, num_head_channels=64, num_heads_upsample=-1, use_scale_shift_norm=True, dropout=0.0,
                        resblock_updown=True, use_fp16=False)
    m.load_state_dict(random_state_dict_openai(m, 1234))
    fb = a.forward_batch
    xf, tf = x[:fb].contiguous(), torch.full((fb,), 500.0, device=dev)
    h, _ = m.stage_low_res(low[:fb].contiguous(), fb)
    of = torch.empty(fb, 6, R, R, device=dev)
    fwd = lambda: _lib.check(_lib.lib().ddnm_unet_forward(h, _lib.ptr(xf), _lib.ptr(tf), _lib.ptr(of), _lib.cur_stream()))  # noqa: E731
    for _ in range(2):
        fwd()
    fwd_ms = sorted(events(fwd, a.forward_iters) for _ in range(a.rounds))
    stem_share = [op for op in m.profile(xf, tf) if op["name"] == "stem.sr"][0]["ms"]

    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    line = dict(gpu_info(), batch=B, size=R, small=s, cout=Co, iters=a.iters, rounds=a.rounds,
                fused_ms=res["fused_ms"], composed_ms=res["composed_ms"], composed_torch_ms=res["composed_torch_ms"],
                composed_conv_ms=res["composed_conv_ms"], fused_median_ms=med(res["fused_ms"]),
                composed_median_ms=med(res["composed_ms"]), fused_vs_composed_max_abs_diff=agree,
                peak_extra_bytes_fused=peak_fused, peak_extra_bytes_composed=peak_comp,
                forward_batch=fb, forward_ms=fwd_ms, forward_median_ms=med(fwd_ms), forward_stem_ms_eager=stem_share,
                workspace_bytes=m.info(fb)["workspace_bytes"])
    print(json.dumps(line))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
