"""Where a form of the wgmma convolution moves time, layer by layer, on the celeba `Model` at B = 16 (the bench workload).
--switch halo (default): the HALO form; --switch pingpong: the ping-pong kernel; --switch pppair: CTA pairs in the ping-pong kernel
(not the upsample phases).

1. Every celeba layer shape the HALO form applies to (3x3 stride 1 and upsample phases on maps >= 64 px wide), timed with
   `ddnm_conv_tc_bench` on pseudo-random operands, the form off and on alternately: ms, algorithmic TFLOP/s and the L2 -> shared
   memory fill bytes per launch computed from the shape (HALO; pppair: the weights once per pair of tiles).  With --switch pingpong
   and pppair the epilogue features are the network's (GroupNorm sums, residual, channel add).
2. One eager forward per arm (`Model.profile`, CUDA events around every launch), twice per arm in alternation: per tensor-core launch
   ms both ways, and the totals.

The GPU's name, power limit and SM clocks are printed with the numbers (read-only nvidia-smi queries).
Usage: python tools/halo_layers.py [--switch halo|pingpong|pppair] [--iters 20] [--json OUT]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ddnm_b200 import _lib                                           # noqa: E402
from ddnm_b200.model import Model                                    # noqa: E402
from ddnm_b200.weights import random_state_dict                      # noqa: E402

N = 16
BK = 64
# (label, H = W of the source, Cin, Cout, up2) of the celeba network's HALO-eligible launches; conv2's 1x1 shortcut (extra K blocks of
# the same launch) is not part of the op-level shape
SHAPES = [
    ("256 conv 128->128", 256, 128, 128, False),
    ("256 conv 256->128", 256, 256, 128, False),
    ("128 conv 128->128", 128, 128, 128, False),
    ("128 conv 256->128", 128, 256, 128, False),
    ("128 conv 384->128", 128, 384, 128, False),
    ("64 conv 128->256", 64, 128, 256, False),
    ("64 conv 256->256", 64, 256, 256, False),
    ("64 conv 384->256", 64, 384, 256, False),
    ("64 conv 512->256", 64, 512, 256, False),
    ("up2 128->256 128ch (phase)", 128, 128, 128, True),
    ("up2 64->128 256ch (phase)", 64, 256, 256, True),
]
FEAT_STATS, FEAT_RES, FEAT_CHANADD, FEAT_UP2 = 16, 32, 64, 128   # ddnm_conv_tc_bench mode bits (see api.cu)
SWITCHES = {"halo": "ddnm_tc_debug_halo", "pingpong": "ddnm_tc_debug_pingpong", "pppair": "ddnm_tc_debug_pp_pair"}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() or r.stderr.strip()


def fill_bytes(H, W, Cin, Cout, up2, halo, bn=128, pair=False):
    """L2 -> shared-memory bytes of one launch (hi + lo planes): per tile, the weights of every k-block (pair: half of them, the
    other half arrives by multicast) plus the A operand, one 128-row box per k-block or one halo unit per (dy, channel slice)."""
    bw = min(W, 128)
    bh = 128 // bw
    tiles = N * H * W // 128 * (Cout // bn)
    cb = Cin // BK
    r = 2 if up2 else 3
    kb = r * r * cb
    b = kb * 2 * bn * BK * 2 // (2 if pair else 1)
    a = r * cb * 2 * (bw + r - 1) * bh * 128 if halo else kb * 2 * 128 * BK * 2
    return tiles * (a + b)


def bench_shapes(L, switch, iters):
    ms, fl = C.c_float(), C.c_double()
    rows = []
    for label, H, Cin, Cout, up2 in SHAPES:
        if switch == "ddnm_tc_debug_pp_pair" and up2:   # the upsample phases stay on single CTAs
            continue
        # 3x3 stride 1 (mode 0) + the epilogue features the network uses (the op-level upsample phase takes no residual)
        mode = FEAT_STATS | (FEAT_UP2 if up2 else 0)
        if switch in ("ddnm_tc_debug_pingpong", "ddnm_tc_debug_pp_pair"):
            mode |= FEAT_CHANADD | (0 if up2 else FEAT_RES)
        t = {0: [], 1: []}
        for rep in range(2):
            for halo in (0, 1):
                _lib.check(getattr(L, switch)(halo))
                _lib.check(L.ddnm_conv_tc_bench(N, H, H, Cin, Cout, mode, -iters, C.byref(ms), C.byref(fl)))
                t[halo].append(ms.value)
        _lib.check(getattr(L, switch)(1))
        m0, m1 = min(t[0]), min(t[1])
        if switch == "ddnm_tc_debug_pp_pair":   # the HALO form either way, the weights once or twice per pair of tiles
            f0, f1 = fill_bytes(H, H, Cin, Cout, up2, True), fill_bytes(H, H, Cin, Cout, up2, True, pair=True)
        else:
            f0, f1 = fill_bytes(H, H, Cin, Cout, up2, False), fill_bytes(H, H, Cin, Cout, up2, True)
        rows.append(dict(layer=label, ms_off=m0, ms_on=m1, tflops_off=fl.value / m0 / 1e9, tflops_on=fl.value / m1 / 1e9,
                         fill_mb_off=f0 / 1e6, fill_mb_on=f1 / 1e6))
        r = rows[-1]
        print(f"{label:28s} {r['ms_off']:8.3f} {r['ms_on']:8.3f} {100 * (r['ms_on'] / r['ms_off'] - 1):+6.1f}%  "
              f"{r['tflops_off']:6.1f} {r['tflops_on']:6.1f}  {r['fill_mb_off']:9.1f} {r['fill_mb_on']:9.1f}", flush=True)
    return rows


def forward_profiles(L, switch):
    ns = types.SimpleNamespace
    cfg = ns(model=ns(type="simple", ch=128, out_ch=3, ch_mult=[1, 1, 2, 2, 4, 4], num_res_blocks=2, attn_resolutions=[16], dropout=0.0,
                      in_channels=3, resamp_with_conv=True), data=ns(image_size=256), diffusion=ns(num_diffusion_timesteps=1000))
    sd = random_state_dict(cfg, 1234)
    torch.manual_seed(0)
    x = torch.randn(N, 3, 256, 256, device="cuda")
    t = torch.full((N,), 500.0, device="cuda")
    runs = {0: [], 1: []}
    for halo in (0, 1, 0, 1):
        _lib.check(getattr(L, switch)(halo))     # read when the engine builds its launches
        model = Model(cfg)
        model.load_state_dict(sd)
        model.profile(x, t)                      # warm-up: module load, first launches
        runs[halo].append(model.profile(x, t))
        model._destroy()
        del model
        torch.cuda.empty_cache()
    _lib.check(getattr(L, switch)(1))
    return runs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--switch", choices=sorted(SWITCHES), default="halo")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    L = _lib.lib()
    switch = SWITCHES[a.switch]
    print("GPU:", gpu_info(), "| switch:", a.switch, flush=True)
    print(f"\n[1] op-level, N = {N}, pseudo-random operands, best of 2 alternating runs of {a.iters} launches per arm")
    print(f"{'layer':28s} {'ms off':>8s} {'ms on':>8s} {'delta':>7s}  {'TF off':>6s} {'TF on':>6s}  {'fill MB off':>9s} {'fill MB on':>9s}")
    rows = bench_shapes(L, switch, a.iters)

    print("\n[2] eager forward, per tensor-core launch (second profile of each engine), arms alternated off/on/off/on")
    runs = forward_profiles(L, switch)
    tot = {h: [sum(o["ms"] for o in r) for r in runs[h]] for h in runs}
    tc = {h: [sum(o["ms"] for o in r if o["kind"] == "tc") for r in runs[h]] for h in runs}
    best = {h: min(range(2), key=lambda i: tot[h][i]) for h in runs}
    off, on = runs[0][best[0]], runs[1][best[1]]
    print(f"{'launch':40s} {'ms off':>8s} {'ms on':>8s} {'delta':>7s} {'TF off':>6s} {'TF on':>6s}")
    for o0, o1 in zip(off, on):
        if o0["kind"] != "tc" or o0["name"] != o1["name"]:
            continue
        tf = lambda o: o["flops"] / o["ms"] / 1e9 if o["ms"] > 0 else 0.0   # noqa: E731
        print(f"{o0['name']:40s} {o0['ms']:8.3f} {o1['ms']:8.3f} {100 * (o1['ms'] / o0['ms'] - 1):+6.1f}% {tf(o0):6.1f} {tf(o1):6.1f}")
    print(f"\nforward total ms  off: {', '.join(f'{v:.2f}' for v in tot[0])}   on: {', '.join(f'{v:.2f}' for v in tot[1])}")
    print(f"tc launches ms    off: {', '.join(f'{v:.2f}' for v in tc[0])}   on: {', '.join(f'{v:.2f}' for v in tc[1])}")
    print("GPU:", gpu_info(), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu_info(), switch=a.switch, shapes=rows, forward=dict(total_ms=tot, tc_ms=tc, off=off, on=on)), f, indent=1)


if __name__ == "__main__":
    main()
