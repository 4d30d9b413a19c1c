"""Torch-drawn noise against library-seeded noise on the sampling loop: images/s and peak memory of each arm.

Two workloads, both on the 256 x 256 celeba_hq denoiser with random weights: BASELINE config 2 (4x SR, DDNM, T = 100) and the
shape of config 4 (inpainting, DDNM+, travel_length = travel_repeat = 3: 496 pairs at T = 100).  The arms alternate, ``--repeats``
times each in one process, after one warm-up run per arm; a device synchronise closes every timed run.  The card's name, power
limit and maximum SM clock are printed with the numbers.  There is no CPU path: without a CUDA device the script fails.

    python tools/noise_bench.py [--batch 16] [--steps 100] [--repeats 3] [--configs sr4 inpaint_plus]

The sampler-step kernels are ~1 % of such a run (the denoiser is the rest), so the end-to-end rate is not expected to move; the
step kernels' own time is not measured here.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {"sr4": dict(plus=False, tl=1, tr=1), "inpaint_plus": dict(plus=True, tl=3, tr=3)}


def parse(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--batch", type=int, default=16)
    p.add_argument("--steps", type=int, default=100, help="T_sampling")
    p.add_argument("--repeats", type=int, default=3, help="timed runs per arm (arms alternate)")
    p.add_argument("--configs", nargs="+", default=list(CONFIGS), choices=list(CONFIGS))
    p.add_argument("--seed", type=int, default=1234)
    a = p.parse_args(argv)
    if a.batch < 1 or a.steps < 1 or a.repeats < 1:
        p.error("--batch, --steps and --repeats must be >= 1")
    return a


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi query failed)"


def main(argv=None):
    a = parse(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("noise_bench needs a CUDA device (H100): there is no CPU path")
    from ddnm_b200 import operators as E
    from ddnm_b200.model import Model
    from ddnm_b200.sampler import sample_device
    from ddnm_b200.schedule import time_pairs
    from ddnm_b200.weights import random_state_dict
    dev, R, B = "cuda", 256, a.batch
    ns = types.SimpleNamespace
    mc = ns(model=ns(type="simple", ch=128, out_ch=3, ch_mult=[1, 1, 2, 2, 4, 4], num_res_blocks=2, attn_resolutions=[16], dropout=0.0,
                     in_channels=3, resamp_with_conv=True), data=ns(image_size=R), diffusion=ns(num_diffusion_timesteps=1000))
    model = Model(mc)
    model.load_state_dict(random_state_dict(mc, 1234))
    betas = torch.linspace(1e-4, 2e-2, 1000, dtype=torch.float64).float().to(dev)
    g = torch.Generator().manual_seed(0)
    missing = torch.nonzero(torch.rand(R * R, generator=g) < 0.5).long().reshape(-1) * 3
    ops = {"sr4": lambda: E.SuperResolution(3, R, 4, dev),
           "inpaint_plus": lambda: E.Inpainting(3, R, torch.cat([missing, missing + 1, missing + 2]), dev)}
    x_T = torch.randn(B, 3, R, R, device=dev)
    x = torch.rand(B, 3, R, R, device=dev) * 2 - 1
    info = card()
    for name in a.configs:
        c = CONFIGS[name]
        op = ops[name]()
        y = op.A(x)
        conf = ns(diffusion=ns(num_diffusion_timesteps=1000), time_travel=ns(T_sampling=a.steps, travel_length=c["tl"], travel_repeat=c["tr"]))
        n_pairs = len(time_pairs(1000, a.steps, c["tl"], c["tr"]))
        arms = {"torch_drawn": {}, "seeded": dict(seed=a.seed)}
        rates = {k: [] for k in arms}
        peaks = {k: 0 for k in arms}

        def run(kw):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            t0 = time.perf_counter()
            sample_device(x_T, model, betas, 0.85, op, y, 0.1 if c["plus"] else 0.0, c["plus"], conf, **kw)
            torch.cuda.synchronize()
            return B / (time.perf_counter() - t0), torch.cuda.max_memory_allocated() - base
        for kw in arms.values():
            run(kw)                                             # warm-up: engine build, graph capture, scratch
        for _ in range(a.repeats):
            for arm, kw in arms.items():
                r, pk = run(kw)
                rates[arm].append(r)
                peaks[arm] = max(peaks[arm], pk)
        print(json.dumps({"config": name, "card": info, "batch": B, "T_sampling": a.steps, "n_pairs": n_pairs,
                          "images_per_s": {k: [round(v, 4) for v in rates[k]] for k in arms},
                          "peak_bytes_over_call": peaks}), flush=True)


if __name__ == "__main__":
    main()
