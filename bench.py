#!/usr/bin/env python
"""bench.py — restored 256x256 images/sec @100 DDIM steps (BASELINE.json metric), one JSON line.

Default workload (BASELINE configs[1], `--config 2`): celeba_hq.yml denoiser (random init, seed 1234) x SuperResolution(4x average
pooling), sigma_y=0, T_sampling=100, eta=0.85, 16 images per GPU.  A "step" = one full sampling of the per-GPU batch.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--config 2|3|4|5a|5b] [--precision fp32|fp16]
                    [--dump-outputs DIR]

`value`  : the loop with x_T / y resident in HBM; the per-pair Gaussian draws ARE inside the timed region (drawn chunk by chunk on a
           side stream by ddnm_b200.sampler, like the reference's one randn_like per step).
`e2e`    : the public drop-in call (ddnm_diffusion / ddnm_plus_diffusion) with pinned HOST x_T / y and CPU results.
N>1 is launched by torchrun (one rank per GPU): rows shard over ranks, no traffic inside the loop, one all-gather of the restored
images per step (weak scaling); an untimed sharded-vs-unsharded check runs first (`shard_check`).
`--impl reference` times the UNMODIFIED reference (oracle/_ref, see oracle/make_ref.py) on the host cores on a bounded sample.
The other BASELINE configs (`--config 3|4|5a|5b`) and the fp16 fast mode print the same line for their workload.
`--dump-outputs DIR` writes what the timed path returned in its last timed step (x_0 and x0_pred of the batch) as float32 .npy files
under DIR, so that two builds can be compared output for output on identical seeded inputs.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

UNIT = "images/sec"
ETA, RES = 0.85, 256
CONFIGS = {
    # key: BASELINE.json configs index + 1 (SURVEY section 8d numbering)
    "2": dict(net="celeba", op="sr4", T=100, tl=1, tr=1, sigma_y=0.0, B=16,
              workload="celeba_hq.yml simple-UNet (113.7M params, random init seed 1234) + sr_averagepooling x4, sigma_y=0, T_sampling=100, eta=0.85, batch 16/GPU"),
    "3": dict(net="imagenet", op="color", T=100, tl=1, tr=1, sigma_y=0.0, B=8,
              workload="imagenet_256.yml UNetModel (552.8M params, random init seed 1234, learn_sigma) + colorization, sigma_y=0, T_sampling=100, eta=0.85, batch 8/GPU (64 over 8 GPUs)"),
    "4": dict(net="imagenet", op="inpaint", T=100, tl=3, tr=3, sigma_y=0.1, B=8,
              workload="imagenet_256.yml UNetModel + inpainting (exp/inp_masks/mask.npy), DDNM+ sigma_y=0.05 (0.1 internal), T_sampling=100, travel_length=3, travel_repeat=3 (298 UNet evals + 198 travel-back pairs), batch 8/GPU"),
    "5a": dict(net="celeba", op="deblur", T=250, tl=1, tr=1, sigma_y=0.0, B=16,
               workload="celeba_hq.yml simple-UNet + deblur_gauss (sigma 10, 5 taps), sigma_y=0, T_sampling=250, batch 16/GPU (128 over 8 GPUs)"),
    "5b": dict(net="celeba", op="wh", T=250, tl=1, tr=1, sigma_y=0.0, B=16,
               workload="celeba_hq.yml simple-UNet + cs_walshhadamard ratio 0.25, sigma_y=0, T_sampling=250, batch 16/GPU (128 over 8 GPUs)"),
}
STEP_KERNELS = {"sr4": 1, "color": 1, "inpaint": 1, "wh": 7, "deblur": 13}   # own launches of the fused per-pair update (operators.cu step())


def metric_name(c):
    return f"restored 256x256 images/sec @{c['T']} DDIM steps"


def peaks():
    try:
        p = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        return dict(hbm=p["hbm_gbs"], tf_burst=p["bf16_tflops"], tf_sust=p["bf16_tflops_sustained"], src="measured (MEASURED_PEAKS.json)")
    except Exception:
        # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 TFLOP/s dense FP16/BF16 — never reached, an upper bound only
        return dict(hbm=3350.0, tf_burst=989.0, tf_sust=989.0, src="H100 SXM data sheet (not measured)")


def sampler_cfg(c):
    import types
    ns = types.SimpleNamespace
    return ns(diffusion=ns(num_diffusion_timesteps=1000), time_travel=ns(T_sampling=c["T"], travel_length=c["tl"], travel_repeat=c["tr"]))


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms during the timed region (read-only queries)."""
    Q = "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, gpu_index):
        self.idx, self.p, self.path = gpu_index, None, f"/tmp/ddnm_clocks_{os.getpid()}.csv"

    def start(self):
        try:
            self.p = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "200", "-i", str(self.idx)],
                                      stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except Exception:
            self.p = None

    def stop(self):
        out = dict(sm_mhz=None, sm_max_mhz=None, reasons=[], power_w_max=None, samples=0)
        if self.p is None:
            return out
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except Exception:
            self.p.kill()
        sm, mx, pw, reasons = [], [], [], set()
        for line in open(self.path):
            f = [s.strip() for s in line.split(",")]
            if len(f) < 8:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2])); pw.append(float(f[3]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        if sm:
            sm.sort()
            out.update(sm_mhz=sm[len(sm) // 2], sm_max_mhz=max(mx), power_w_max=max(pw), samples=len(sm), reasons=sorted(reasons))
        try:
            os.remove(self.path)
        except OSError:
            pass
        return out


# torch's CPU conv path collapses when oversubscribed (one image-forward of the reference gets slower beyond ~16 threads on a
# many-core host), so the CPU arms run at no more than 16 threads
def cpu_threads():
    return min(os.cpu_count() or 1, 16)


def cpu_reference_rate(steps, warmup, sample_batch=2, sample_T=3):
    """Reference CPU path for configs[1] on the host cores.  kind "reference": the UNMODIFIED reference code (oracle/_ref: its own
    Model + SuperResolution + ddnm_diffusion, .to('cuda') redirected) on `sample_batch` images with a `sample_T`-step schedule;
    every DDIM step costs the same (one UNet forward + projection + re-noising), so images/sec @100 steps = rate x sample_T / 100.
    Falls back to the oracle port (kind "port") only if oracle/_ref was never built."""
    import torch
    nthreads = cpu_threads()
    T100 = CONFIGS["2"]["T"]
    from oracle import make_ref
    if make_ref.available():
        from oracle import ref_runner
        secs, resid = ref_runner.time_reference_sr4(sample_batch, sample_T, nthreads, repeats=warmup + steps)
        dt = sum(secs[warmup:]) / steps
        kind = "reference"
        what = (f"UNMODIFIED reference (functions/svd_ddnm.py::ddnm_diffusion + guided_diffusion/models.py::Model + "
                f"svd_operators.py::SuperResolution from oracle/_ref, torch CPU fp32), |A x0 - y| = {resid:.1e}")
    else:
        from oracle import operators as O, sampler as S, schedule as SCH, unet_simple as U
        torch.set_num_threads(nthreads)
        cfg = U.SimpleUNetConfig.celeba_hq()
        sd = U.init_state_dict(cfg, 1234)
        op = O.SuperResolution.make(3, RES, 4)
        g = torch.Generator().manual_seed(1234)
        x_orig = torch.rand(sample_batch, 3, RES, RES, generator=g) * 2 - 1
        y = op.A(x_orig.reshape(sample_batch, -1))
        x_T = torch.randn(sample_batch, 3, RES, RES, generator=g)
        betas = SCH.linear_betas()

        def one():
            with torch.no_grad():
                S.ddnm_sample(x_T, lambda a, b: U.forward(sd, a, b, cfg), betas, ETA, op, y,
                              lambda k: torch.randn(sample_batch, 3, RES, RES, generator=g), t_sampling=sample_T)
        for _ in range(warmup):
            one()
        t0 = time.perf_counter()
        for _ in range(steps):
            one()
        dt = (time.perf_counter() - t0) / steps
        kind, what = "port", "oracle port of the reference sampler (oracle/_ref absent), torch CPU fp32"
    rate = sample_batch / (dt / sample_T * T100)
    return rate, dt, dict(cores=nthreads, kind=kind,
                          sample=f"{sample_batch} images x a {sample_T}-step DDNM schedule per bench step ({what}; {nthreads} of {os.cpu_count()} host "
                                 f"threads: more threads are slower), scaled x{T100 / sample_T:.1f} to 100 steps (per-step cost is t-independent)")


def run_reference(args, emit):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    assert args.config == "2", "the reference arm is defined for configs[1] (celeba sr4)"
    c = CONFIGS["2"]
    steps, warm = max(1, min(args.steps, 3)), min(args.warmup, 1)
    rate, dt, cb = cpu_reference_rate(steps, warm)
    cb["value"], cb["unit"] = rate, UNIT
    line = dict(impl="reference", metric=metric_name(c), value=rate, unit=UNIT, n_gpus=args.gpus, steps=steps, warmup=warm,
                ms_per_step=dt * 1e3, higher_is_better=True, scaling="weak", vs_baseline=None, dtype="fp32", data="synthetic",
                config=dict(workload=c["workload"], note="CPU path of the reference; bounded sample, see cpu_baseline.sample"),
                cpu_baseline=cb, e2e=dict(value=rate, unit=UNIT, h2d_bytes_per_step=0, d2h_bytes_per_step=0), gpu_launches=0)
    emit(line)


def build_workload(c, dev, precision):
    """(model, operator, plus) of a config on `dev`; weights random-init seed 1234 (no checkpoints offline)."""
    import types
    import numpy as np
    import torch
    from ddnm_b200 import operators as E
    from ddnm_b200.model import Model, create_model
    from ddnm_b200.weights import random_state_dict, random_state_dict_openai
    ns = types.SimpleNamespace
    if c["net"] == "celeba":     # configs/celeba_hq.yml model section
        mcfg = ns(model=ns(type="simple", ch=128, out_ch=3, ch_mult=[1, 1, 2, 2, 4, 4], num_res_blocks=2, attn_resolutions=[16],
                           dropout=0.0, in_channels=3, resamp_with_conv=True),
                  data=ns(image_size=RES), diffusion=ns(num_diffusion_timesteps=1000))
        model = Model(mcfg)
        model.precision = precision
        model.load_state_dict(random_state_dict(mcfg, 1234))
    else:                        # configs/imagenet_256.yml model section
        model = create_model(image_size=256, num_channels=256, num_res_blocks=2, learn_sigma=True, attention_resolutions="32,16,8",
                             num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True, use_fp16=True)
        model.precision = precision
        model.load_state_dict(random_state_dict_openai(model, 1234))
    if c["op"] == "sr4":
        op = E.SuperResolution(3, RES, 4, dev)
    elif c["op"] == "color":
        op = E.Colorization(RES, dev)
    elif c["op"] == "inpaint":   # exp/inp_masks/mask.npy (bits shipped in the fixtures), index construction diffusion.py:466-470
        bits = np.load(os.path.join(ROOT, "tests", "golden", "fullsize.npz"))["mask_bits"]
        mask = torch.from_numpy(np.unpackbits(bits)[: RES * RES].astype(np.int64))
        mr = torch.nonzero(mask == 0).long().reshape(-1) * 3
        op = E.Inpainting(3, RES, torch.cat([mr, mr + 1, mr + 2]), dev)
    elif c["op"] == "deblur":    # diffusion.py:504-509
        sigma = 10
        pdf = lambda z: torch.exp(torch.Tensor([-0.5 * (z / sigma) ** 2]))   # noqa: E731
        k = torch.Tensor([pdf(-2), pdf(-1), pdf(0), pdf(1), pdf(2)])
        op = E.Deblurring((k / k.sum()).to(dev), 3, RES, dev)
    elif c["op"] == "wh":        # diffusion.py:455-459 (global-RNG randperm)
        op = E.WalshHadamardCS(3, RES, 4, torch.randperm(RES ** 2, generator=torch.Generator().manual_seed(1234)).to(dev), dev)
    else:
        raise KeyError(c["op"])
    return model, op, c["sigma_y"] > 0


DUMP_BUDGET = 64_000_000 - 4096   # bytes written by --dump-outputs, .npy headers included


def dump_outputs(d, arrays):
    """Each array as DIR/<name>.npy in float32.  Beyond an equal share of DUMP_BUDGET an array is replaced by a fixed, seeded sample of
    its flattened elements (the same positions on every run of the same shape)."""
    import numpy as np
    os.makedirs(d, exist_ok=True)
    share = DUMP_BUDGET // len(arrays) // 4
    for name, t in arrays.items():
        a = t.detach().float().cpu().numpy()
        if a.size > share:
            idx = np.sort(np.random.default_rng(1234).choice(a.size, share, replace=False))
            a = a.reshape(-1)[idx]
        np.save(os.path.join(d, name + ".npy"), np.ascontiguousarray(a, dtype=np.float32))


def main():
    # exactly ONE line on stdout: libraries (NCCL prints its version banner) write to fd 1, so park the real stdout and
    # point fd 1 at stderr until the JSON line is ready
    real_stdout = os.dup(1)
    os.dup2(2, 1)
    sys.stdout = os.fdopen(os.dup(2), "w")

    def emit(line):
        os.write(real_stdout, (json.dumps(line) + "\n").encode())

    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ddnm_b200")
    ap.add_argument("--config", default="2", choices=sorted(CONFIGS), help="BASELINE config (2 = configs[1], the driver's line)")
    ap.add_argument("--precision", default="fp32", choices=["fp32", "fp16"],
                    help="fp32 = fp32-grade 3x fp16 products (parity mode); fp16 = 1 product per MAC, the analogue of use_fp16 (NOT parity grade)")
    ap.add_argument("--batch", type=int, default=0, help="images per GPU (default: the config's)")
    ap.add_argument("--e2e-steps", type=int, default=0, help="timed steps of the end-to-end leg (default: --steps)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--profile-steps", type=int, default=0, help="(profiler runs) skip the e2e / baseline legs")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="write the last timed step's outputs (x0, x0_pred) as float32 .npy files under DIR (at most 64 MB in all)")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args, emit)
    assert args.warmup >= 3 or args.profile_steps, "timing rules: at least 3 warm-up steps"

    import torch
    import torch.distributed as dist
    from ddnm_b200.parallel import shard_rows, sharded_sample
    from ddnm_b200.sampler import ddnm_diffusion, ddnm_plus_diffusion, sample_device
    from ddnm_b200.schedule import time_pairs
    import types

    c = dict(CONFIGS[args.config])
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world} (launch N>1 with torchrun)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    B = args.batch or c["B"]
    model, op, plus = build_workload(c, dev, args.precision)
    sy = c["sigma_y"]
    conf = sampler_cfg(c)
    betas = torch.from_numpy(__import__("numpy").linspace(1e-4, 2e-2, 1000, dtype="float64")).float().to(dev)
    pairs = time_pairs(1000, c["T"], c["tl"], c["tr"])
    n_pairs, evals = len(pairs), sum(1 for i, j in pairs if j < i)

    # global synthetic batch (identical on every rank), sharded by rows
    Bg = B * world
    g = torch.Generator().manual_seed(1234)
    x_orig = torch.rand(Bg, 3, RES, RES, generator=g) * 2 - 1
    x_T_host = torch.randn(Bg, 3, RES, RES, generator=g).pin_memory()
    lo = rank * B
    y_dev = op.A(x_orig[lo:lo + B].to(dev))
    if plus:
        y_dev = y_dev + sy * torch.randn(y_dev.shape, generator=g).to(dev)
    y_host = y_dev.cpu().pin_memory()
    x_T_dev = x_T_host[lo:lo + B].to(dev)
    torch.manual_seed(1234 + rank)       # per-pair draws differ per rank (independent trajectories)

    def local_fn(xr, yr, nz=None):
        return sample_device(xr, model, betas, ETA, op, yr, sy, plus, conf, noise=nz)

    # ---- untimed: sharded == unsharded on this hardware (SURVEY section 4).  A short schedule over the global batch through
    # parallel.sharded_sample (rows sharded, one all-gather); every rank then recomputes ANOTHER rank's rows itself and compares.
    shard_check = None
    if world > 1:
        cs = dict(c, T=3, tl=1, tr=1)
        conf_s = sampler_cfg(cs)
        gs = torch.Generator().manual_seed(4321)
        xs_g = torch.randn(Bg, 3, RES, RES, generator=gs).to(dev)
        tape = torch.randn(3, Bg, 3, RES, RES, generator=gs).to(dev)
        ys_g = op.A(x_orig.to(dev))
        fn = lambda xr, yr, nz: sample_device(xr, model, betas, ETA, op, yr, 0.0, False, conf_s, noise=nz.contiguous())   # noqa: E731
        full0, _ = sharded_sample(fn, xs_g, ys_g, tape)
        other = (rank + 1) % world
        l2, h2 = shard_rows(Bg, other, world)
        mine, _ = fn(xs_g[l2:h2], ys_g[l2:h2], tape[:, l2:h2])
        diff = torch.tensor([(mine - full0[l2:h2]).abs().max().item()], device=dev)
        dist.all_reduce(diff, op=dist.ReduceOp.MAX)
        shard_check = dict(max_abs_diff=diff.item(), rows=Bg, T_sampling=3,
                           note="parallel.sharded_sample over the global batch vs each rank recomputing the next rank's rows; bit-identical expected")
        del xs_g, tape, ys_g, full0, mine

    last = {}

    def step_device():
        # hot path with x_T / y resident in HBM, draws included (+ the single end-of-run all-gather when N > 1)
        x0, x0p = local_fn(x_T_dev, y_dev)
        last["out"] = (x0, x0p)
        if world == 1:
            return x0, x0p
        outs = [torch.empty_like(x0) for _ in range(world)]
        dist.all_gather(outs, x0)
        last["out"] = (torch.cat(outs), x0p)
        return outs, x0p

    def step_e2e():
        # public API with HOST buffers: H2D of x_T and y, noise drawn by the API, D2H of both results
        if plus:
            return ddnm_plus_diffusion(x_T_host[lo:lo + B], model, betas, ETA, op, y_host, sy, config=conf)
        return ddnm_diffusion(x_T_host[lo:lo + B], model, betas, ETA, op, y_host, config=conf)

    def timed(fn, steps, warm):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.barrier()
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return ms.item()

    if args.profile_steps:      # profiler launch list: just run the hot path
        for _ in range(args.profile_steps):
            step_device()
        torch.cuda.synchronize()
        emit(dict(note="profile run, no timing"))
        return

    clocks = ClockSampler(local)
    clocks.start()
    ms_total = timed(step_device, args.steps, args.warmup)
    clk = clocks.stop()
    if args.dump_outputs:
        x0_all, x0p = last["out"]
        if world > 1:   # x0_pred of every rank (outside the timed region: the timed step gathers x0 only)
            parts = [torch.empty_like(x0p) for _ in range(world)]
            dist.all_gather(parts, x0p)
            x0p = torch.cat(parts)
        if rank == 0:
            dump_outputs(args.dump_outputs, dict(x0=x0_all, x0_pred=x0p))
    e2e_steps = args.e2e_steps or args.steps
    ms_e2e = timed(step_e2e, e2e_steps, 2)
    ms_step = ms_total / args.steps
    value = Bg * 1e3 / ms_step
    e2e_value = Bg * 1e3 / (ms_e2e / e2e_steps)

    if rank == 0:
        info = model.info(B)
        pk = peaks()
        # roofline of the dominant kernel family (the wgmma convolution): per-launch CUDA-event timing of one eager forward
        xt = torch.randn(B, 3, RES, RES, device=dev)
        # three eager passes, per launch the fastest: in the regions of short launches the elapsed time between two events measures the
        # host's issue rate rather than the kernel, and that jitter is one-sided
        tt = torch.full((B,), 500.0, device=dev)
        prof = model.profile(xt, tt)
        for _ in range(2):
            for a, b in zip(prof, model.profile(xt, tt)):
                a["ms"] = min(a["ms"], b["ms"])
        tc = [p for p in prof if p["kind"] == "tc"]
        tc_ms, tc_fl = sum(p["ms"] for p in tc), sum(p["flops"] for p in tc)
        all_ms = sum(p["ms"] for p in prof)
        ach = tc_fl / tc_ms / 1e9 if tc_ms > 0 else 0.0
        fwd_launches = sum(4 if p["kind"] == "temb" else (0 if p["kind"] == "memset" else 1) for p in prof)
        terms = 3 if args.precision == "fp32" else 1
        roof = dict(bound="tensor", kernel="conv_tc_kernel (wgmma implicit GEMM, TMA-staged, register accumulators)", achieved=ach,
                    peak=pk["tf_sust"], unit="TFLOP/s", frac=ach / pk["tf_sust"], hw_mma_factor=terms, frac_hw=terms * ach / pk["tf_sust"],
                    peak_source=pk["src"],
                    launches_per_forward=len(tc), avg_launch_ms=tc_ms / max(1, len(tc)), share_of_forward=tc_ms / all_ms,
                    note=f"achieved = algorithmic conv/GEMM FLOPs (2*M*N*K once) / summed per-launch CUDA-event time; each algorithmic MAC costs {terms} fp16 MMA(s)"
                         + (" (hi*hi+hi*lo+lo*hi) for fp32-grade products, so frac_hw = 3*frac is the tensor-pipe utilisation and 1/3 the ceiling of frac" if terms == 3 else ""))
        line = dict(metric=metric_name(c), value=value, unit=UNIT, n_gpus=world, steps=args.steps, warmup=args.warmup, ms_per_step=ms_step,
                    higher_is_better=True, scaling="weak", vs_baseline=None, dtype="fp32" if args.precision == "fp32" else "fp16", data="synthetic",
                    config=dict(workload=c["workload"], baseline_config=args.config, precision=args.precision, global_batch=Bg,
                                parallelism=f"rows sharded over {world} GPU(s), 1 all-gather at the end",
                                noise="per-pair Gaussian draws inside the timed region (side stream, bounded double buffer)",
                                l2="working set per UNet forward (GiBs of activations) exceeds the 50 MB L2; no flush needed",
                                gpu=torch.cuda.get_device_name(dev),
                                unet_ms_per_forward=all_ms, unet_evals_per_image=evals, time_pairs=n_pairs,
                                unet_flops_per_image_forward=info["flops_per_forward"] / B, workspace_bytes=info["workspace_bytes"]),
                    clocks=clk, roofline=roof,
                    e2e=dict(value=e2e_value, unit=UNIT, h2d_bytes_per_step=int(B * 3 * RES * RES * 4 + B * op.y_dim * 4) * world,
                             d2h_bytes_per_step=int(2 * B * 3 * RES * RES * 4) * world, steps=e2e_steps, warmup=2,
                             note="ddnm_b200.sampler.ddnm_diffusion / ddnm_plus_diffusion with pinned host x_T / y, noise drawn inside the call, results returned as CPU tensors"),
                    gpu_launches=int(args.steps * (evals * (fwd_launches + 1 + STEP_KERNELS[c["op"]]) + (n_pairs - evals) + n_pairs)))
        if shard_check is not None:
            line["shard_check"] = shard_check
        if not args.no_cpu_baseline and world == 1 and args.config == "2":
            rate, dt, cb = cpu_reference_rate(1, 0)
            cb["value"], cb["unit"] = rate, UNIT
            line["cpu_baseline"] = cb
        else:
            line["cpu_baseline"] = None
        emit(line)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
