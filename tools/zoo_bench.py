"""Times guided-diffusion's published ImageNet UNets on the GPU (random weights, fp32-grade parity mode), prints one JSON line per
measurement and a summary line with the GPU's name and power limit:
  * per network (64x64 base, 128x128 base, 64 -> 256 and 128 -> 512 upsamplers) at a batch that fits: one CUDA-graph forward,
    CUDA events around each of --iters launches (median, min, max), and the per-op split of one eager forward from profile():
    attention (qkv split, Q K^T, softmax, V transpose, P V) against the tensor-core convolutions and the rest; for the 64 -> 256
    upsampler the launches of its 96-wide attention heads are listed one by one;
  * the two-stage 64 -> 256 pipeline (superres.sample_then_upsample, classifier-guided at both stages, T = --steps): images/s.

    python tools/zoo_bench.py [--iters 20] [--steps 100] [--pipe-batch 4]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NETS = [("base64", 16), ("base128", 8), ("up256", 4), ("up512", 1)]   # (published shape, batch)
ATTN_PARTS = (".qkv_split", ".qk", ".softmax", ".v_transpose", ".pv")


def smi(q):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                              text=True, timeout=20).stdout.strip()
    except Exception:   # noqa: BLE001
        return "n/a"


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts), min(ts), max(ts)


def split(ops):
    """ms per group: attention core ops, convolutions (tensor-core launches that are not attention), everything else"""
    out = {"attention_ms": 0.0, "conv_ms": 0.0, "other_ms": 0.0}
    for o in ops:
        if any(o["name"].endswith(s) for s in ATTN_PARTS):
            out["attention_ms"] += o["ms"]
        elif o["kind"] == "tc" or o["name"].endswith(".splitk_reduce"):
            out["conv_ms"] += o["ms"]
        else:
            out["other_ms"] += o["ms"]
    return {k: round(v, 3) for k, v in out.items()}


def model(cfg):
    from ddnm_b200.model import SuperResModel, UNetModel
    from oracle import gen_zoo_golden as G
    kw = cfg.reference_kwargs()
    m = SuperResModel(**kw, small_size=cfg.small_size) if cfg.small_size else UNetModel(**kw)
    m.load_state_dict(G.state_dict(cfg))
    return m


def net(key, B, iters):
    from oracle import gen_zoo_golden as G
    cfg = dict((c[0], c[1]) for c in G.published_cases())[key]
    m = model(cfg)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(B, 3, cfg.image_size, cfg.image_size, device="cuda", generator=g)
    t = torch.full((B,), 500.0, device="cuda")
    y = torch.randint(0, 1000, (B,), device="cuda", generator=g)
    low = torch.rand(B, 3, cfg.small_size, cfg.small_size, device="cuda", generator=g) * 2 - 1 if cfg.small_size else None
    fwd = (lambda: m(x, t, y, low_res=low)) if low is not None else (lambda: m(x, t, y))   # noqa: E731
    med, lo, hi = timed(fwd, iters)
    ops = m.profile(x, t)   # eager, with the labels and low_res the timed forwards staged
    rec = dict(net=key, batch=B, image_size=cfg.image_size, graph_forward_ms=round(med, 3), min_ms=round(lo, 3), max_ms=round(hi, 3),
               images_per_s=round(B / med * 1e3, 2), eager_profile_ms=round(sum(o["ms"] for o in ops), 3), **split(ops))
    if key == "up256":
        # the 32 x 32 attention blocks: 4 heads of 96, Q K^T and P V of 2 * B * 4 * T^2 * 96 flops each (T = 1024)
        f96 = 2.0 * B * 4 * 1024 * 1024 * 96
        rec["attn96"] = [dict(name=o["name"], kind=o["kind"], ms=round(o["ms"], 4), tflops=round(o["flops"] / o["ms"] / 1e9, 1))
                         for o in ops if o["name"].endswith((".qk", ".pv")) and abs(o["flops"] - f96) <= 1e-4 * f96]
    print(json.dumps(rec), flush=True)
    del m
    torch.cuda.empty_cache()
    return rec


def pipeline(steps, B):
    import types
    from ddnm_b200.guidance import make_cond_fn
    from ddnm_b200.model import EncoderUNetModel
    from ddnm_b200.operators import SuperResolution
    from ddnm_b200.superres import sample_then_upsample
    from ddnm_b200.weights import random_state_dict_classifier
    from oracle import gen_zoo_golden as G
    from oracle.classifier import ClassifierConfig
    from oracle.gen_classifier_golden import shape
    from oracle.schedule import linear_betas
    ns = types.SimpleNamespace
    cfgs = dict((c[0], c[1]) for c in G.published_cases())
    base, sr = model(cfgs["base64"]), model(cfgs["up256"])

    def classifier(cfg):
        c = EncoderUNetModel(**cfg.kwargs())
        c.load_state_dict(random_state_dict_classifier(shape(cfg), 1234))
        return make_cond_fn(c, 1.0)
    cls_fn = classifier(dict((c[0], c[1]) for c in G.classifier_cases())["cls64"])
    sr_cls_fn = classifier(ClassifierConfig.imagenet_256())
    g = torch.Generator(device="cuda").manual_seed(3)
    A = SuperResolution(3, 64, 4, "cuda")
    y = A.A(torch.rand(B, 3, 64, 64, device="cuda", generator=g) * 2 - 1)
    x_T, x_T_sr = torch.randn(B, 3, 64, 64, device="cuda", generator=g), torch.randn(B, 3, 256, 256, device="cuda", generator=g)
    conf = ns(diffusion=ns(num_diffusion_timesteps=1000), time_travel=ns(T_sampling=steps, travel_length=1, travel_repeat=1))
    betas = linear_betas().cuda()
    run = lambda: sample_then_upsample(x_T, base, betas, 0.85, A, y, sr, x_T_sr, config=conf, cls_fn=cls_fn, sr_cls_fn=sr_cls_fn,  # noqa: E731
                                       seed=5)
    run()   # engines, graphs
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    rec = dict(pipeline="64->256 sample_then_upsample, classifier-guided", steps=steps, batch=B, seconds=round(dt, 3),
               images_per_s=round(B / dt, 4))
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--pipe-batch", type=int, default=4)
    ap.add_argument("--nets", default=",".join(k for k, _ in NETS))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("zoo_bench measures on the GPU; no CUDA device is visible")
    info = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=smi("power.limit"), sm_clock_mhz=smi("clocks.sm"))
    print(json.dumps(info), flush=True)
    recs = [net(k, B, a.iters) for k, B in NETS if k in a.nets.split(",")]
    recs.append(pipeline(a.steps, a.pipe_batch))
    print(json.dumps(dict(summary=recs, **info)), flush=True)


if __name__ == "__main__":
    main()
