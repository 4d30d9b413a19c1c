"""Times classifier guidance on the GPU, imagenet_256_cc.yml shapes, random weights, one JSON line with the GPU's name, power limit
and median SM clock:
  * per call: ddnm_classifier_grad (the library's forward + backward, CUDA graph) against PyTorch autograd through the torch
    restatement of EncoderUNetModel (oracle/classifier.py: the reference module's layers as the same torch calls; cuDNN defaults)
    in fp32 and with the torso in fp16 (what convert_to_fp16 does to the reference module);
  * the guided loop (class-conditional UNetModel + classifier, 4x SR, --pairs denoising pairs): images/s with the native gradient
    against the Python-callback path running the fp32 autograd cond_fn, arms alternated --rounds times.

    python tools/classifier_bench.py [--batch 8] [--iters 10] [--pairs 4] [--rounds 2]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def guided_loop(clf, sd, cfg, B, pairs, rounds):
    """images/s of ddnm_diffusion with the imagenet_256_cc.yml UNetModel and classifier: native guidance vs the Python callback"""
    import types
    from ddnm_b200.guidance import make_cond_fn
    from ddnm_b200.model import create_model
    from ddnm_b200.operators import SuperResolution
    from ddnm_b200.sampler import ddnm_diffusion
    from ddnm_b200.weights import random_state_dict_openai
    from oracle import classifier as OC
    from oracle.schedule import linear_betas
    ns = types.SimpleNamespace
    unet = create_model(image_size=256, num_channels=256, num_res_blocks=2, learn_sigma=True, class_cond=True, attention_resolutions="32,16,8",
                        num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True)
    usd = random_state_dict_openai(unet, 1234)   # draws no label embedding: nn.Embedding's N(0, 1) init (unet.py:478-479)
    usd["label_emb.weight"] = torch.randn(1000, 4 * 256, generator=torch.Generator().manual_seed(1235))
    unet.load_state_dict(usd)
    op = SuperResolution(3, 256, 4, torch.device("cuda"))
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 3, 256, 256, generator=g).cuda()
    y = op.A(x)
    conf = ns(diffusion=ns(num_diffusion_timesteps=1000), time_travel=ns(T_sampling=pairs, travel_length=1, travel_repeat=1))
    betas = linear_betas().cuda()
    arms = {"native": make_cond_fn(clf, 10.0), "callback": OC.cond_fn(sd, cfg, 10.0)}
    res = {k: [] for k in arms}
    for r in range(rounds + 1):               # round 0 warms both arms up (engines, graphs, cuDNN algorithms)
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ddnm_diffusion(x, unet, betas, 0.85, op, y, cls_fn=fn, config=conf)
            torch.cuda.synchronize()
            if r:
                res[k].append(B / (time.perf_counter() - t0))
    return dict(pairs=pairs, images_per_s={k: [round(v, 4) for v in vs] for k, vs in res.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--pairs", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    from ddnm_b200.model import create_classifier
    from ddnm_b200.weights import random_state_dict_classifier
    from oracle import classifier as OC
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    cfg = OC.ClassifierConfig.imagenet_256()
    m = create_classifier(256, False, 128, 2, "32,16,8", True, True, "attention")
    sd = random_state_dict_classifier(m, 1234)
    m.load_state_dict(sd)
    B = a.batch
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, 256, 256, generator=g).cuda()
    t = torch.full((B,), 500.0, device="cuda")
    y = torch.arange(B, device="cuda") * 97 % 1000
    clocks, stop = [], threading.Event()

    def sample():
        while not stop.is_set():
            v = smi("clocks.sm")
            if v.isdigit():
                clocks.append(int(v))
            time.sleep(0.5)
    th = threading.Thread(target=sample, daemon=True)
    th.start()
    native = timed(lambda: m.grad(x, t, y, 10.0), a.iters)
    sdc = {k: v.cuda() for k, v in sd.items()}
    ref_fn = OC.cond_fn(sdc, cfg, 10.0)
    torch_fp32 = timed(lambda: ref_fn(x, t, y), a.iters)
    ref16 = OC.cond_fn(sdc, cfg, 10.0, torso_dtype=torch.float16)
    torch_fp16 = timed(lambda: ref16(x, t, y), a.iters)
    loop = guided_loop(m, sdc, cfg, B, a.pairs, a.rounds)
    stop.set()
    th.join()
    gn = m.grad(x, t, y, 10.0)
    gr = ref_fn(x, t, y)
    info = m.info(B)
    prof = m.profile(x, t) if os.environ.get("CLS_PROFILE") else None
    res = dict(gpu=torch.cuda.get_device_name(0), power_limit_w=smi("power.limit"), median_sm_clock_mhz=statistics.median(clocks) if clocks else None,
               batch=B, native_ms=native, torch_autograd_fp32_ms=torch_fp32, torch_autograd_fp16_torso_ms=torch_fp16, guided_loop=loop, workspace_bytes=info["workspace_bytes"], launches=info["launches"],
               rel_diff_native_vs_torch=((gn - gr).norm() / gr.norm()).item(), max_abs_grad=gr.abs().max().item())
    print(json.dumps(res))
    if prof:
        agg = {}
        for op in prof:
            agg[op["kind"]] = agg.get(op["kind"], 0) + op["ms"]
        print(json.dumps({k: round(v, 3) for k, v in sorted(agg.items(), key=lambda kv: -kv[1])}))


if __name__ == "__main__":
    main()
