"""Cost of the batch-invariant mode on the GPU: each measurement alternates mode off / on, `--rounds` times in one process, and prints
one JSON line with the GPU's name and power limit.

  celeba_fwd_ms    celeba_hq.yml Model forward, B = 16, CUDA graph (median of --iters per round)
  bench_img_s      bench.py's default workload: celeba Model + sr_averagepooling x4, T_sampling = 100, eta 0.85, 16 images, seeded
  imagenet_fwd_ms  imagenet_256.yml UNetModel forward, B = 8
  clf_grad_ms      imagenet_256_cc.yml classifier, ddnm_classifier_grad (logits + input gradient), B = 8

  python tools/batch_invariant_bench.py [--rounds 3] [--iters 20]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from classifier_bench import smi, timed   # noqa: E402


def pair(make):
    """(model off, model on) built by make()"""
    off, on = make(), make()
    on.batch_invariant = True
    return off, on


def alternate(fns, rounds):
    """{mode: [value per round]} with the modes taking turns"""
    out = {"off": [], "on": []}
    for _ in range(rounds):
        for mode in ("off", "on"):
            out[mode].append(fns[mode]())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    import bench
    from ddnm_b200.model import EncoderUNetModel, create_model
    from ddnm_b200.sampler import ddnm_diffusion
    from ddnm_b200.weights import random_state_dict_classifier, random_state_dict_openai
    from oracle import classifier as OC
    from oracle.schedule import linear_betas

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"), "rounds": args.rounds}
    g = torch.Generator().manual_seed(0)

    def ms(m, *a):
        def f():
            with torch.no_grad():
                return timed(lambda: m(*a), args.iters)[0]
        return f

    # celeba forward and the bench workload
    c = bench.CONFIGS["2"]
    (m_off, op), (m_on, _) = [bench.build_workload(c, dev, "fp32")[:2] for _ in range(2)]
    m_on.batch_invariant = True
    x = torch.randn(16, 3, 256, 256, generator=g).to(dev)
    t = torch.randint(0, 1000, (16,), generator=g).float().to(dev)
    res["celeba_fwd_ms"] = alternate({"off": ms(m_off, x, t), "on": ms(m_on, x, t)}, args.rounds)
    y = op.A(torch.rand(16, 3, 256, 256, generator=g).to(dev) * 2 - 1)
    conf = bench.sampler_cfg(c)
    betas = linear_betas().to(dev)

    def e2e(m):
        def f():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ddnm_diffusion(x, m, betas, 0.85, op, y, config=conf, seed=1234)
            torch.cuda.synchronize()
            return 16 / (time.perf_counter() - t0)
        return f
    e2e(m_off)(), e2e(m_on)()   # engines, graphs, buffers
    res["bench_img_s"] = alternate({"off": e2e(m_off), "on": e2e(m_on)}, args.rounds)
    del m_off, m_on

    # imagenet UNetModel forward
    def imagenet():
        m = create_model(image_size=256, num_channels=256, num_res_blocks=2, learn_sigma=True, attention_resolutions="32,16,8",
                         num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True, use_fp16=True)
        m.load_state_dict(random_state_dict_openai(m, 1234))
        return m
    u_off, u_on = pair(imagenet)
    res["imagenet_fwd_ms"] = alternate({"off": ms(u_off, x[:8], t[:8]), "on": ms(u_on, x[:8], t[:8])}, args.rounds)
    del u_off, u_on

    # classifier gradient
    cfg = OC.ClassifierConfig.imagenet_256()

    class Shape:
        model_channels, channel_mult, in_channels, num_res_blocks = cfg.model_channels, cfg.channel_mult, 3, cfg.num_res_blocks
        attention_resolutions, pool, image_size, out_channels = cfg.attention_resolutions, cfg.pool, cfg.image_size, cfg.out_channels
    sd = random_state_dict_classifier(Shape, 1234)

    def clf():
        m = EncoderUNetModel(**cfg.kwargs())
        m.load_state_dict(sd)
        return m
    c_off, c_on = pair(clf)
    labels = torch.arange(8, device=dev) * 100
    res["clf_grad_ms"] = alternate({"off": ms(lambda a, b: c_off.grad(a, b, labels, 1.0), x[:8], t[:8]),
                                    "on": ms(lambda a, b: c_on.grad(a, b, labels, 1.0), x[:8], t[:8])}, args.rounds)
    for k in ("celeba_fwd_ms", "bench_img_s", "imagenet_fwd_ms", "clf_grad_ms"):
        v = res[k]
        res[k + "_median"] = {mode: round(statistics.median(v[mode]), 4) for mode in v}
        v["off"] = [round(a, 4) for a in v["off"]]
        v["on"] = [round(a, 4) for a in v["on"]]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
