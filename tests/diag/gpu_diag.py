"""GPU diagnostics for the tensor-core path (run on an H100; each group in its own process).
Lives under tests/ because several groups use the oracle as their checker (oracle/ is test infrastructure only)."""
import ctypes as C
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from ddnm_b200 import _lib  # noqa: E402

if os.environ.get("DDNM_DIAG_LIB"):      # A/B runs of two builds on one box: point the binding at another .so before it loads
    _lib.LIB_PATH = os.path.abspath(os.environ["DDNM_DIAG_LIB"])

L = _lib.lib()
dev = "cuda"


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def conv_tc(x, w, b, mode=0, up2=False, side=None, side_w=None, res=None):
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    oH, oW = (H // 2, W // 2) if mode == 2 else ((2 * H, 2 * W) if up2 else (H, W))
    out = torch.empty(N, oH, oW, Cout, device=dev)
    xs = nhwc(x)
    sx = nhwc(side) if side is not None else None
    rs = nhwc(res) if res is not None else None
    _lib.check(L.ddnm_conv_tc(_lib.ptr(xs), N, H, W, Cin, _lib.ptr(w.contiguous()), _lib.ptr(b), Cout, mode, int(up2),
                              _lib.ptr(sx), 0 if side is None else side.shape[1],
                              _lib.ptr(side_w.contiguous()) if side_w is not None else None, _lib.ptr(rs), _lib.ptr(out), None))
    torch.cuda.synchronize()
    return out.permute(0, 3, 1, 2)


def ref_conv(x, w, b, mode=0, up2=False, side=None, side_w=None, res=None):
    x, w, b = x.double().cpu(), w.double().cpu(), b.double().cpu()
    if up2:
        x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    if mode == 0:
        o = F.conv2d(x, w, b, padding=1)
    elif mode == 1:
        o = F.conv2d(x, w, b)
    else:
        o = F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)
    if side is not None:
        o = o + F.conv2d(side.double().cpu(), side_w.double().cpu())
    if res is not None:
        o = o + res.double().cpu()
    return o


def report(name, got, ref):
    got = got.double().cpu()
    err = (got - ref).abs()
    scale = ref.abs().max().item()
    print(f"[{name}] max_abs_err {err.max().item():.3e}  ref_absmax {scale:.3e}  rel {err.max().item() / max(scale, 1e-30):.3e}"
          f"  mean_err {err.mean().item():.3e}", flush=True)
    bad = err.max().item() > 1e-4 * max(scale, 1.0)
    if bad:
        e = err[0]
        print("   err by out-channel block of 8 (first 8):", [f"{e[c*8:(c+1)*8].max().item():.2e}" for c in range(min(8, e.shape[0] // 8))])
        print("   err by row (first 8):", [f"{e[:, r].max().item():.2e}" for r in range(min(8, e.shape[1]))])
        print("   err by col (first 16):", [f"{e[:, :, c].max().item():.2e}" for c in range(min(16, e.shape[2]))])
        print("   sample got/ref [0,0,0,:6]:", got[0, 0, 0, :6].tolist(), ref[0, 0, 0, :6].tolist())
    return not bad


def group_gemm():
    torch.manual_seed(0)
    ok = True
    for (N, H, W, Cin, Cout) in [(1, 1, 128, 64, 64), (1, 2, 128, 64, 128), (1, 4, 128, 128, 256), (2, 8, 16, 192, 128),
                                 (3, 8, 8, 64, 64), (1, 16, 16, 512, 1536)]:
        x = torch.randn(N, Cin, H, W, device=dev)
        w = torch.randn(Cout, Cin, 1, 1, device=dev) / Cin ** 0.5
        b = torch.randn(Cout, device=dev)
        ok &= report(f"gemm1x1 N{N} {H}x{W} {Cin}->{Cout}", conv_tc(x, w, b, mode=1), ref_conv(x, w, b, mode=1))
    print("GROUP gemm:", "PASS" if ok else "FAIL")


def group_conv():
    torch.manual_seed(1)
    ok = True
    for (N, H, W, Cin, Cout) in [(1, 16, 16, 64, 64), (2, 32, 32, 128, 128), (1, 64, 64, 128, 256), (1, 256, 256, 64, 128),
                                 (3, 8, 8, 128, 64), (1, 128, 128, 192, 128)]:
        x = torch.randn(N, Cin, H, W, device=dev)
        w = torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5
        b = torch.randn(Cout, device=dev)
        ok &= report(f"conv3x3 N{N} {H}x{W} {Cin}->{Cout}", conv_tc(x, w, b, mode=0), ref_conv(x, w, b, mode=0))
    print("GROUP conv3x3:", "PASS" if ok else "FAIL")


def group_variants():
    torch.manual_seed(2)
    ok = True
    N, H, W, Cin, Cout = 2, 32, 32, 128, 128
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)
    ok &= report("stride2", conv_tc(x, w, b, mode=2), ref_conv(x, w, b, mode=2))
    ok &= report("up2", conv_tc(x, w, b, up2=True), ref_conv(x, w, b, up2=True))
    res = torch.randn(N, Cout, H, W, device=dev)
    ok &= report("residual", conv_tc(x, w, b, res=res), ref_conv(x, w, b, res=res))
    side = torch.randn(N, 192, H, W, device=dev)
    sw = torch.randn(Cout, 192, 1, 1, device=dev) / 192 ** 0.5
    ok &= report("side1x1", conv_tc(x, w, b, side=side, side_w=sw), ref_conv(x, w, b, side=side, side_w=sw))
    x8 = torch.randn(3, 64, 16, 16, device=dev)
    w8 = torch.randn(64, 64, 3, 3, device=dev) / 24.0
    b8 = torch.randn(64, device=dev)
    ok &= report("stride2->8x8 N3", conv_tc(x8, w8, b8, mode=2), ref_conv(x8, w8, b8, mode=2))
    # dynamic range: large and tiny magnitudes through the fp16 split
    xl = torch.randn(1, 64, 16, 16, device=dev) * torch.logspace(-6, 3, 64, device=dev).view(1, 64, 1, 1)
    ok &= report("range", conv_tc(xl, w8, b8), ref_conv(xl, w8, b8))
    print("GROUP variants:", "PASS" if ok else "FAIL")


def group_bench():
    ms, fl = C.c_float(), C.c_double()
    for (N, H, W, Cin, Cout, mode) in [(16, 256, 256, 128, 128, 0), (16, 256, 256, 256, 128, 0), (16, 128, 128, 256, 256, 0),
                                       (16, 64, 64, 256, 256, 0), (16, 32, 32, 512, 512, 0), (16, 16, 16, 512, 512, 0),
                                       (16, 8, 8, 512, 512, 0), (16, 256, 256, 256, 128, 1), (4, 256, 256, 128, 128, 0)]:
        _lib.check(L.ddnm_conv_tc_bench(N, H, W, Cin, Cout, mode, 10, C.byref(ms), C.byref(fl)))
        print(f"[bench] N{N} {H}x{W} {Cin}->{Cout} mode{mode}: {ms.value:.3f} ms  {fl.value / ms.value / 1e9:.1f} TFLOP/s (algorithmic)", flush=True)


def group_bn_sweep():
    """N-tile width vs layer shape (all conv shapes of the two networks' low / mid resolution levels): data for the BN heuristic."""
    ms, fl = C.c_float(), C.c_double()
    shapes = [(16, 8, 8, 512, 512, 0), (16, 8, 8, 1024, 512, 0), (16, 16, 16, 512, 512, 0), (16, 16, 16, 1024, 512, 0),
              (16, 16, 16, 256, 512, 0), (16, 16, 16, 512, 512, 1), (16, 16, 16, 512, 1536, 1), (16, 32, 32, 256, 256, 0),
              (16, 32, 32, 512, 256, 0), (16, 32, 32, 768, 256, 0), (16, 64, 64, 256, 256, 0), (16, 64, 64, 512, 256, 0),
              (16, 128, 128, 128, 128, 0), (16, 128, 128, 256, 128, 0), (16, 256, 256, 256, 128, 0),
              (8, 8, 8, 1024, 1024, 0), (8, 8, 8, 2048, 1024, 0), (8, 16, 16, 1024, 1024, 0), (8, 16, 16, 2048, 1024, 0),
              (8, 32, 32, 512, 512, 0), (8, 32, 32, 1024, 512, 0), (8, 64, 64, 512, 512, 0), (8, 128, 128, 256, 256, 0)]
    def run(bn, iters):
        _lib.check(L.ddnm_tc_debug_force_bn(bn))
        _lib.check(L.ddnm_conv_tc_bench(N, H, W, Cin, Cout, mode, iters, C.byref(ms), C.byref(fl)))
        return ms.value * 1e3

    key = {(16, 256, 256, 256, 128, 0), (16, 128, 128, 256, 128, 0), (16, 64, 64, 512, 256, 0), (16, 16, 16, 512, 512, 0),
           (8, 128, 128, 256, 256, 0), (8, 64, 64, 512, 512, 0)}
    print("[bn_sweep] us per launch: BN64 / BN128 | heuristic's choice", flush=True)
    for (N, H, W, Cin, Cout, mode) in shapes:
        for label, iters in (("zeros ", 20), ("random", -20)):
            if label == "random" and (N, H, W, Cin, Cout, mode) not in key:
                continue
            row = ["   -   " if Cout % bn else f"{run(bn, iters):7.1f}" for bn in (64, 128)]
            print(f"[bn_sweep] {label} N{N} {H}x{W} {Cin}->{Cout} mode{mode}: {' '.join(row)} | {run(0, iters):7.1f}", flush=True)
    _lib.check(L.ddnm_tc_debug_force_bn(0))


def _cfg_ns(cfg):
    import types
    ns = types.SimpleNamespace
    return ns(model=ns(type="simple", ch=cfg.ch, out_ch=cfg.out_ch, ch_mult=list(cfg.ch_mult), num_res_blocks=cfg.num_res_blocks,
                       attn_resolutions=list(cfg.attn_resolutions), dropout=0.0, in_channels=cfg.in_channels, resamp_with_conv=True),
              data=ns(image_size=cfg.resolution), diffusion=ns(num_diffusion_timesteps=1000))


def group_unet(which="tiny", B=2, graph=1):
    from oracle import unet_simple as U
    from ddnm_b200.model import Model
    cfg = U.SimpleUNetConfig.tiny() if which == "tiny" else U.SimpleUNetConfig.celeba_hq()
    sd = U.init_state_dict(cfg, 1234)
    m = Model(_cfg_ns(cfg))
    m.use_cuda_graph = bool(int(graph))
    m.load_state_dict(sd)
    B = int(B)
    g = torch.Generator().manual_seed(99)
    x = torch.randn(B, 3, cfg.resolution, cfg.resolution, generator=g)
    t = torch.tensor([417.0, 3.0, 999.0, 0.0][:B] if B <= 4 else [float((37 * i) % 1000) for i in range(B)])
    taps = {}
    with torch.no_grad():
        ref = U.forward(sd, x, t, cfg, taps=taps)
    t0 = time.time()
    out = m(x.to(dev), t.to(dev))
    torch.cuda.synchronize()
    print(f"engine build+first forward {time.time() - t0:.2f}s; info {m.info(B)}")
    out2 = m(x.to(dev), t.to(dev))
    torch.cuda.synchronize()
    print("replay identical:", torch.equal(out, out2))
    order = ["conv_in"]
    nlev = len(cfg.ch_mult)
    for lv in range(nlev):
        order += [f"down.{lv}.{ib}" for ib in range(cfg.num_res_blocks)]
        if lv != nlev - 1:
            order.append(f"down.{lv}.ds")
    order += ["mid.block_1", "mid.attn_1", "mid.block_2"]
    for lv in reversed(range(nlev)):
        order += [f"up.{lv}.{ib}" for ib in range(cfg.num_res_blocks + 1)]
        if lv != 0:
            order.append(f"up.{lv}.us")
    for name in order:
        r = taps[name]
        got = m.read_tap(B, name, tuple(r.shape)).cpu()
        err = (got - r).abs().max().item()
        print(f"   tap {name:14s} shape {tuple(r.shape)} max_err {err:.3e} ref_absmax {r.abs().max().item():.3e}")
    err = (out.cpu() - ref).abs()
    tol = 1e-4 + 1e-3 * ref.abs()
    viol = (err > tol).float().mean().item()
    print(f"[unet {which} B{B}] max_abs_err {err.max().item():.3e} ref_absmax {ref.abs().max().item():.3e} "
          f"violations(rtol1e-3,atol1e-4) {viol * 100:.4f}%  ->", "PASS" if viol == 0 else "FAIL", flush=True)
    return m, x, t


def group_openai(which="tiny", B=2, graph=1):
    from oracle import unet_openai as UO
    from ddnm_b200.model import create_model
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from helpers import openai_model_kwargs
    cfg = UO.OpenAIUNetConfig.tiny() if which == "tiny" else UO.OpenAIUNetConfig.imagenet_256()
    sd = UO.init_state_dict(cfg, 1234)
    m = create_model(**openai_model_kwargs(cfg))
    m.use_cuda_graph = bool(int(graph))
    m.load_state_dict(sd)
    B = int(B)
    g = torch.Generator().manual_seed(99)
    x = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=g)
    t = torch.tensor([417.0, 3.0, 999.0, 0.0][:B])
    taps = {}
    with torch.no_grad():
        ref = UO.forward(sd, x, t, cfg, taps=taps)
    t0 = time.time()
    out = m(x.to(dev), t.to(dev))
    torch.cuda.synchronize()
    print(f"engine build+first forward {time.time() - t0:.2f}s; info {m.info(B)}")
    for name in sorted(taps, key=lambda k: (k.split('.')[0] != 'in', k.split('.')[0] == 'out', int(k.split('.')[1]) if '.' in k else 0)):
        r = taps[name]
        got = m.read_tap(B, name, tuple(r.shape)).cpu()
        print(f"   tap {name:8s} shape {tuple(r.shape)} max_err {(got - r).abs().max().item():.3e} ref_absmax {r.abs().max().item():.3e}")
    err = (out.cpu() - ref).abs()
    viol = (err > 1e-4 + 1e-3 * ref.abs()).float().mean().item()
    print(f"[openai {which} B{B}] max_abs_err {err.max().item():.3e} ref_absmax {ref.abs().max().item():.3e} "
          f"violations(rtol1e-3,atol1e-4) {viol * 100:.4f}%  ->", "PASS" if viol == 0 else "FAIL", flush=True)


def group_openai_bench(B=8, iters=3, prec="fp32"):
    from ddnm_b200.model import create_model
    from ddnm_b200.weights import random_state_dict_openai
    B, iters = int(B), int(iters)
    m = create_model(image_size=256, num_channels=256, num_res_blocks=2, learn_sigma=True, attention_resolutions="32,16,8",
                     num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True, use_fp16=True)
    m.precision = prec
    m.load_state_dict(random_state_dict_openai(m, 1234))
    x = torch.randn(B, 3, 256, 256, device=dev)
    t = torch.full((B,), 500.0, device=dev)
    for _ in range(2):
        m(x, t)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        m(x, t)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    info = m.info(B)
    print(f"[openai bench imagenet_256 B{B}] {ms:.2f} ms/forward  {B / ms * 1e3:.1f} img-fwd/s  "
          f"{info['flops_per_forward'] / ms / 1e9:.1f} TFLOP/s algorithmic; workspace {info['workspace_bytes'] / 2**30:.2f} GiB; launches {info['launches']}")
    prof = m.profile(x, t)
    agg = {}
    for p in prof:
        a = agg.setdefault(p["kind"], [0.0, 0.0, 0.0, 0])
        a[0] += p["ms"]; a[1] += p["flops"]; a[2] += p["bytes"]; a[3] += 1
    tot = sum(a[0] for a in agg.values())
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1][0]):
        print(f"   {k:10s} n={a[3]:4d} {a[0]:8.3f} ms ({a[0] / tot * 100:5.1f}%)  {a[1] / max(a[0], 1e-9) / 1e9:8.1f} TFLOP/s  {a[2] / max(a[0], 1e-9) / 1e6:8.1f} GB/s")
    os.makedirs("diag_out", exist_ok=True)
    json.dump(prof, open(f"diag_out/unet_profile_openai_B{B}.json", "w"))


def group_cpu_threads():
    """how the CPU reference scales with torch threads on this host (choose the reference arm's thread count)"""
    from oracle import unet_simple as U
    cfg = U.SimpleUNetConfig.celeba_hq()
    sd = U.init_state_dict(cfg, 1234)
    x = torch.randn(1, 3, 256, 256)
    t = torch.tensor([500.0])
    print("cpu_count", os.cpu_count())
    for nt in (8, 16, 32, 64, os.cpu_count()):
        torch.set_num_threads(nt)
        with torch.no_grad():
            U.forward(sd, x, t, cfg)
            t0 = time.time()
            U.forward(sd, x, t, cfg)
            print(f"   threads {nt}: {time.time() - t0:.2f} s / image-forward", flush=True)


def group_unet_bench(which="celeba", B=16, iters=5, prec="fp32", deal=-1, tag=""):
    from oracle import unet_simple as U
    from ddnm_b200.model import Model
    B, iters = int(B), int(iters)
    _lib.check(L.ddnm_tc_debug_deal(int(deal)))
    cfg = U.SimpleUNetConfig.tiny() if which == "tiny" else U.SimpleUNetConfig.celeba_hq()
    sd = U.init_state_dict(cfg, 1234)
    m = Model(_cfg_ns(cfg))
    m.precision = prec
    m.load_state_dict(sd)
    x = torch.randn(B, 3, cfg.resolution, cfg.resolution, device=dev)
    t = torch.full((B,), 500.0, device=dev)
    for _ in range(3):
        m(x, t)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        m(x, t)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    info = m.info(B)
    print(f"[unet bench {which} B{B}] {ms:.2f} ms/forward  {B / ms * 1e3:.1f} img-fwd/s  "
          f"{info['flops_per_forward'] / ms / 1e9:.1f} TFLOP/s algorithmic; workspace {info['workspace_bytes'] / 2**30:.2f} GiB; launches {info['launches']}")
    prof = m.profile(x, t)
    agg = {}
    for p in prof:
        a = agg.setdefault(p["kind"], [0.0, 0.0, 0.0, 0])
        a[0] += p["ms"]; a[1] += p["flops"]; a[2] += p["bytes"]; a[3] += 1
    tot = sum(a[0] for a in agg.values())
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1][0]):
        print(f"   {k:10s} n={a[3]:4d} {a[0]:8.3f} ms ({a[0] / tot * 100:5.1f}%)  {a[1] / max(a[0], 1e-9) / 1e9:8.1f} TFLOP/s  {a[2] / max(a[0], 1e-9) / 1e6:8.1f} GB/s")
    top = sorted(prof, key=lambda p: -p["ms"])[:12]
    for p in top:
        print(f"   top {p['name']:28s} {p['ms']:.3f} ms  {p['flops'] / max(p['ms'], 1e-9) / 1e9:.1f} TF/s  {p['bytes'] / max(p['ms'], 1e-9) / 1e6:.1f} GB/s")
    os.makedirs("diag_out", exist_ok=True)
    json.dump(prof, open(f"diag_out/unet_profile_{which}_B{B}{tag}.json", "w"))


def group_lanes(which="celeba", B=16, lanes=2, iters=5, openai=0):
    """Prototype: the batch as `lanes` independent sub-batches, one engine + stream each — does the block scheduler overlap
    one lane's HBM-bound GroupNorm passes with the other's tensor-core convolutions?"""
    from oracle import unet_simple as U
    from ddnm_b200.model import Model
    B, lanes, iters = int(B), int(lanes), int(iters)
    cfg = U.SimpleUNetConfig.tiny() if which == "tiny" else U.SimpleUNetConfig.celeba_hq()
    sd = U.init_state_dict(cfg, 1234)
    sub = B // lanes
    ms_, xs, ts, ss = [], [], [], []
    for l in range(lanes):
        m = Model(_cfg_ns(cfg))
        m.load_state_dict(sd)
        ms_.append(m)
        xs.append(torch.randn(sub, 3, cfg.resolution, cfg.resolution, device=dev))
        ts.append(torch.full((sub,), 500.0, device=dev))
        ss.append(torch.cuda.Stream())
    for l in range(lanes):
        for _ in range(3):
            ms_[l](xs[l], ts[l])
    torch.cuda.synchronize()
    def run(n, concurrent):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        if concurrent:
            start = torch.cuda.Event(); start.record()
            for _ in range(n):
                for l in range(lanes):
                    with torch.cuda.stream(ss[l]):
                        ms_[l](xs[l], ts[l])
            for l in range(lanes):
                torch.cuda.current_stream().wait_stream(ss[l])
        else:
            for _ in range(n):
                for l in range(lanes):
                    ms_[l](xs[l], ts[l])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n
    for l in range(lanes):
        ss[l].wait_stream(torch.cuda.current_stream())
    a = run(iters, False)
    b = run(iters, True)
    b2 = run(iters, True)
    print(f"[lanes {which} B{B} = {lanes} x {sub}] serial {a:.2f} ms per {B} images; concurrent {b:.2f} / {b2:.2f} ms per {B} images")


def group_epi_bench(iters=-20, deal=-1):
    """Epilogue features as the network uses them (mode bits 16: GroupNorm sums, 32: residual, 64: channel add, 128: upsample phase)
    on the layer shapes where the epilogue is exposed (short K)."""
    ms, fl = C.c_float(), C.c_double()
    iters = int(iters)
    _lib.check(L.ddnm_tc_debug_deal(int(deal)))
    print(f"[epi_bench] deal mode {deal}")
    for (N, H, W, Cin, Cout) in [(16, 256, 256, 128, 128), (16, 128, 128, 128, 128), (16, 256, 256, 256, 128), (16, 64, 64, 256, 256),
                                 (16, 32, 32, 256, 256), (16, 8, 8, 512, 512)]:
        row = []
        for feat in (0, 16, 32, 64, 16 + 64, 16 + 32 + 64):
            _lib.check(L.ddnm_conv_tc_bench(N, H, W, Cin, Cout, feat, iters, C.byref(ms), C.byref(fl)))
            row.append(f"{ms.value * 1e3:7.1f}")
        print(f"[epi_bench] N{N} {H}x{W} {Cin}->{Cout} 3x3: plain {row[0]} | stats {row[1]} | residual {row[2]} | chanadd {row[3]} | stats+chanadd {row[4]} | all {row[5]} us", flush=True)
    for (N, H, W, Cin, Cout) in [(16, 128, 128, 128, 128), (16, 64, 64, 256, 128), (16, 32, 32, 256, 256)]:
        row = []
        for feat in (128, 128 + 16, 128 + 64, 128 + 16 + 64):
            _lib.check(L.ddnm_conv_tc_bench(N, H, W, Cin, Cout, feat, iters, C.byref(ms), C.byref(fl)))
            row.append(f"{ms.value * 1e3:7.1f}")
        print(f"[epi_bench] N{N} {H}x{W} {Cin}->{Cout} up-phase: plain {row[0]} | stats {row[1]} | chanadd {row[2]} | stats+chanadd {row[3]} us", flush=True)


def group_chunk_bench(iters=10):
    """GroupNorm pass + convolution over 16 images in chunks sharing a chunk-sized plane scratch: do the planes stay in L2?"""
    ms = C.c_float()
    for (N, H, W, Cin, Cout) in [(16, 256, 256, 128, 128), (16, 256, 256, 256, 128), (16, 128, 128, 128, 128), (16, 128, 128, 256, 128)]:
        row = []
        for chunk in (16, 8, 4, 2, 1):
            _lib.check(L.ddnm_gnconv_chunk_bench(N, chunk, H, W, Cin, Cout, int(iters), C.byref(ms)))
            row.append(f"chunk {chunk:2d}: {ms.value * 1e3:7.1f}")
        print(f"[chunk_bench] N{N} {H}x{W} {Cin}->{Cout} gn+conv us per 16 images: " + " | ".join(row), flush=True)


def group_eager(which="celeba", B=16, iters=3):
    """The competitor SURVEY §8d names: the reference's network as plain PyTorch eager on this GPU (the oracle restatement is
    the reference's op sequence, bit-exact on CPU), with the reference's own settings (main.py:145 cudnn.benchmark = True; TF32
    convolutions allowed, torch's default) and with TF32 off (strict fp32, the precision class ddnm_b200's parity mode delivers)."""
    B, iters = int(B), int(iters)
    if which == "openai":
        from oracle import unet_openai as UM
        cfg = UM.OpenAIUNetConfig.imagenet_256()
    else:
        from oracle import unet_simple as UM
        cfg = UM.SimpleUNetConfig.celeba_hq()
    sd = {k: v.to(dev) for k, v in UM.init_state_dict(cfg, 1234).items()}
    res = cfg.image_size if which == "openai" else cfg.resolution
    x = torch.randn(B, 3, res, res, device=dev)
    t = torch.full((B,), 500.0, device=dev)
    torch.backends.cudnn.benchmark = True
    out = {}
    for tf32 in (True, False):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        with torch.no_grad():
            for _ in range(3):
                UM.forward(sd, x, t, cfg)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                UM.forward(sd, x, t, cfg)
            e1.record()
            torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        out["tf32_conv" if tf32 else "fp32_strict"] = ms
        print(f"[eager torch {which} B{B}] cudnn TF32 convs {'on ' if tf32 else 'off'}: {ms:.2f} ms/forward = {B / ms * 1e3:.1f} image-forwards/s", flush=True)
    os.makedirs("diag_out", exist_ok=True)
    json.dump(dict(model=which, batch=B, ms_per_forward=out, torch=torch.__version__, cudnn=torch.backends.cudnn.version(),
                   note="oracle restatement of the reference network run as PyTorch eager on the GPU; cudnn.benchmark=True"),
              open(f"diag_out/eager_torch_{which}_B{B}.json", "w"))


if __name__ == "__main__":
    print("device:", torch.cuda.get_device_name(0), flush=True)
    globals()["group_" + sys.argv[1]](*sys.argv[2:])
