"""GPU (H100) parity tests: the CUDA engine, called through the C ABI (ctypes shims), against the oracle and the
committed golden vectors of the reference.  Tolerance is north_star's rtol=1e-3 / atol=1e-4 fp32 (usually far
tighter); inpainting indexing must be bit-exact."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sampler as S
from oracle import schedule as SCH
from oracle import unet_openai as UO
from oracle import unet_simple as U

from helpers import LAMBDA_CASES, assert_close, engine_op, model_config, openai_model_kwargs, oracle_ops, sampler_config
from test_oracle_golden import SAMPLER_CASES, SIMPLIFIED_CASES, sampler_inputs, simplified_inputs

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def lib():
    from ddnm_b200 import _lib
    return _lib


def _conv_tc(lib, x, w, b, mode=0, up2=False, side=None, side_w=None, res=None):
    L = lib.lib()
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    oH, oW = (H // 2, W // 2) if mode == 2 else ((2 * H, 2 * W) if up2 else (H, W))
    out = torch.empty(N, oH, oW, Cout, device=dev)
    nhwc = lambda t: None if t is None else t.permute(0, 2, 3, 1).contiguous()   # noqa: E731
    xs, sx, rs = nhwc(x), nhwc(side), nhwc(res)
    lib.check(L.ddnm_conv_tc(lib.ptr(xs), N, H, W, Cin, lib.ptr(w.contiguous()), lib.ptr(b), Cout, mode, int(up2), lib.ptr(sx),
                             0 if side is None else side.shape[1], lib.ptr(side_w.contiguous()) if side_w is not None else None,
                             lib.ptr(rs), lib.ptr(out), None))
    return out.permute(0, 3, 1, 2)


def _conv_ref(x, w, b, mode=0, up2=False, side=None, side_w=None, res=None):
    x, w, b = x.double().cpu(), w.double().cpu(), b.double().cpu()
    if up2:
        x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    o = F.conv2d(x, w, b, padding=1) if mode == 0 else (F.conv2d(x, w, b) if mode == 1 else F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2))
    if side is not None:
        o = o + F.conv2d(side.double().cpu(), side_w.double().cpu())
    if res is not None:
        o = o + res.double().cpu()
    return o


@pytest.mark.parametrize("shape", [(1, 16, 16, 64, 64, 0), (2, 32, 32, 128, 128, 0), (1, 64, 64, 128, 256, 0), (3, 8, 8, 128, 64, 0),
                                   (1, 128, 128, 192, 128, 0), (1, 16, 16, 512, 1536, 1), (2, 32, 32, 128, 128, 2), (3, 16, 16, 64, 64, 2),
                                   (2, 256, 256, 64, 128, 0), (4, 128, 128, 128, 256, 0), (4, 128, 128, 128, 128, 0), (4, 128, 128, 64, 128, 1),
                                   (8, 128, 128, 64, 128, 2), (2, 128, 128, 64, 384, 0)],
                         ids=str)
def test_tc_conv_vs_fp64(lib, shape):
    # tolerance: fp32 accumulation over K <= 4608 terms on the tensor core (truncating adds) gives ~3e-6 relative to the
    # output scale; the 3x fp16 split itself contributes ~5e-7
    N, H, W, Cin, Cout, mode = shape
    torch.manual_seed(0)
    k = 1 if mode == 1 else 3
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, k, k, device=dev) / (k * k * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)
    assert_close(_conv_tc(lib, x, w, b, mode=mode), _conv_ref(x, w, b, mode=mode), rtol=1e-4, atol=5e-5, what=f"tc conv {shape}")


def test_tc_conv_fusions(lib):
    torch.manual_seed(2)
    N, H, W, Cin, Cout = 2, 32, 32, 128, 128
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)
    res = torch.randn(N, Cout, H, W, device=dev)
    side = torch.randn(N, 192, H, W, device=dev)
    sw = torch.randn(Cout, 192, 1, 1, device=dev) / 192 ** 0.5
    assert_close(_conv_tc(lib, x, w, b, up2=True), _conv_ref(x, w, b, up2=True), 1e-4, 5e-5, "upsample conv")
    assert_close(_conv_tc(lib, x, w, b, res=res), _conv_ref(x, w, b, res=res), 1e-4, 5e-5, "residual epilogue")
    assert_close(_conv_tc(lib, x, w, b, side=side, side_w=sw), _conv_ref(x, w, b, side=side, side_w=sw), 1e-4, 5e-5, "1x1 side input")
    # matches the CUDA-core direct convolution too
    L = lib.lib()
    out = torch.empty(N, H, W, Cout, device=dev)
    lib.check(L.ddnm_conv_direct(lib.ptr(x.permute(0, 2, 3, 1).contiguous()), N, H, W, Cin, lib.ptr(w), lib.ptr(b), Cout, 0, 0, lib.ptr(out), None))
    torch.cuda.synchronize()
    assert_close(_conv_tc(lib, x, w, b), out.permute(0, 3, 1, 2), 1e-4, 5e-5, "tc vs direct")
    # the same fusions on maps where CTAs walk several tiles (ping-pong, CTA pairs, HALO)
    torch.manual_seed(6)
    N, H, W, Cin, Cout = 8, 64, 64, 64, 128
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)
    assert_close(_conv_tc(lib, x, w, b, up2=True), _conv_ref(x, w, b, up2=True), 1e-4, 5e-5, "upsample conv (four parity phases), 8x64x64")
    N, H, W = 4, 128, 128
    x = torch.randn(N, Cin, H, W, device=dev)
    res = torch.randn(N, Cout, H, W, device=dev)
    side = torch.randn(N, 128, H, W, device=dev)
    sw = torch.randn(Cout, 128, 1, 1, device=dev) / 128 ** 0.5
    assert_close(_conv_tc(lib, x, w, b, res=res), _conv_ref(x, w, b, res=res), 1e-4, 5e-5, "residual epilogue, 4x128x128")
    assert_close(_conv_tc(lib, x, w, b, side=side, side_w=sw), _conv_ref(x, w, b, side=side, side_w=sw), 1e-4, 5e-5,
                 "1x1 side input, 4x128x128")


# at most one tile per SM, so both forms run on conv_tc_kernel: BN = 64 and 128, with and without HALO, 1x1 and stride 2
@pytest.mark.parametrize("shape", [(2, 32, 32, 128, 128, 0), (1, 64, 64, 128, 256, 0), (3, 8, 8, 128, 64, 0), (2, 64, 64, 192, 128, 1),
                                   (1, 128, 128, 128, 128, 0), (16, 32, 32, 128, 128, 0), (2, 16, 16, 256, 512, 0), (1, 64, 64, 128, 128, 2)],
                         ids=str)
def test_tc_conv_dual_accumulator_vs_three_instruction_form(lib, shape):
    """DUAL kernel (hi*hi and hi*lo issued as one m64 x 2BN wgmma over the adjacent B_hi / B_lo planes, partial sums added in the
    epilogue) against the plain three-instruction form: the same products, two fp32 additions re-associated."""
    N, H, W, Cin, Cout, mode = shape
    torch.manual_seed(7)
    k = 1 if mode == 1 else 3
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, k, k, device=dev) / (k * k * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)
    L = lib.lib()
    try:
        lib.check(L.ddnm_tc_debug_dual_mode(0))
        plain = _conv_tc(lib, x, w, b, mode=mode).clone()
        lib.check(L.ddnm_tc_debug_dual_mode(1))
        dual = _conv_tc(lib, x, w, b, mode=mode)
    finally:
        L.ddnm_tc_debug_dual_mode(1)
    torch.cuda.synchronize()
    assert_close(dual, plain, 2e-5, 1e-5, f"dual vs plain {shape}")
    assert_close(dual, _conv_ref(x, w, b, mode=mode), rtol=1e-4, atol=5e-5, what=f"dual conv {shape}")


def test_groupnorm_silu(lib):
    torch.manual_seed(3)
    for (N, H, W, Cc) in [(2, 16, 16, 64), (1, 32, 32, 384), (2, 8, 8, 1024)]:
        x = torch.randn(N, Cc, H, W, device=dev) * 2 + 0.5
        g, b = torch.randn(Cc, device=dev), torch.randn(Cc, device=dev)
        out = torch.empty(N, H, W, Cc, device=dev)
        lib.check(lib.lib().ddnm_groupnorm(lib.ptr(x.permute(0, 2, 3, 1).contiguous()), N, H, W, Cc, 32, lib.ptr(g), lib.ptr(b), 1e-6, 1, lib.ptr(out), None))
        ref = F.group_norm(x.double().cpu(), 32, g.double().cpu(), b.double().cpu(), 1e-6)
        ref = ref * torch.sigmoid(ref)
        assert_close(out.permute(0, 3, 1, 2), ref, 1e-5, 1e-5, f"groupnorm+silu C={Cc}")


# ------------------------------------------------------------------------------------------------ denoiser
def _engine_model(cfg, graph=True):
    from ddnm_b200.model import Model
    m = Model(model_config(cfg))
    m.use_cuda_graph = graph
    m.load_state_dict(U.init_state_dict(cfg, 1234))
    return m


@pytest.mark.parametrize("graph", [False, True])
def test_unet_tiny_vs_reference_golden(gold, graph):
    g = gold["unet_simple"]
    cfg = U.SimpleUNetConfig.tiny()
    m = _engine_model(cfg, graph)
    x, t = torch.from_numpy(g["tiny_x"]).to(dev), torch.from_numpy(g["tiny_t"]).to(dev)
    out = m(x, t)
    out2 = m(x, t)   # graph replay
    assert_close(out, g["tiny_out"], what="unet tiny vs reference")
    assert_close(out2, g["tiny_out"], what="unet tiny replay vs reference")
    for k in ("conv_in", "down.0.0", "down.0.ds", "down.1.0", "mid.attn_1", "up.1.us", "up.0.1"):
        r = g["tiny_tap_s2_" + k]   # stored as the [..., ::2, ::2] sample of the tap
        full = m.read_tap(2, k, (r.shape[0], r.shape[1], 2 * r.shape[2], 2 * r.shape[3]))
        assert_close(full[:, :, ::2, ::2], r, what="tap " + k)


def test_unet_celeba_vs_reference_golden(gold):
    g = gold["unet_simple"]
    cfg = U.SimpleUNetConfig.celeba_hq()
    m = _engine_model(cfg)
    gen = torch.Generator().manual_seed(99)
    x = torch.randn(1, 3, 256, 256, generator=gen)
    out = m(x.to(dev), torch.from_numpy(g["celeba_t"]).to(dev))
    assert_close(out[:, :, ::8, ::8], g["celeba_out_s8"], what="celeba UNet vs reference (strided sample)")
    assert abs(out.double().sum().item() - g["celeba_out_sum"][0]) <= 1e-3 * g["celeba_out_sum"][1]
    # and against the full oracle forward (every element)
    with torch.no_grad():
        ref = U.forward(U.init_state_dict(cfg, 1234), x, torch.from_numpy(g["celeba_t"]), cfg)
    assert_close(out, ref, what="celeba UNet vs oracle")


def test_unet_fast_fp16_mode_is_close_but_flagged_non_parity(gold):
    """precision='fp16' (one fp16 product per MAC): stays within ~1e-2 of the fp32 model — the ballpark of the reference's
    own use_fp16 torso (SURVEY.md section 7: 1.7e-3 relative) — and is NOT what the parity claims are made on."""
    g = gold["unet_simple"]
    cfg = U.SimpleUNetConfig.tiny()
    from ddnm_b200.model import Model
    m = Model(model_config(cfg))
    m.precision = "fp16"
    m.load_state_dict(U.init_state_dict(cfg, 1234))
    out = m(torch.from_numpy(g["tiny_x"]).to(dev), torch.from_numpy(g["tiny_t"]).to(dev)).cpu()
    ref = torch.from_numpy(g["tiny_out"])
    err = (out - ref).abs().max().item()
    assert err < 2e-2 * ref.abs().max().item(), err
    assert err > 1e-5, "fast mode unexpectedly as accurate as the 3-term mode: is the flag wired?"


def test_unet_forward_is_bit_reproducible():
    """GroupNorm sums are accumulated by many CTAs with atomics; they are fixed-point integer accumulators (StatAcc: two carry-free
    64-bit words, 48 fractional bits), so the arrival order cannot change the result: every replay of a forward is bit-identical
    (eager and CUDA-graph alike)."""
    cfg = U.SimpleUNetConfig.celeba_hq()
    torch.manual_seed(17)
    x = torch.randn(2, 3, 256, 256, device=dev)
    t = torch.tensor([700.0, 31.0], device=dev)
    for graph in (True, False):
        m = _engine_model(cfg, graph)
        first = m(x, t).clone()
        for _ in range(3):
            assert torch.equal(m(x, t), first), f"forward not reproducible (graph={graph})"
    cfg = U.SimpleUNetConfig.tiny()
    m = _engine_model(cfg)
    x = torch.randn(4, 3, 32, 32, device=dev)
    t = torch.tensor([10.0, 500.0, 999.0, 0.0], device=dev)
    first = m(x, t).clone()
    for _ in range(5):
        assert torch.equal(m(x, t), first)


def test_unet_tile_order_does_not_change_the_result():
    """The tile -> CTA map of the convolutions (round-robin, or one contiguous range per CTA on the layers where that saves the
    per-tile flush of the GroupNorm sums) only regroups fp32 partial sums: the forward agrees to fp32 rounding of the statistics."""
    from ddnm_b200 import _lib
    cfg = U.SimpleUNetConfig.celeba_hq()
    torch.manual_seed(23)
    x = torch.randn(2, 3, 256, 256, device=dev)
    t = torch.tensor([612.0, 87.0], device=dev)
    outs = []
    try:
        for mode in (0, -1):
            _lib.check(_lib.lib().ddnm_tc_debug_deal(mode))
            outs.append(_engine_model(cfg)(x, t).clone())
    finally:
        _lib.check(_lib.lib().ddnm_tc_debug_deal(-1))
    scale = outs[0].abs().max().item()
    err = (outs[0] - outs[1]).abs().max().item()
    assert err <= 2e-5 * scale, (err, scale)


def test_unet_batch_rows_independent():
    """Rows of a batch are independent trajectories (the property multi-GPU sharding relies on)."""
    cfg = U.SimpleUNetConfig.tiny()
    m = _engine_model(cfg)
    torch.manual_seed(5)
    x = torch.randn(4, 3, 32, 32, device=dev)
    t = torch.tensor([10.0, 500.0, 999.0, 0.0], device=dev)
    full = m(x, t)
    for i in range(4):
        assert_close(m(x[i:i + 1], t[i:i + 1]), full[i:i + 1], 1e-5, 1e-5, f"row {i}")


def test_ragged_last_batch_reuses_the_bigger_engine(gold):
    """A dataset's last, smaller batch is padded to the engine that already exists (no second engine with its own weight copy and
    workspace); rows are independent, so the real rows' results are those of an engine built for exactly that batch."""
    from ddnm_b200.sampler import ddnm_diffusion
    cfg = U.SimpleUNetConfig.tiny()
    torch.manual_seed(9)
    x = torch.randn(4, 3, 32, 32, device=dev)
    t = torch.tensor([10.0, 500.0, 999.0, 0.0], device=dev)
    big = _engine_model(cfg)
    full = big(x, t)
    part = big(x[:3], t[:3])
    assert list(big._engines) == [4], "the 3-row call must ride on the 4-row engine"
    exact = _engine_model(cfg)
    ref = exact(x[:3], t[:3])
    assert torch.equal(part, ref) and torch.equal(part, full[:3])
    oop = oracle_ops(gold["operators"], 32)["sr4"]
    eop = engine_op("sr4", oop, 32)
    y = eop.A(x)
    conf = sampler_config(5, 1, 1)
    betas = SCH.linear_betas().to(dev)
    tape = torch.randn(5, 3, 3, 32, 32, device=dev)
    a = ddnm_diffusion(x[:3], big, betas, 0.85, eop, y[:3], config=conf, noise=tape)
    b = ddnm_diffusion(x[:3], exact, betas, 0.85, eop, y[:3], config=conf, noise=tape)
    assert list(big._engines) == [4] and torch.equal(a[0][0], b[0][0]) and torch.equal(a[1][0], b[1][0])
    torch.manual_seed(3)
    c = ddnm_diffusion(x[:3], big, betas, 0.85, eop, y[:3], config=conf)          # draws inside: same generator consumption
    torch.manual_seed(3)
    d = ddnm_diffusion(x[:3], exact, betas, 0.85, eop, y[:3], config=conf)
    assert torch.equal(c[0][0], d[0][0])


def _engine_openai(cfg, graph=True):
    from ddnm_b200.model import create_model
    m = create_model(**openai_model_kwargs(cfg))
    m.convert_to_fp16()                       # what the reference runner does (diffusion.py:145-146); a no-op here
    m.use_cuda_graph = graph
    m.load_state_dict(UO.init_state_dict(cfg, 1234))
    return m


@pytest.mark.parametrize("graph", [False, True])
def test_openai_unet_tiny_vs_reference_golden(gold, graph):
    g = gold["unet_openai"]
    cfg = UO.OpenAIUNetConfig.tiny()
    m = _engine_openai(cfg, graph)
    x, t = torch.from_numpy(g["tiny_x"]).to(dev), torch.from_numpy(g["tiny_t"]).to(dev)
    out = m(x, t)
    assert out.shape == (2, 6, 32, 32)
    assert_close(out, g["tiny_out"], what="openai unet tiny vs reference")
    assert_close(m(x, t), g["tiny_out"], what="openai unet tiny replay vs reference")
    for k in ("in.0", "in.1", "in.2", "in.3", "mid", "out.0", "out.2", "out.5"):
        r = g["tiny_tap_s2_" + k]   # stored as the [..., ::2, ::2] sample of the tap
        full = m.read_tap(2, k, (r.shape[0], r.shape[1], 2 * r.shape[2], 2 * r.shape[3]))
        assert_close(full[:, :, ::2, ::2], r, what="openai tap " + k)


def test_openai_unet_imagenet_vs_reference_golden(gold):
    g = gold["unet_openai"]
    cfg = UO.OpenAIUNetConfig.imagenet_256()
    m = _engine_openai(cfg)
    gen = torch.Generator().manual_seed(99)
    x = torch.randn(1, 3, 256, 256, generator=gen)
    out = m(x.to(dev), torch.from_numpy(g["imagenet_t"]).to(dev))
    assert_close(out[:, :, ::8, ::8], g["imagenet_out_s8"], what="imagenet UNetModel vs reference (strided sample)")
    assert abs(out.double().sum().item() - g["imagenet_out_sum"][0]) <= 1e-3 * g["imagenet_out_sum"][1]


def test_sampler_with_openai_unet_six_channels(gold):
    """DDNM+ colorization with the 6-channel (learn_sigma) net: the sampler keeps eps = channels 0..2 (svd_ddnm.py:54-55)."""
    from ddnm_b200.sampler import ddnm_plus_diffusion
    cfg = UO.OpenAIUNetConfig.tiny()
    sd = UO.init_state_dict(cfg, 1234)
    m = _engine_openai(cfg)
    oop = oracle_ops(gold["operators"], 32)["color"]
    eop = engine_op("color", oop, 32)
    gsm = gold["sampler_tiny"]
    g = torch.Generator().manual_seed(31)
    x_orig = torch.rand(2, 3, 32, 32, generator=g) * 2 - 1
    x_T = torch.randn(2, 3, 32, 32, generator=g)
    y = oop.A(x_orig.reshape(2, -1))
    T, tl, tr, sy = 6, 2, 2, 0.1
    npairs = len(SCH.time_pairs(1000, T, tl, tr))
    tape = [torch.randn(2, 3, 32, 32, generator=g) for _ in range(npairs)]
    betas = torch.from_numpy(gsm["betas"])
    xs, x0s = ddnm_plus_diffusion(x_T.to(dev), m, betas.to(dev), 0.85, eop, y.to(dev), sy, config=sampler_config(T, tl, tr),
                                  noise=torch.stack(tape).to(dev))
    with torch.no_grad():
        ox, ox0 = S.ddnm_sample(x_T, lambda a, b: UO.forward(sd, a, b, cfg), betas, 0.85, oop, y, tape, t_sampling=T, travel_length=tl,
                                travel_repeat=tr, sigma_y=sy)
    assert_close(xs[0], ox, 1e-3, 3e-3, "openai-net sampler vs oracle")
    assert_close(x0s[0], ox0, 1e-3, 3e-3, "openai-net sampler x0_pred vs oracle")


# ------------------------------------------------------------------------------------------------ operators
@pytest.mark.parametrize("dim", [32, 256])
def test_operators_vs_oracle_and_golden(gold, dim):
    g = gold["operators"]
    tag = f"d{dim}"
    B = 2 if dim == 32 else 1
    rng = torch.Generator().manual_seed(4321)
    x = torch.rand(B, 3, dim, dim, generator=rng) * 2 - 1
    v = torch.randn(B, 3 * dim * dim, generator=rng)
    e = torch.randn(B, 3 * dim * dim, generator=rng)
    sub = (lambda z: z.reshape(B, -1)) if dim == 32 else (lambda z: z.reshape(B, -1)[:, ::61])
    xd, vd, ed = x.to(dev), v.to(dev), e.to(dev)
    for name, o in oracle_ops(g, dim).items():
        eop = engine_op(name, o, dim)
        golden = not (dim == 256 and name in ("deblur", "bicubic", "deblur2d"))
        y = o.A(x.reshape(B, -1))
        ye = eop.A(xd)
        assert ye.shape == y.shape
        yq = y * 0.9 + 0.05
        if name == "inpaint":   # pure indexing: bit-exact
            assert torch.equal(ye.cpu(), y), "inpainting A must be bit-exact"
            assert torch.equal(eop.A_pinv(yq.to(dev)).cpu(), o.A_pinv(yq.clone()))
            assert torch.equal(eop.project(xd, yq.to(dev)).cpu().reshape(B, -1), o.project(x, yq).reshape(B, -1))
        assert_close(ye, y, 1e-4, 1e-5, f"{name} A")
        assert_close(eop.A_pinv(yq.to(dev)), o.A_pinv(yq.clone()), 1e-4, 1e-5, f"{name} A_pinv")
        assert_close(eop.project(xd, yq.to(dev)).reshape(B, -1), o.project(x, yq).reshape(B, -1), 1e-4, 2e-5, f"{name} project")
        if golden:
            assert_close(sub(ye), g[f"{tag}_{name}_A"], 1e-4, 1e-5, f"{name} A vs reference")
            assert_close(sub(eop.project(xd, yq.to(dev))), g[f"{tag}_{name}_proj"], 1e-4, 2e-5, f"{name} project vs reference")
        if name in ("bicubic", "deblur2d", "cs"):
            with pytest.raises(NotImplementedError):
                eop.Lambda(vd, 0.9, 0.1, 0.3, 0.85)
            continue
        for ci, (a, sy, st) in enumerate(LAMBDA_CASES):
            at, stt = torch.tensor(a), torch.tensor(st)
            L = eop.Lambda(vd, at, sy, stt, 0.85)
            Ln = eop.Lambda_noise(vd, at, sy, stt, 0.85, ed)
            assert_close(L, o.Lambda(v.clone(), at, sy, stt, 0.85), 1e-4, 2e-5, f"{name} Lambda{ci}")
            assert_close(Ln, o.Lambda_noise(v.clone(), at, sy, stt, 0.85, e.clone()), 1e-4, 2e-5, f"{name} Lambda_noise{ci}")
            if golden:
                assert_close(sub(L), g[f"{tag}_{name}_L{ci}"], 1e-4, 2e-5, f"{name} Lambda{ci} vs reference")
                assert_close(sub(Ln), g[f"{tag}_{name}_Ln{ci}"], 1e-4, 2e-5, f"{name} Lambda_noise{ci} vs reference")
        assert torch.equal(vd.cpu(), v), "operator mutated its input"


def test_operator_properties_full_size(gold):
    """Size-independent properties at 256x256 on the GPU: A A^+ y = y, projection is idempotent and consistent."""
    g = gold["operators"]
    torch.manual_seed(11)
    B = 4
    x = (torch.rand(B, 3, 256, 256, device=dev) * 2 - 1)
    for name, o in oracle_ops(g, 256).items():
        eop = engine_op(name, o, 256)
        y = eop.A(x)
        assert_close(eop.A(eop.A_pinv(y)), y, 1e-3, 2e-4, f"{name}: A A^+ y = y")
        z = torch.randn_like(x)
        p = eop.project(z, y)
        assert_close(eop.A(p), y, 1e-3, 3e-4, f"{name}: A(project(z, y)) = y")
        assert_close(eop.project(p, y), p, 1e-3, 3e-4, f"{name}: projection idempotent")


# ------------------------------------------------------------------------------------------------ sampler
@pytest.mark.parametrize("case", SAMPLER_CASES, ids=lambda c: f"{c[0]}-T{c[1]}-l{c[2]}r{c[3]}-s{c[4]}")
def test_sampler_vs_oracle_and_golden(gold, case):
    from ddnm_b200.sampler import ddnm_diffusion, ddnm_plus_diffusion
    name, T, tl, tr, sy = case
    g = gold["sampler_tiny"]
    cfg = U.SimpleUNetConfig.tiny()
    sd = U.init_state_dict(cfg, 1234)
    key = f"{name}_T{T}_l{tl}_r{tr}_s{sy}"
    npairs = len(SCH.time_pairs(1000, T, tl, tr))
    x_T, y, tape = sampler_inputs(g, key, npairs)
    oop = oracle_ops(gold["operators"], 32)[name]
    eop = engine_op(name, oop, 32)
    m = _engine_model(cfg)
    betas = torch.from_numpy(g["betas"]).to(dev)
    noise = torch.stack(tape).to(dev)
    conf = sampler_config(T, tl, tr)
    if sy == 0.0:
        xs, x0s = ddnm_diffusion(x_T.to(dev), m, betas, 0.85, eop, y.to(dev), config=conf, noise=noise)
    else:
        xs, x0s = ddnm_plus_diffusion(x_T.to(dev), m, betas, 0.85, eop, y.to(dev), sy, config=conf, noise=noise)
    assert isinstance(xs, list) and len(xs) == 1 and not xs[0].is_cuda      # reference return convention (svd_ddnm.py:78)
    # (1) teacher-forced: every oracle step re-run on the engine from the oracle's own state must agree to fp32 tolerance
    trace = []
    with torch.no_grad():
        ox, ox0 = S.ddnm_sample(x_T, lambda a, b: U.forward(sd, a, b, cfg), torch.from_numpy(g["betas"]), 0.85, oop, y, tape,
                                t_sampling=T, travel_length=tl, travel_repeat=tr, sigma_y=sy, trace=trace)
    # (2) end to end against the reference's stored result.  Per-step errors (~1e-6) are amplified by the random-init net
    # and the 1/sqrt(alpha-bar) factor of the first steps exactly as oracle-vs-reference rounding is (see gen_golden: 2e-4).
    assert_close(xs[0], g[key + "_x0"], 1e-3, 3e-3, f"sampler {key} x_0 vs reference")
    assert_close(x0s[0], g[key + "_x0pred"], 1e-3, 3e-3, f"sampler {key} x0_pred vs reference")
    assert_close(xs[0], ox, 1e-3, 3e-3, f"sampler {key} vs oracle")


def test_sampler_single_steps_teacher_forced(gold):
    """One engine step from the oracle's state at several points of the trajectory: tight tolerance, no chaos."""
    from ddnm_b200.sampler import ddnm_diffusion, ddnm_plus_diffusion
    g = gold["sampler_tiny"]
    cfg = U.SimpleUNetConfig.tiny()
    sd = U.init_state_dict(cfg, 1234)
    m = _engine_model(cfg)
    betas_c = torch.from_numpy(g["betas"])
    for name, sy in (("sr4", 0.0), ("sr4", 0.1), ("color", 0.1), ("inpaint", 0.1), ("wh", 0.1), ("deblur", 0.1), ("bicubic", 0.0),
                     ("denoise", 0.1), ("deblur2d", 0.0), ("cs", 0.0)):
        oop = oracle_ops(gold["operators"], 32)[name]
        eop = engine_op(name, oop, 32)
        torch.manual_seed(21)
        x_orig = torch.rand(2, 3, 32, 32) * 2 - 1
        y = oop.A(x_orig.reshape(2, -1))
        for (i, j) in ((900, 800), (500, 400), (100, 0), (0, -1)):
            xt = torch.randn(2, 3, 32, 32)
            z = torch.randn(2, 3, 32, 32)
            abar = SCH.alpha_bar_table(betas_c)
            at, atn = abar[i + 1], abar[j + 1]
            with torch.no_grad():
                et = U.forward(sd, xt, torch.ones(2) * i, cfg)
                x0_t = (xt - et * (1 - at).sqrt()) / at.sqrt()
                resid = oop.A_pinv(oop.A(x0_t.reshape(2, -1)) - y)
                if sy == 0.0:
                    ref = atn.sqrt() * (x0_t - resid.reshape(x0_t.shape)) + (1 - atn).sqrt() * 0.85 * z + (1 - atn).sqrt() * ((1 - 0.85 ** 2) ** 0.5) * et
                else:
                    st, a = (1 - atn).sqrt(), atn.sqrt()
                    ref = a * (x0_t - oop.Lambda(resid, a, sy, st, 0.85).reshape(x0_t.shape)) + \
                        oop.Lambda_noise(z.reshape(2, -1), a, sy, st, 0.85, et.reshape(2, -1)).reshape(x0_t.shape)
            # engine: a 1-pair schedule (i -> j) through the public sampler entry point
            conf = sampler_config(1000, 1, 1)
            from ddnm_b200 import sampler as ES
            orig_pairs = ES.time_pairs
            ES.time_pairs = lambda *a_, **k_: [(i, j)]
            try:
                fn = (lambda: ddnm_diffusion(xt.to(dev), m, betas_c.to(dev), 0.85, eop, y.to(dev), config=conf, noise=z[None].to(dev))) if sy == 0.0 else \
                     (lambda: ddnm_plus_diffusion(xt.to(dev), m, betas_c.to(dev), 0.85, eop, y.to(dev), sy, config=conf, noise=z[None].to(dev)))
                xs, x0s = fn()
            finally:
                ES.time_pairs = orig_pairs
            # x0_t = (xt - et*sqrt(1-at))/sqrt(at) scales the eps error by 1/sqrt(alpha-bar) (95x at t=900, |x0_t| ~ 250):
            # the absolute tolerance follows the tensor's scale; at image scale (late steps) it is north_star's 1e-4
            sc = max(1.0, x0_t.abs().max().item())
            assert_close(x0s[0], x0_t, 1e-3, 1e-4 * sc, f"{name} s{sy} step {i}->{j}: x0_t")
            assert_close(xs[0], ref, 1e-3, 1e-4 * sc, f"{name} s{sy} step {i}->{j}: xt_next")


def test_ddnm_plus_with_lambda_less_operator_raises_like_reference(gold):
    from ddnm_b200.sampler import ddnm_plus_diffusion
    cfg = U.SimpleUNetConfig.tiny()
    m = _engine_model(cfg)
    oop = oracle_ops(gold["operators"], 32)["bicubic"]
    eop = engine_op("bicubic", oop, 32)
    x = torch.randn(2, 3, 32, 32, device=dev)
    y = eop.A(x)
    with pytest.raises(NotImplementedError):
        ddnm_plus_diffusion(x, m, SCH.linear_betas().to(dev), 0.85, eop, y, 0.1, config=sampler_config(4, 1, 1))


def test_product_path_has_no_cpu_fallback():
    from ddnm_b200.model import Model
    cfg = U.SimpleUNetConfig.tiny()
    m = Model(model_config(cfg))
    m.load_state_dict(U.init_state_dict(cfg, 1234))
    with pytest.raises(AssertionError):
        m(torch.zeros(1, 3, 32, 32), torch.zeros(1))     # CPU tensors are rejected, never silently computed on the host


# ------------------------------------------------------------------------------------------------ simplified DDNM+
@pytest.mark.parametrize("case", SIMPLIFIED_CASES, ids=lambda c: c[0])
def test_simplified_ddnm_plus_vs_reference_runner(gold, case):
    """README quick-start path (diffusion.py:211-415): engine vs the image the reference runner saved, and vs the oracle."""
    from ddnm_b200.sampler import SimplifiedDegradation, simplified_ddnm_plus
    from oracle import simplified as SP
    deg, scale, sy, T, tl, tr = case
    g = gold["simplified"]
    cfg = U.SimpleUNetConfig.celeba_hq()
    m = _engine_model(cfg)
    x_T, x_orig, mask, tape = simplified_inputs(g, T, tl, tr)
    D = SimplifiedDegradation(deg, scale, mask, 256)
    A, Ap = SP.degradation(deg, scale, mask, 256)
    y = D.A(x_orig.to(dev))
    assert_close(y, A(x_orig), 1e-4, 1e-5, f"simplified {deg}: A")
    assert_close(D.Ap(y), Ap(A(x_orig)), 1e-4, 1e-5, f"simplified {deg}: Ap")
    xs, _ = simplified_ddnm_plus(x_T.to(dev), m, SCH.linear_betas().to(dev), 0.85, D, y, 2 * sy, config=sampler_config(T, tl, tr),
                                 noise=torch.stack(tape).to(dev))
    img = torch.clamp((xs[0] + 1.0) / 2.0, 0.0, 1.0)
    assert_close(img[:, :, ::4, ::4], g[f"{deg}_s{scale}_sy{sy}_T{T}_l{tl}_r{tr}_img_s4"], 1e-3, 5e-4, f"simplified {deg} vs reference runner")


def test_sampler_full_size_data_consistency(gold):
    """Size-independent property at the real 256x256 size: with sigma_y = 0 the last step has alpha-bar = 1, so the
    returned image is exactly the projection x0_hat and must reproduce the measurement, A(x_0) = y (svd_ddnm.py:57-65)."""
    from ddnm_b200.sampler import ddnm_diffusion
    cfg = U.SimpleUNetConfig.celeba_hq()
    m = _engine_model(cfg)
    g = torch.Generator().manual_seed(77)
    B = 2
    x_orig = (torch.rand(B, 3, 256, 256, generator=g) * 2 - 1).to(dev)
    x_T = torch.randn(B, 3, 256, 256, generator=g).to(dev)
    betas = SCH.linear_betas().to(dev)
    for name, o in oracle_ops(gold["operators"], 256).items():
        eop = engine_op(name, o, 256)
        y = eop.A(x_orig)
        xs, x0s = ddnm_diffusion(x_T, m, betas, 0.85, eop, y, config=sampler_config(4, 1, 1))
        assert torch.isfinite(xs[0]).all(), name
        assert_close(eop.A(xs[0].to(dev)), y, 1e-3, 5e-4, f"{name}: A(x_0) = y at 256x256")
