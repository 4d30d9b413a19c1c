"""The super-resolution UNet (guided_diffusion/unet.py::SuperResModel, :667-681) run by libddnm_b200.so: the stem that
convolves cat([x, bilinear(low_res)]) without materialising either tensor, the native SuperResModel against the reference's
outputs (tests/golden/superres.npz, written by oracle/gen_sr_golden.py), sampling with a low_res conditioning image and the
two-stage sample-then-upsample entry point."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import gen_sr_golden as G
from oracle import operators as O
from oracle import sampler as S
from oracle import schedule as SCH

from helpers import assert_close, sampler_config

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "superres.npz")
CASES = {c[0]: c for c in G.cases()}   # key -> (key, config, batch, input seed, t, labels)
dev = "cuda"


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _case(g, key):
    _, cfg, B, seed, _, labels = CASES[key]
    x, low = G.inputs(cfg, B, seed)
    y = None if labels is None else torch.from_numpy(g[key + "_labels"])
    return cfg, x, torch.from_numpy(g[key + "_t"]), low, y, g[key + "_out"]


def _engine(cfg, graph=True):
    from ddnm_b200.model import SuperResModel
    m = SuperResModel(cfg.image_size, 3, cfg.model_channels, cfg.out_channels, cfg.num_res_blocks, cfg.attention_ds,
                      channel_mult=cfg.channel_mult, num_classes=cfg.num_classes, num_head_channels=cfg.num_head_channels,
                      use_scale_shift_norm=True, resblock_updown=True, small_size=cfg.small_size)
    m.use_cuda_graph = graph
    m.load_state_dict(G.state_dict(cfg))
    return m


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("key", list(CASES))
def test_oracle_superres_matches_reference_fixture(gold, key):
    """the torch restatement (cat + bilinear + UNetModel) reproduces the reference SuperResModel's fixture outputs"""
    cfg, x, t, low, y, ref = _case(gold, key)
    with torch.no_grad():
        out = G.forward(G.state_dict(cfg), x, t, low, cfg, y=y)
    np.testing.assert_allclose(out.numpy(), ref, rtol=1e-4, atol=1e-5)


def test_sr_create_model_keeps_the_reference_interface():
    """sr_create_model's parameters are the reference's (script_util.py:335-351); the checkpoint keys double input_blocks.0"""
    import inspect
    from ddnm_b200.model import sr_create_model
    assert list(inspect.signature(sr_create_model).parameters) == [
        "large_size", "small_size", "num_channels", "num_res_blocks", "learn_sigma", "class_cond", "use_checkpoint",
        "attention_resolutions", "num_heads", "num_head_channels", "num_heads_upsample", "use_scale_shift_norm", "dropout",
        "resblock_updown", "use_fp16"]
    cfg = CASES["sr32"][1]
    assert G.state_dict(cfg)["input_blocks.0.0.weight"].shape == (cfg.model_channels, 6, 3, 3)
    m = sr_create_model(256, 64, 192, 2, learn_sigma=True, class_cond=True, use_checkpoint=False, attention_resolutions="32,16,8",
                        num_heads=4, num_head_channels=64, num_heads_upsample=-1, use_scale_shift_norm=True, dropout=0.0,
                        resblock_updown=True, use_fp16=True)
    assert (m.in_channels, m.image_channels, m.small_size, m.resolution, m.num_classes, m.out_ch) == (6, 3, 64, 256, 1000, 6)
    assert m.channel_mult == (1, 1, 2, 2, 4, 4) and m.attention_resolutions == (8, 16, 32)


# ------------------------------------------------------------------------------------------------ GPU
def _stem(x, low, w, b, fused=True, iters=0):
    from ddnm_b200 import _lib
    N, C, H, W = x.shape
    h, wd = (low.shape[2], low.shape[3]) if low is not None else (0, 0)
    xin = x if fused else torch.cat([x, F.interpolate(low, (H, W), mode="bilinear", align_corners=False)], dim=1)
    out = torch.empty(N, H, W, w.shape[0], device=dev)
    _lib.check(_lib.lib().ddnm_conv_stem_sr(_lib.ptr(xin.contiguous()), _lib.ptr(low.contiguous()) if fused else None, N, C, H, W, h,
                                            wd, _lib.ptr(w.contiguous()), _lib.ptr(b), w.shape[0], _lib.ptr(out), iters, None,
                                            _lib.cur_stream()))
    return out.permute(0, 3, 1, 2)


STEM_SHAPES = [  # (N, H, W, h, w, Cout): odd sizes, batch 1, Cout not a multiple of the 128-channel slab, 1x..4x and uneven ratios
    (1, 33, 33, 17, 17, 36), (2, 64, 64, 32, 32, 128), (1, 65, 47, 16, 30, 96), (3, 128, 128, 64, 64, 200),
    (1, 256, 256, 64, 64, 192), (1, 9, 70, 9, 70, 4), (2, 100, 100, 7, 13, 132)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", STEM_SHAPES)
def test_fused_stem_vs_torch_conv_of_cat_interpolate(shape):
    N, H, W, h, w, Cout = shape
    g = torch.Generator(device=dev).manual_seed(sum(shape))
    x = torch.randn(N, 3, H, W, device=dev, generator=g)
    low = torch.rand(N, 3, h, w, device=dev, generator=g) * 2 - 1
    wt = torch.randn(Cout, 6, 3, 3, device=dev, generator=g) * 0.2
    b = torch.randn(Cout, device=dev, generator=g) * 0.1
    up = F.interpolate(low, (H, W), mode="bilinear", align_corners=False)
    ref = F.conv2d(torch.cat([x, up], dim=1).double(), wt.double(), b.double(), padding=1)
    fused = _stem(x, low, wt, b)
    assert_close(fused, ref, 1e-4, 5e-5, f"fused stem {shape}")
    assert_close(_stem(x, low, wt, b, fused=False), ref, 1e-4, 5e-5, f"composed stem {shape}")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 33, 33, 17, 17), (2, 256, 256, 64, 64), (1, 65, 47, 16, 30), (1, 100, 100, 7, 13)])
def test_fused_interpolation_equals_f_interpolate(shape):
    """with identity centre taps the stem's output channels 3..5 ARE its interpolated channels: they match F.interpolate"""
    N, H, W, h, w = shape
    g = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(N, 3, H, W, device=dev, generator=g)
    low = torch.randn(N, 3, h, w, device=dev, generator=g)
    wt = torch.zeros(8, 6, 3, 3, device=dev)
    for c in range(6):
        wt[c, c, 1, 1] = 1.0
    out = _stem(x, low, wt, torch.zeros(8, device=dev))
    up = F.interpolate(low, (H, W), mode="bilinear", align_corners=False)
    assert torch.equal(out[:, :3], x)
    err = (out[:, 3:6] - up).abs().max().item()
    assert err <= 1e-6 * max(1.0, up.abs().max().item()), f"interpolation differs from F.interpolate by {err:.3e}"
    assert (out[:, 6:] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(CASES))
def test_superres_forward_vs_reference_golden(gold, key):
    cfg, x, t, low, y, ref = _case(gold, key)
    m = _engine(cfg)
    args = (x.to(dev), t.to(dev)) + (() if y is None else (y.to(dev),))
    out = m(*args, low_res=low.to(dev))
    assert out.shape == ref.shape
    assert_close(out, ref, what=f"SuperResModel {key} vs reference")
    assert_close(m(*args, low_res=low.to(dev)), ref, what=f"SuperResModel {key} replay vs reference")


@pytest.mark.gpu
def test_superres_forward_eager_equals_graph_and_is_reproducible(gold):
    cfg, x, t, low, _, _ = _case(gold, "sr32")
    a = _engine(cfg, graph=False)(x.to(dev), t.to(dev), low_res=low.to(dev))
    m = _engine(cfg, graph=True)
    b = m(x.to(dev), t.to(dev), low_res=low.to(dev))
    c = m(x.to(dev), t.to(dev), low_res=low.to(dev))
    assert torch.equal(a, b) and torch.equal(b, c)
    # the conditioning image matters: another low_res changes the output
    d = m(x.to(dev), t.to(dev), low_res=(low * 0.5).to(dev))
    assert not torch.equal(c, d)


@pytest.mark.gpu
def test_superres_argument_errors(gold):
    from ddnm_b200 import _lib
    from ddnm_b200.sampler import ddnm_diffusion
    cfg, x, t, low, _, _ = _case(gold, "sr32")
    m = _engine(cfg)
    with pytest.raises(_lib.DDNMError):
        m(x.to(dev), t.to(dev))                                        # no low_res
    with pytest.raises(_lib.DDNMError):
        m(x.to(dev), t.to(dev), low_res=low[:, :, :16, :16].to(dev))   # not small_size
    op = O.SuperResolution.make(3, 64, 2)
    from ddnm_b200.operators import SuperResolution
    eop = SuperResolution(3, 64, 2, dev, artefacts=(op.U_small, op.singulars_small, op.V_small))
    y = eop.A(x.to(dev))
    with pytest.raises(ValueError):
        ddnm_diffusion(x.to(dev), m, SCH.linear_betas().to(dev), 0.85, eop, y, config=sampler_config(2, 1, 1), seed=1)


def _sr_sampling_setup(gold):
    from ddnm_b200.operators import SuperResolution
    cfg, _, _, low, _, _ = _case(gold, "sr32")
    g = torch.Generator().manual_seed(17)
    x_orig = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
    x_T = torch.randn(2, 3, 64, 64, generator=g)
    oop = O.SuperResolution.make(3, 64, 2)
    eop = SuperResolution(3, 64, 2, dev, artefacts=(oop.U_small, oop.singulars_small, oop.V_small))
    y = oop.A(x_orig.reshape(2, -1))
    return cfg, low, x_T, oop, eop, y


@pytest.mark.gpu
def test_seeded_superres_sampling_is_bit_reproducible_and_matches_composed_reference(gold):
    """DDNM with the super-resolution denoiser, library-drawn noise: two runs give identical bits, and the run equals the loop
    composed in PyTorch (oracle sampler + cat/interpolate/UNet restatement) fed the same draws"""
    from ddnm_b200.noise import TAG_LOOP, randn
    from ddnm_b200.sampler import ddnm_diffusion
    cfg, low, x_T, oop, eop, y = _sr_sampling_setup(gold)
    m = _engine(cfg)
    T, seed = 3, 2024
    betas = SCH.linear_betas()
    conf = sampler_config(T, 1, 1)
    run = lambda: ddnm_diffusion(x_T.to(dev), m, betas.to(dev), 0.85, eop, y.to(dev), config=conf, seed=seed,   # noqa: E731
                                 low_res=low.to(dev))
    a, b = run(), run()
    assert torch.isfinite(a[0][0]).all()
    assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[1][0], b[1][0])
    pairs = SCH.time_pairs(1000, T, 1, 1)
    tape = [randn(seed, x_T.shape, TAG_LOOP, draw=k).cpu() for k in range(len(pairs))]
    sd = G.state_dict(cfg)
    with torch.no_grad():
        ox, ox0 = S.ddnm_sample(x_T, lambda xt, t: G.forward(sd, xt, t, low, cfg), betas, 0.85, oop, y, tape, t_sampling=T)
    assert_close(a[0][0], ox, 1e-3, 3e-3, "seeded SR sampling vs composed reference")
    assert_close(a[1][0], ox0, 1e-3, 3e-3, "seeded SR sampling x0_pred vs composed reference")


@pytest.mark.gpu
def test_superres_sampling_with_torch_drawn_and_simplified_loops(gold):
    """the low_res kwarg of the tape / torch-drawn DDNM+ loop and of the simplified loop"""
    from ddnm_b200.sampler import SimplifiedDegradation, ddnm_plus_diffusion, simplified_ddnm_plus
    cfg, low, x_T, oop, eop, y = _sr_sampling_setup(gold)
    m = _engine(cfg)
    betas = SCH.linear_betas()
    conf = sampler_config(2, 1, 1)
    tape = torch.randn(2, 2, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    xs, _ = ddnm_plus_diffusion(x_T.to(dev), m, betas.to(dev), 0.85, eop, y.to(dev), 0.1, config=conf, noise=tape.to(dev),
                                low_res=low.to(dev))
    sd = G.state_dict(cfg)
    with torch.no_grad():
        ox, _ = S.ddnm_sample(x_T, lambda xt, t: G.forward(sd, xt, t, low, cfg), betas, 0.85, oop, y, tape, t_sampling=2, sigma_y=0.1)
    assert_close(xs[0], ox, 1e-3, 3e-3, "DDNM+ SR sampling vs composed reference")
    deg = SimplifiedDegradation("sr_averagepooling", 2, image_size=64)
    ys = deg.A(x_T.to(dev))
    s1 = simplified_ddnm_plus(x_T.to(dev), m, betas.to(dev), 0.85, deg, ys, 0.0, config=conf, seed=9, low_res=low.to(dev))
    s2 = simplified_ddnm_plus(x_T.to(dev), m, betas.to(dev), 0.85, deg, ys, 0.0, config=conf, seed=9, low_res=low.to(dev))
    assert torch.isfinite(s1[0][0]).all() and torch.equal(s1[0][0], s2[0][0])


@pytest.mark.gpu
def test_sample_then_upsample(gold):
    """base sample at 32 px (classifier-guided when asked), then the 32 -> 64 super-resolution stage conditioned on it: the
    second stage's 2x2 average pool is the first stage's image, and seeded runs repeat bit for bit"""
    from ddnm_b200.model import create_model
    from ddnm_b200.operators import SuperResolution
    from ddnm_b200.superres import sample_then_upsample
    from oracle import unet_openai as UO
    from helpers import openai_model_kwargs
    base_cfg = UO.OpenAIUNetConfig.tiny()
    base = create_model(**openai_model_kwargs(base_cfg))
    base.load_state_dict(UO.init_state_dict(base_cfg, 1234))
    sr = _engine(CASES["sr32"][1])
    g = torch.Generator().manual_seed(23)
    x_orig = torch.rand(2, 3, 32, 32, generator=g) * 2 - 1
    oop = O.SuperResolution.make(3, 32, 4)
    A = SuperResolution(3, 32, 4, dev, artefacts=(oop.U_small, oop.singulars_small, oop.V_small))
    y = A.A(x_orig.to(dev))
    x_T, x_T_sr = torch.randn(2, 3, 32, 32, generator=g).to(dev), torch.randn(2, 3, 64, 64, generator=g).to(dev)
    betas = SCH.linear_betas().to(dev)
    run = lambda: sample_then_upsample(x_T, base, betas, 0.85, A, y, sr, x_T_sr, config=sampler_config(3, 1, 1), seed=5)   # noqa: E731
    lo, hi = run()
    lo2, hi2 = run()
    assert lo.shape == (2, 3, 32, 32) and hi.shape == (2, 3, 64, 64)
    assert torch.equal(lo, lo2) and torch.equal(hi, hi2)
    assert_close(F.avg_pool2d(hi, 2), lo, 1e-3, 1e-4, "average pool of the upsampled image vs the base sample")
    assert_close(A.A(lo), y, 1e-3, 1e-4, "base sample keeps its measurement")
    # classifier-guided first stage (class-conditional base denoiser, a guidance callable as ddnm_diffusion takes it)
    cc_cfg = UO.OpenAIUNetConfig.tiny_class_cond()
    kw = openai_model_kwargs(cc_cfg)
    kw["class_cond"] = True
    cc = create_model(**kw)
    cc.load_state_dict(UO.init_state_dict(cc_cfg, 1234))
    calls = []

    def cond_fn(x, t, classes):
        calls.append(int(t[0].item()))
        return 0.05 * x
    lo_g, hi_g = sample_then_upsample(x_T, cc, betas, 0.85, A, y, sr, x_T_sr, config=sampler_config(3, 1, 1), cls_fn=cond_fn, seed=5)
    assert len(calls) == 3 and torch.isfinite(hi_g).all() and not torch.equal(lo_g, lo)
    assert_close(F.avg_pool2d(hi_g, 2), lo_g, 1e-3, 1e-4, "guided base: average pool of the upsampled image vs the base sample")
