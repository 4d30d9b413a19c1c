"""Ping-pong form of the wgmma convolution: two consumer warpgroups that each own a whole 128-row tile and take turns on the tensor
cores, so one tile's epilogue overlaps the next tile's MMAs.  It issues the products of the three-instruction form in the same order
for every output element, so a convolution is bit-identical to conv_tc_kernel with DUAL off.  Every op-level case has more tiles than
CTAs, so the launch runs on the ping-pong kernel; with DUAL on (the default) the other kernel would not give the same bits.  Split-K,
residual modes 1 / 2, per-image channel adds, GroupNorm sums, attention GEMMs and the one-product fp16 mode are checked op by op
against fp64 in test_gpu_epilogue.py; the engine-level checks here add that whole forwards with ping-pong on and off agree to fp32
rounding of the statistics, and that each is bit-reproducible."""
import pytest
import torch

from oracle import unet_openai as UO
from oracle import unet_simple as U

from helpers import assert_close, model_config, openai_model_kwargs
from test_gpu_parity import _conv_ref, _conv_tc

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def lib():
    from ddnm_b200 import _lib
    return _lib


def _arms(lib, run, bn=0):
    """(conv_tc_kernel without DUAL, the default launch with ping-pong on)"""
    L = lib.lib()
    try:
        lib.check(L.ddnm_tc_debug_force_bn(bn))
        lib.check(L.ddnm_tc_debug_pingpong(0))
        lib.check(L.ddnm_tc_debug_dual_mode(0))
        plain = run().clone()
        lib.check(L.ddnm_tc_debug_pingpong(1))
        lib.check(L.ddnm_tc_debug_dual_mode(1))
        pp = run()
    finally:
        L.ddnm_tc_debug_force_bn(0)
        L.ddnm_tc_debug_pingpong(1)
        L.ddnm_tc_debug_dual_mode(1)
    torch.cuda.synchronize()
    return plain, pp


# (N, H, W, Cin, Cout, mode, up2, side channels, residual, BN).  mode 0: 3x3, 1: 1x1, 2: 3x3 stride 2.  64^2 / 128^2 / 256^2 3x3 and
# the upsample phases run the HALO form; N = 3 at 128^2 deals 384 tiles to 132 CTAs, so CTAs walk 2 or 3 tiles (an odd count: the
# second warpgroup sits out the last turn); 8^2 with N = 33 packs two images per tile and leaves the last tile half empty.
SHAPES = [
    (4, 64, 64, 128, 256, 0, False, 0, False, 0),
    (2, 128, 128, 192, 128, 0, False, 0, True, 0),
    (1, 256, 256, 128, 128, 0, False, 0, False, 0),
    (3, 128, 128, 128, 128, 0, False, 0, False, 0),
    (8, 128, 128, 64, 128, 2, False, 0, False, 0),
    (4, 64, 64, 192, 256, 1, False, 0, False, 0),
    (4, 64, 64, 128, 256, 0, True, 0, False, 0),
    (2, 128, 128, 128, 128, 0, False, 64, True, 0),
    (2, 128, 128, 128, 128, 0, False, 0, True, 64),
    (4, 64, 64, 128, 256, 0, True, 0, False, 64),
    (33, 8, 8, 64, 1024, 0, False, 0, True, 0),
]


@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_pingpong_conv_bit_identical_to_three_instruction_form(lib, shape):
    N, H, W, Cin, Cout, mode, up2, cs, with_res, bn = shape
    torch.manual_seed(31)
    k = 1 if mode == 1 else 3
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, k, k, device=dev) / (k * k * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)   # the epilogue's channel add
    side = torch.randn(N, cs, H, W, device=dev) if cs else None
    sw = torch.randn(Cout, cs, 1, 1, device=dev) / cs ** 0.5 if cs else None
    oH, oW = (H // 2, W // 2) if mode == 2 else ((2 * H, 2 * W) if up2 else (H, W))
    res = torch.randn(N, Cout, oH, oW, device=dev) if with_res else None
    plain, pp = _arms(lib, lambda: _conv_tc(lib, x, w, b, mode=mode, up2=up2, side=side, side_w=sw, res=res), bn)
    assert torch.equal(plain, pp), f"ping-pong {shape}: max diff {(plain - pp).abs().max().item():.3e}"
    assert_close(pp, _conv_ref(x, w, b, mode=mode, up2=up2, side=side, side_w=sw, res=res), rtol=1e-4, atol=5e-5,
                 what=f"ping-pong conv {shape}")


def _forward_both_ways(make, x, t, precision=None):
    from ddnm_b200 import _lib
    outs = {}
    try:
        for on in (0, 1):
            _lib.check(_lib.lib().ddnm_tc_debug_pingpong(on))   # read when the engine builds its launches
            m = make()
            if precision:
                m.precision = precision
            first = m(x, t).clone()
            assert torch.equal(m(x, t), first), f"forward not reproducible (ping-pong {on})"
            outs[on] = first
    finally:
        _lib.check(_lib.lib().ddnm_tc_debug_pingpong(1))
    return outs[0], outs[1]


def _simple(cfg):
    from ddnm_b200.model import Model
    m = Model(model_config(cfg))
    m.load_state_dict(U.init_state_dict(cfg, 1234))
    return m


def _openai(cfg):
    from ddnm_b200.model import create_model
    m = create_model(**openai_model_kwargs(cfg))
    m.load_state_dict(UO.init_state_dict(cfg, 1234))
    return m


def test_pingpong_celeba_forward():
    """celeba network, B = 2: HALO layers, conv2 + 1x1 shortcut launches, GroupNorm sums over contiguous tile ranges, split-K at 8x8."""
    cfg = U.SimpleUNetConfig.celeba_hq()
    torch.manual_seed(41)
    x = torch.randn(2, 3, 256, 256, device=dev)
    t = torch.tensor([612.0, 87.0], device=dev)
    off, on = _forward_both_ways(lambda: _simple(cfg), x, t)
    scale = off.abs().max().item()
    assert (off - on).abs().max().item() <= 2e-5 * scale


def test_pingpong_openai_tiny_forward():
    """openai network (residual modes 1 / 2 of the up/down ResBlocks, scale-shift norm, attention GEMMs with batched B) at B = 32,
    so its 32^2 level and attention GEMMs have more tiles than CTAs."""
    cfg = UO.OpenAIUNetConfig.tiny()
    torch.manual_seed(42)
    x = torch.randn(32, 3, 32, 32, device=dev)
    t = torch.linspace(0, 999, 32, device=dev)
    off, on = _forward_both_ways(lambda: _openai(cfg), x, t)
    scale = off.abs().max().item()
    assert (off - on).abs().max().item() <= 2e-5 * scale


def test_pingpong_fp16_mode_forward():
    """precision = 'fp16': one fp16 product per MAC (the TERMS = 1 instantiations)."""
    cfg = U.SimpleUNetConfig.tiny()
    torch.manual_seed(43)
    x = torch.randn(32, 3, 32, 32, device=dev)
    t = torch.linspace(0, 999, 32, device=dev)
    off, on = _forward_both_ways(lambda: _simple(cfg), x, t, precision="fp16")
    scale = off.abs().max().item()
    assert (off - on).abs().max().item() <= 2e-5 * scale
