"""CTA pairs in the ping-pong wgmma convolution: two CTAs of a cluster each load half of every weight k-block and multicast it to
both.  The pairs keep the single-CTA tile deal (the CTAs of a cluster act as workers w and w + n_tiles), so every warpgroup computes
the same tiles in the same order: outputs and GroupNorm sums are bit-identical with pairs on and off.  Cases cover the HALO 3x3 form,
the per-tap form with a 1x1 side input, residual and channel add, one and two N tiles, batch 1 and 16, and deals where the two CTAs
of a cluster get unequal tile counts (one of them walks the extra step as a ghost that only loads and releases its weight halves)."""
import re

import pytest
import torch

from oracle import unet_simple as U

from helpers import assert_close, model_config
from test_gpu_parity import _conv_ref, _conv_tc

pytestmark = pytest.mark.gpu
dev = "cuda"
PAIRED = re.compile(r"conv_tc_pingpong_kernel<\d+, \d, (true|false), false, true>")


@pytest.fixture(scope="module")
def lib():
    from ddnm_b200 import _lib
    return _lib


def _paired_kernel_ran(run):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    return any(PAIRED.search(e.name) for e in prof.events())


def _arms(lib, run, deal=-1):
    """(pairs off, pairs on) of the same launch, and whether the paired arm ran on the paired kernel"""
    L = lib.lib()
    try:
        lib.check(L.ddnm_tc_debug_deal(deal))
        lib.check(L.ddnm_tc_debug_pp_pair(0))
        single = run().clone()
        lib.check(L.ddnm_tc_debug_pp_pair(1))
        paired = run().clone()
        ran = _paired_kernel_ran(run)
    finally:
        L.ddnm_tc_debug_deal(-1)
        L.ddnm_tc_debug_pp_pair(1)
    torch.cuda.synchronize()
    return single, paired, ran


# (N, H, W, Cin, Cout, up2, side channels, residual, deal).  Cout = 128 is one N tile at BN = 128, Cout = 256 two (clusters pair
# workers w and w + 2); 133 images of 8^2 at Cout = 256 are 134 tiles round-robin, so workers 0 / 1 walk two and their peers 2 / 3 one.  256^2 / 128^2 / 64^2 3x3 run the
# HALO form, side-input launches the per-tap form.  deal 1 forces contiguous tile ranges: 512 tiles over 132 CTAs give the CTAs of
# some clusters 3 and 4 tiles.  265 images of 8^2 pack two per tile: 133 tiles round-robin, so CTA 0 walks two and its peer one.
SHAPES = [
    (1, 256, 256, 128, 128, False, 0, False, -1),
    (1, 256, 256, 128, 128, False, 0, True, 1),
    (3, 128, 128, 256, 128, False, 0, True, -1),
    (16, 64, 64, 128, 128, False, 0, False, 1),
    (16, 64, 64, 256, 128, False, 0, False, 1),
    (2, 128, 128, 128, 128, False, 64, True, -1),
    (2, 128, 128, 128, 128, False, 128, False, 1),
    (265, 8, 8, 64, 128, False, 0, True, -1),
    (16, 64, 64, 128, 256, False, 0, True, -1),
    (16, 32, 32, 256, 256, False, 128, False, -1),
    (133, 8, 8, 64, 256, False, 0, True, -1),
]


@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_pair_conv_bit_identical_to_single_cta(lib, shape):
    N, H, W, Cin, Cout, up2, cs, with_res, deal = shape
    torch.manual_seed(71)
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)   # the epilogue's channel add
    side = torch.randn(N, cs, H, W, device=dev) if cs else None
    sw = torch.randn(Cout, cs, 1, 1, device=dev) / cs ** 0.5 if cs else None
    oH, oW = (2 * H, 2 * W) if up2 else (H, W)
    res = torch.randn(N, Cout, oH, oW, device=dev) if with_res else None
    single, paired, ran = _arms(lib, lambda: _conv_tc(lib, x, w, b, up2=up2, side=side, side_w=sw, res=res), deal)
    assert ran, f"{shape}: the launch did not run on CTA pairs"
    assert torch.equal(single, paired), f"CTA pairs {shape}: max diff {(single - paired).abs().max().item():.3e}"
    assert_close(paired, _conv_ref(x, w, b, up2=up2, side=side, side_w=sw, res=res), rtol=1e-4, atol=5e-5, what=f"paired conv {shape}")


def _celeba(graph):
    from ddnm_b200.model import Model
    cfg = U.SimpleUNetConfig.celeba_hq()
    m = Model(model_config(cfg))
    m.load_state_dict(U.init_state_dict(cfg, 1234))
    m.use_cuda_graph = graph
    return m


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_pair_celeba_forward_bit_identical(lib, graph):
    """celeba network at B = 2: GroupNorm sums over contiguous tile ranges (the paired forward reads them back through every
    normalisation, so a changed sum changes the output), conv2 + 1x1 shortcut launches; each arm replays bit-identically."""
    torch.manual_seed(73)
    x = torch.randn(2, 3, 256, 256, device=dev)
    t = torch.tensor([612.0, 87.0], device=dev)
    outs = {}
    try:
        for on in (0, 1):
            lib.check(lib.lib().ddnm_tc_debug_pp_pair(on))   # read when the engine builds its launches
            m = _celeba(graph)
            first = m(x, t).clone()
            assert torch.equal(m(x, t), first), f"forward not reproducible (pairs {on})"
            outs[on] = first
            if on:
                assert _paired_kernel_ran(lambda: m(x, t)), "no launch of the forward ran on CTA pairs"
    finally:
        lib.check(lib.lib().ddnm_tc_debug_pp_pair(1))
    assert torch.equal(outs[0], outs[1]), f"paired forward differs: max diff {(outs[0] - outs[1]).abs().max().item():.3e}"
