"""HALO form of the wgmma convolution: for 3x3 stride-1 and upsample-phase layers on maps at least 64 px wide, one TMA load of halo
rows per (dy, 64-channel slice) feeds all column taps through descriptors shifted by 128 B per pixel, and the K order becomes
(dy, slice, dx).  Each case runs with the form forced on and forced off: both must match the fp64 reference, and each other to the
level of reordered fp32 sums.  Launches with a 1x1 side input keep the per-tap form, so there the switch changes no bit."""
import pytest
import torch

from helpers import assert_close
from test_gpu_parity import _conv_ref, _conv_tc

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def lib():
    from ddnm_b200 import _lib
    return _lib


def _both_forms(lib, run):
    L = lib.lib()
    try:
        lib.check(L.ddnm_tc_debug_halo(0))
        plain = run().clone()
        lib.check(L.ddnm_tc_debug_halo(1))
        halo = run()
    finally:
        L.ddnm_tc_debug_halo(1)
    torch.cuda.synchronize()
    return plain, halo


# (N, H, W, Cin, Cout, side channels, residual, up2).  H = W = 64 tiles two image rows of 64 px (halo unit 2 x 66 rows), 128 and 256
# one row of 128 px (1 x 130); Cin = 128..384 gives 2-6 channel slices.  N = 3 at 128^2: 384 tiles over the persistent CTAs, so the
# last round is ragged and CTAs walk different numbers of tiles.
SHAPES = [
    (2, 64, 64, 128, 128, 0, False, False),
    (1, 64, 64, 384, 256, 192, True, False),
    (2, 64, 64, 256, 256, 0, False, False),
    (2, 128, 128, 192, 128, 0, True, False),
    (1, 128, 128, 256, 128, 0, False, False),
    (1, 128, 128, 256, 128, 128, False, False),
    (3, 128, 128, 128, 128, 0, False, False),
    (1, 256, 256, 128, 128, 64, True, False),
    (2, 64, 64, 128, 128, 0, False, True),
    (1, 64, 64, 320, 256, 0, False, True),
    (1, 128, 128, 128, 128, 0, False, True),
]


@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_halo_conv_vs_fp64_and_per_tap_form(lib, shape):
    N, H, W, Cin, Cout, cs, with_res, up2 = shape
    torch.manual_seed(11)
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)   # the epilogue's channel add
    side = torch.randn(N, cs, H, W, device=dev) if cs else None
    sw = torch.randn(Cout, cs, 1, 1, device=dev) / cs ** 0.5 if cs else None
    res = torch.randn(N, Cout, H, W, device=dev) if with_res else None
    plain, halo = _both_forms(lib, lambda: _conv_tc(lib, x, w, b, up2=up2, side=side, side_w=sw, res=res))
    if cs:   # a launch with a 1x1 side input keeps the per-tap form
        assert torch.equal(plain, halo), f"side-input launch {shape} changed with the HALO switch"
    else:    # the two K orders sum the same products in a different order: equal to fp32 rounding, not bit-identical
        assert not torch.equal(plain, halo), f"halo and per-tap forms bit-identical {shape}: the HALO form did not run"
    assert_close(halo, plain, 2e-5, 1e-5, f"halo vs per-tap {shape}")
    assert_close(halo, _conv_ref(x, w, b, up2=up2, side=side, side_w=sw, res=res), rtol=1e-4, atol=5e-5, what=f"halo conv {shape}")


@pytest.mark.parametrize("bn,dual", [(64, 1), (64, 0), (128, 0)], ids=str)
@pytest.mark.parametrize("up2", [False, True], ids=["3x3", "up2"])
def test_halo_conv_other_forms(lib, bn, dual, up2):
    """BN = 64 (4 B stages next to the A units) and the three-instruction (non-DUAL) wgmma sequence."""
    torch.manual_seed(12)
    N, H, W, Cin, Cout = 1, 64, 128, 192, 128
    x = torch.randn(N, Cin, H, W, device=dev)
    w = torch.randn(Cout, Cin, 3, 3, device=dev) / (9 * Cin) ** 0.5
    b = torch.randn(Cout, device=dev)
    L = lib.lib()
    try:
        lib.check(L.ddnm_tc_debug_force_bn(bn))
        lib.check(L.ddnm_tc_debug_dual_mode(dual))
        plain, halo = _both_forms(lib, lambda: _conv_tc(lib, x, w, b, up2=up2))
    finally:
        L.ddnm_tc_debug_force_bn(0)
        L.ddnm_tc_debug_dual_mode(1)
    assert not torch.equal(plain, halo)
    assert_close(halo, plain, 2e-5, 1e-5, "halo vs per-tap")
    assert_close(halo, _conv_ref(x, w, b, up2=up2), rtol=1e-4, atol=5e-5, what="halo conv")


def test_halo_conv_reproducible(lib):
    """Fixed K order and tile -> CTA map: two runs are bit-identical."""
    torch.manual_seed(13)
    x = torch.randn(2, 256, 128, 128, device=dev)
    w = torch.randn(128, 256, 3, 3, device=dev) / (9 * 256) ** 0.5
    b = torch.randn(128, device=dev)
    first = _conv_tc(lib, x, w, b).clone()
    assert torch.equal(first, _conv_tc(lib, x, w, b))
