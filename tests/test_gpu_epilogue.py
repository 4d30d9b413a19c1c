"""The tensor-core epilogue and the attention GEMM against fp64, op by op, in every launch form.

Every wgmma convolution ends in the same epilogue (tc_epilogue_rows: alpha * acc + per-image channel add + residual in modes 0 / 1 / 2,
strided stores), then the GroupNorm-sum bookkeeping of its output (per-warp partials, running pairs carried across a CTA's tiles,
fixed-point flushes) or, for split-K launches, splitk_reduce_kernel.  A/B tests between launch forms cannot see a fault in that
shared code, and whole-network tolerances are too coarse for a dropped or doubled tile of GroupNorm sums, so here each piece is
checked against a float64 reference of the same operation:

  * ddnm_conv_tc_ex builds its launches with the engine's own builders (tc_make_launch, tc_make_up2_launch and the split-K plan
    tc_plan_conv that UNetEngine::emit_tc runs) and returns the GroupNorm sums of its output;
  * ddnm_gemm_tc runs the batched attention GEMM (tc_make_gemm_launch) on operands split by the attention core's raw split.

The GroupNorm sums are checked twice: tightly against the fp64 sums of the kernel's own output (so GEMM rounding drops out and any
misattributed tile, image or N block shows by orders of magnitude) and loosely against the reference output."""
import contextlib
import ctypes
import zlib

import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close

pytestmark = pytest.mark.gpu
dev = "cuda"


@pytest.fixture(scope="module")
def lib():
    from ddnm_b200 import _lib
    return _lib


@contextlib.contextmanager
def _knobs(lib, pingpong=1, dual=1, pair=1, halo=1, deal=-1, bn=0, sms=0):
    """the launch-form debug knobs for the launches built inside the block, reset to their defaults afterwards"""
    L = lib.lib()
    try:
        lib.check(L.ddnm_tc_debug_pingpong(pingpong))
        lib.check(L.ddnm_tc_debug_dual_mode(dual))
        lib.check(L.ddnm_tc_debug_pp_pair(pair))
        lib.check(L.ddnm_tc_debug_halo(halo))
        lib.check(L.ddnm_tc_debug_deal(deal))
        lib.check(L.ddnm_tc_debug_force_bn(bn))
        lib.check(L.ddnm_tc_debug_sm_count(sms))
        yield
    finally:
        L.ddnm_tc_debug_pingpong(1)
        L.ddnm_tc_debug_dual_mode(1)
        L.ddnm_tc_debug_pp_pair(1)
        L.ddnm_tc_debug_halo(1)
        L.ddnm_tc_debug_deal(-1)
        L.ddnm_tc_debug_force_bn(0)
        L.ddnm_tc_debug_sm_count(0)


def _out_hw(H, W, mode, up2):
    return (H // 2, W // 2) if mode == 2 else ((2 * H, 2 * W) if up2 else (H, W))


def _res_hw(oH, oW, res_mode):
    return {0: (oH, oW), 1: (oH // 2, oW // 2), 2: (2 * oH, 2 * oW)}[res_mode]


def _conv_ex(lib, x, w, ca, ca_ld, *, mode=0, up2=False, side=None, side_w=None, res=None, res_mode=0, out_ld=None, split_k=-1,
             invariant=False, terms=3, spare=2):
    """ddnm_conv_tc_ex.  x NCHW; ca [rows][ca_ld] (ca_ld = 0: one broadcast row); res NCHW at its own resolution.  Returns
    (out NHWC [N + spare][oH][oW][out_ld] — NaN wherever the launch must not store —, stats [N][Cout][2] float64, S used)."""
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    oH, oW = _out_hw(H, W, mode, up2)
    out_ld = out_ld or Cout
    out = torch.full((N + spare, oH, oW, out_ld), float("nan"), device=dev)
    stats = torch.zeros(N, Cout, 2, dtype=torch.float64)
    S = ctypes.c_int(0)
    nhwc = lambda t: None if t is None else t.permute(0, 2, 3, 1).contiguous()   # noqa: E731
    # every operand is bound to a name until the call returns: a temporary freed after lib.ptr() would hand its memory to the next one
    xs, ss, ws, sws, cas = nhwc(x), nhwc(side), w.contiguous(), None if side_w is None else side_w.contiguous(), ca.contiguous()
    rs = None
    if res is not None:
        # one spare image behind the residual: a read one image too far stays inside the allocation
        rs = torch.cat([nhwc(res), torch.zeros_like(nhwc(res[:1]))])
    L = lib.lib()
    lib.check(L.ddnm_conv_tc_ex(lib.ptr(xs), N, H, W, Cin, lib.ptr(ws), lib.ptr(cas), ca_ld, Cout, mode, int(up2), lib.ptr(ss),
                                0 if side is None else side.shape[1], lib.ptr(sws), lib.ptr(rs), res_mode, lib.ptr(out), out_ld,
                                split_k, int(invariant), terms, ctypes.cast(stats.data_ptr(), ctypes.POINTER(ctypes.c_double)),
                                ctypes.byref(S), None))
    torch.cuda.synchronize()
    return out, stats, S.value


def _conv_ref(x, w, ca, ca_ld, *, mode=0, up2=False, side=None, side_w=None, res=None, res_mode=0):
    """float64 reference: conv (+ 1x1 side input) + per-image channel add + residual (mode 1: nearest x2 of an H/2 x W/2 map,
    mode 2: 2x2 average of a 2H x 2W map)"""
    x, w = x.double().cpu(), w.double().cpu()
    N, Cout = x.shape[0], w.shape[0]
    if up2:
        x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    o = F.conv2d(x, w, padding=1) if mode == 0 else (F.conv2d(x, w) if mode == 1 else F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2))
    if side is not None:
        o = o + F.conv2d(side.double().cpu(), side_w.double().cpu())
    rows = ca.double().cpu().reshape(-1)
    rows = rows[:Cout].expand(N, Cout) if ca_ld == 0 else rows.reshape(-1, ca_ld)[:N, :Cout]
    o = o + rows[:, :, None, None]
    if res is not None:
        r = res.double().cpu()
        o = o + (r if res_mode == 0 else (F.interpolate(r, scale_factor=2.0, mode="nearest") if res_mode == 1 else F.avg_pool2d(r, 2)))
    return o


def _check_conv(out, stats, ref, N, Cout, what, rtol=1e-4, atol=5e-5):
    """1. output vs fp64; 2. GroupNorm sums vs the fp64 sums of the kernel's own output (tight); 3. vs the reference output (loose);
    4. columns [Cout, ld) and images past the batch keep the NaN sentinel"""
    got = out[:N, :, :, :Cout].double().cpu()                       # N H W C
    refn = ref.permute(0, 2, 3, 1)
    scale = refn.abs().max().item()
    assert_close(got, refn, rtol=rtol, atol=atol * scale, what=what)
    HW = got.shape[1] * got.shape[2]
    v = got.reshape(N, HW, Cout)
    s1, s2, a1 = v.sum(1), (v * v).sum(1), v.abs().sum(1)
    e1 = (stats[:, :, 0] - s1).abs() / (a1 + 1e-30)
    e2 = (stats[:, :, 1] - s2).abs() / (s2 + 1e-30)
    assert e1.max().item() <= 1e-6 and e2.max().item() <= 1e-6, \
        f"{what}: GroupNorm sums vs the kernel's own output: {e1.max().item():.3e} (sum), {e2.max().item():.3e} (sum of squares) " \
        f"at (image, channel) {divmod(int(torch.maximum(e1, e2).argmax()), Cout)}"
    r = refn.reshape(N, HW, Cout)
    ra = r.abs()
    tol = atol * scale + rtol * ra                                    # the per-element output tolerance, summed
    assert ((stats[:, :, 0] - r.sum(1)).abs() <= tol.sum(1)).all(), f"{what}: GroupNorm sums vs the fp64 reference"
    assert ((stats[:, :, 1] - (r * r).sum(1)).abs() <= (2 * ra * tol + tol * tol).sum(1)).all(), \
        f"{what}: GroupNorm sums of squares vs the fp64 reference"
    tail = out[:, :, :, Cout:]
    assert torch.isnan(tail).all(), f"{what}: {int((~torch.isnan(tail)).sum())} stores into columns [Cout, ld)"
    past = out[N:]
    assert torch.isnan(past).all(), f"{what}: {int((~torch.isnan(past)).sum())} stores into images past the batch"


# (id, N, H, W, Cin, Cout, mode, up2, res_mode (None: no residual), per-image chanadd, out_ld extra, split_k, invariant, knobs)
# mode 0: 3x3, 1: 1x1, 2: 3x3 stride 2.  The knobs pick the launch form: ping-pong / DUAL / CTA pairs / HALO / tile deal / BN / SMs.
_PP_OFF = dict(pingpong=0)
_PLAIN = dict(pingpong=0, dual=0)
CONV_CASES = [
    # 8x8, N = 33: two images per tile, the last tile half empty; 64 -> 512 channels (several N tiles)
    ("8x8-n33-pp", 33, 8, 8, 64, 512, 0, False, 0, True, 64, -1, False, dict(sms=16)),
    ("8x8-n33-dual", 33, 8, 8, 64, 512, 0, False, None, True, 0, 1, False, _PP_OFF),
    ("8x8-n33-plain-bn64", 33, 8, 8, 64, 192, 0, False, 0, True, 0, 1, False, dict(_PLAIN, bn=64)),
    ("8x8-n33-inv", 33, 8, 8, 64, 512, 0, False, 0, True, 0, -1, True, {}),
    # split-K at the 8x8 level: the engine's rule (S = 4 on 132 SMs), forced 2 and 4, the batch-invariant rule, a 1x1 side input
    ("8x8-split-rule", 4, 8, 8, 256, 512, 0, False, 0, True, 64, -1, False, {}),
    ("8x8-split2", 33, 8, 8, 256, 192, 0, False, 0, True, 0, 2, False, {}),
    ("8x8-split4-side", 5, 8, 8, 256, 64, 0, False, 0, True, 64, 4, False, dict(side=128)),
    ("8x8-split-inv", 3, 8, 8, 256, 512, 0, False, None, True, 0, -1, True, {}),
    ("8x8-s2-split2", 4, 16, 16, 256, 256, 2, False, None, True, 0, 2, False, {}),
    # 16x16: two tiles per image
    ("16x16-split4", 3, 16, 16, 128, 192, 0, False, 0, True, 0, 4, False, {}),
    ("16x16-split2-bn64", 2, 16, 16, 256, 512, 0, False, 0, False, 64, 2, False, dict(bn=64)),
    ("16x16-res1", 4, 16, 16, 128, 128, 0, False, 1, True, 0, 1, False, {}),
    ("16x16-res2-sms", 6, 16, 16, 128, 128, 0, False, 2, True, 64, 1, False, dict(sms=7)),
    # residual modes of the up / down ResBlocks at the HALO / ping-pong sizes
    ("32x32-res1-pp", 4, 32, 32, 64, 256, 0, False, 1, True, 0, 1, False, dict(sms=16)),
    ("64x64-res2-halo", 2, 64, 64, 128, 128, 0, False, 2, True, 64, 1, False, {}),
    ("64x64-res2-inv", 2, 64, 64, 128, 128, 0, False, 2, True, 0, 1, True, _PP_OFF),
    # 128x128, N = 3: contiguous deal ranges straddle image boundaries; few SMs so CTAs walk many tiles
    ("128-n3-deal", 3, 128, 128, 64, 64, 0, False, 0, True, 0, 1, False, {}),
    ("128-n3-deal-sms", 3, 128, 128, 64, 64, 0, False, None, True, 64, 1, False, dict(sms=10)),
    ("128-n3-deal-nopair", 3, 128, 128, 64, 64, 0, False, 1, True, 0, 1, False, dict(pair=0, sms=22)),
    ("128-n3-rr-sms", 3, 128, 128, 64, 64, 0, False, 0, True, 0, 1, False, dict(deal=0, sms=12)),
    ("128-n3-dual-deal", 3, 128, 128, 64, 64, 0, False, 0, True, 0, 1, False, dict(_PP_OFF, deal=1, sms=40, halo=0)),
    ("128-n3-inv-sms", 3, 128, 128, 64, 64, 0, False, 0, True, 0, 1, True, dict(sms=10)),
    ("128-n2-bn128", 2, 128, 128, 64, 256, 0, False, 0, True, 0, 1, False, dict(bn=128)),
    # 256x256, N = 1
    ("256-n1", 1, 256, 256, 64, 128, 0, False, 0, True, 64, 1, False, {}),
    ("256-n1-sms", 1, 256, 256, 64, 64, 0, False, None, False, 0, 1, False, dict(sms=9)),
    # upsample phases with a per-image channel add (the four phases add into one stats buffer), stride 2, 1x1
    ("up2-64", 2, 32, 32, 128, 128, 0, True, None, True, 0, 1, False, {}),
    ("up2-8to16", 5, 8, 8, 128, 192, 0, True, None, True, 64, 1, False, dict(sms=8)),
    ("up2-inv", 2, 64, 64, 64, 64, 0, True, None, True, 0, 1, True, {}),
    ("s2-128", 3, 128, 128, 64, 128, 2, False, None, True, 0, 1, False, {}),
    ("s2-inv-sms", 2, 64, 64, 128, 64, 2, False, None, True, 64, 1, True, dict(sms=11)),
    ("1x1-side", 2, 32, 32, 128, 384, 1, False, 0, True, 128, 1, False, dict(side=64)),
]


def _conv_inputs(seed, N, H, W, Cin, Cout, mode, up2, res_mode, per_image, side_c=0, ca_ld=None):
    g = torch.Generator(device=dev).manual_seed(seed)
    k = 1 if mode == 1 else 3
    x = torch.randn(N, Cin, H, W, device=dev, generator=g)
    w = torch.randn(Cout, Cin, k, k, device=dev, generator=g) / (k * k * Cin) ** 0.5
    ca_ld = (Cout + 64 if per_image else 0) if ca_ld is None else ca_ld
    ca = torch.randn(N if ca_ld else 1, ca_ld or Cout, device=dev, generator=g)
    oH, oW = _out_hw(H, W, mode, up2)
    res = None
    if res_mode is not None:
        rH, rW = _res_hw(oH, oW, res_mode)
        res = torch.randn(N, Cout, rH, rW, device=dev, generator=g)
    side = torch.randn(N, side_c, oH, oW, device=dev, generator=g) if side_c else None
    sw = torch.randn(Cout, side_c, 1, 1, device=dev, generator=g) / side_c ** 0.5 if side_c else None
    return x, w, ca, ca_ld, res, side, sw


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: c[0])
def test_conv_epilogue_and_groupnorm_sums_vs_fp64(lib, case):
    name, N, H, W, Cin, Cout, mode, up2, res_mode, per_image, ld_extra, split_k, invariant, knobs = case
    knobs = dict(knobs)
    side_c = knobs.pop("side", 0)
    x, w, ca, ca_ld, res, side, sw = _conv_inputs(zlib.crc32(name.encode()) % 1000, N, H, W, Cin, Cout, mode, up2, res_mode, per_image, side_c)
    with _knobs(lib, **knobs):
        out, stats, S = _conv_ex(lib, x, w, ca, ca_ld, mode=mode, up2=up2, side=side, side_w=sw, res=res, res_mode=res_mode or 0,
                                 out_ld=Cout + ld_extra, split_k=split_k, invariant=invariant)
    if split_k > 0:
        assert S == split_k
    ref = _conv_ref(x, w, ca, ca_ld, mode=mode, up2=up2, side=side, side_w=sw, res=res, res_mode=res_mode or 0)
    _check_conv(out, stats, ref, N, Cout, f"conv {name} (S = {S})")


def test_split_rule_is_the_engines(lib):
    """the engine's split-K rule as the op-level entry reports it: the 8x8 level splits, a residual in mode 1 / 2 never does"""
    N, Cin, Cout = 4, 256, 512
    x, w, ca, ca_ld, res, _, _ = _conv_inputs(5, N, 8, 8, Cin, Cout, 0, False, 0, True)
    assert _conv_ex(lib, x, w, ca, ca_ld, res=res)[2] == 4
    assert _conv_ex(lib, x, w, ca, ca_ld, res=res, invariant=True)[2] == 2
    x, w, ca, ca_ld, res, _, _ = _conv_inputs(5, N, 8, 8, Cin, Cout, 0, False, 1, True)
    assert _conv_ex(lib, x, w, ca, ca_ld, res=res, res_mode=1)[2] == 1
    x, w, ca, ca_ld, res, _, _ = _conv_inputs(5, 2, 64, 64, Cin, 128, 0, False, 0, True)   # 128 tiles: more than half the SMs
    assert _conv_ex(lib, x, w, ca, ca_ld, res=res)[2] == 1


def _group_rstd(s1, s2, cnt, groups, eps=1e-6):
    """mean / rstd per (image, group) from per-channel sums, as gn_apply_kernel forms them: in double, var = s2 / n - mean^2"""
    N, C = s1.shape
    s1 = s1.reshape(N, groups, C // groups).sum(-1)
    s2 = s2.reshape(N, groups, C // groups).sum(-1)
    mean = s1 / cnt
    var = (s2 / cnt - mean * mean).clamp_min(0)
    return 1.0 / torch.sqrt(var + eps)


# largest relative rstd error measured over these cases on an H100 SXM (700 W): 5e-7 at 10x, 4.4e-6 at 30x, 4.3e-5 at 100x
# (DESIGN.md, GroupNorm sums)
@pytest.mark.parametrize("factor", [10, 30, 100])
@pytest.mark.parametrize("shape", [(2, 32, 32, 128, 128, 1), (4, 8, 8, 256, 256, -1), (1, 128, 128, 64, 64, 1)], ids=str)
def test_groupnorm_conditioning_with_large_channel_offsets(lib, shape, factor):
    """Per-channel offsets (the bias + timestep add) of `factor` x the output's standard deviation: var = s2/n - mean^2 cancels
    catastrophically if the fp32 partial sums lose too much.  rstd per group from stats_out vs fp64 torch.var of the same output."""
    N, H, W, Cin, Cout, split_k = shape
    groups = 32
    x, w, _, _, _, _, _ = _conv_inputs(factor, N, H, W, Cin, Cout, 0, False, None, False)
    g = torch.Generator(device=dev).manual_seed(factor + 1)
    ca = factor * torch.randn(N, Cout, device=dev, generator=g).sign()   # the conv output has unit standard deviation
    out, stats, _ = _conv_ex(lib, x, w, ca, Cout, out_ld=Cout, split_k=split_k)
    v = out[:N].double().cpu().reshape(N, H * W, groups, Cout // groups)
    var = v.permute(0, 2, 1, 3).reshape(N, groups, -1).var(-1, unbiased=False)
    ref_rstd = 1.0 / torch.sqrt(var + 1e-6)
    rstd = _group_rstd(stats[:, :, 0], stats[:, :, 1], H * W * (Cout // groups), groups)
    err = ((rstd - ref_rstd).abs() / ref_rstd).max().item()
    print(f"groupnorm conditioning {shape} offset {factor}x: max relative rstd error {err:.2e}")
    bound = 1e-4 if factor <= 30 else 2e-4
    assert err <= bound, f"rstd off by {err:.2e} relative at offsets of {factor} x the standard deviation"


def test_fast_fp16_conv_with_stats_is_close_but_not_fp32_grade(lib):
    """terms = 1 (one fp16 product per MAC): outside the fp32-grade tolerance, inside the fp16-product one; its GroupNorm sums still
    match its own output tightly"""
    N, H, W, Cin, Cout = 2, 32, 32, 256, 128
    x, w, ca, ca_ld, res, _, _ = _conv_inputs(77, N, H, W, Cin, Cout, 0, False, 0, True)
    out, stats, _ = _conv_ex(lib, x, w, ca, ca_ld, res=res, terms=1)
    ref = _conv_ref(x, w, ca, ca_ld, res=res)
    got = out[:N, :, :, :Cout].double().cpu()
    refn = ref.permute(0, 2, 3, 1)
    err = ((got - refn).abs() / refn.abs().max()).max().item()
    assert 1e-5 < err < 2e-2, err
    v = got.reshape(N, H * W, Cout)
    assert ((stats[:, :, 0] - v.sum(1)).abs() <= 1e-6 * v.abs().sum(1)).all()
    assert ((stats[:, :, 1] - (v * v).sum(1)).abs() <= 1e-6 * (v * v).sum(1)).all()


# ------------------------------------------------------------------------------------------------------------------------------
# attention GEMMs: QK^T straight from a [T][3C] qkv buffer (legacy order: head stride 3 ch; new order: head stride ch), PV into a
# [T][C] output where head h owns columns [h ch, (h + 1) ch)
# ------------------------------------------------------------------------------------------------------------------------------
def _gemm(lib, a, a_off, a_s, b, b_off, b_s, M, N, K, heads, images, alpha, out, out_s, invariant=False):
    L = lib.lib()
    lib.check(L.ddnm_gemm_tc(lib.ptr(a), a.numel(), a_off, *a_s, lib.ptr(b), b.numel(), b_off, *b_s, M, N, K, heads, images,
                             ctypes.c_float(alpha), lib.ptr(out), *out_s, int(invariant), None))
    torch.cuda.synchronize()


def _gemm_check(got, A, B, alpha, what):
    """got / A / B: [img][head][m][n], [img][head][m][k], [img][head][n][k]; rtol 1e-4 of the row scale sum_k |a||b|"""
    A, B = A.double().cpu(), B.double().cpu()
    ref = alpha * A @ B.transpose(-1, -2)
    scale = abs(alpha) * A.abs() @ B.abs().transpose(-1, -2)
    err = (got.double().cpu() - ref).abs()
    bad = err > 1e-4 * scale + 1e-30
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off, worst {(err / scale).max().item():.2e} of the row scale"


# (T, heads, ch, images) and the launch knobs; T % 128 == 0, ch % 8 == 0 (40 and 96 end in a partial k-block / N tile)
GEMM_CASES = [
    (128, 1, 64, 1, {}),
    (256, 4, 32, 2, {}),
    (256, 3, 40, 5, {}),
    (1024, 4, 64, 2, dict(bn=128)),
    (1024, 8, 96, 1, {}),
    (128, 8, 128, 5, dict(pingpong=0)),
    (256, 3, 96, 2, dict(pingpong=0, dual=0)),
    (1024, 1, 40, 2, dict(pingpong=0, bn=64)),
    (4096, 1, 128, 1, dict(bn=128)),
    (256, 4, 96, 5, dict(sms=9)),
    (128, 3, 40, 2, dict(pingpong=0, sms=5)),
]


@pytest.mark.parametrize("new_order", [False, True], ids=["legacy", "new_order"])
@pytest.mark.parametrize("invariant", [False, True], ids=["", "inv"])
@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: f"T{c[0]}-h{c[1]}-ch{c[2]}-n{c[3]}-{'-'.join(f'{k}{v}' for k, v in c[4].items())}")
def test_attention_gemms_vs_fp64(lib, case, invariant, new_order):
    T, heads, ch, images, knobs = case
    if T >= 4096 and (invariant or new_order):
        pytest.skip("one 4096-token case is enough")
    C = heads * ch
    g = torch.Generator(device=dev).manual_seed(T + heads + ch + images)
    qkv = torch.randn(images, T, 3 * C, device=dev, generator=g)
    hs, q_off, k_off, v_off = (ch, 0, C, 2 * C) if new_order else (3 * ch, 0, ch, 2 * ch)
    alpha = ch ** -0.5
    S = torch.full((images, heads, T, T), float("nan"), device=dev)
    with _knobs(lib, **knobs):
        # S[img, head, i, j] = alpha q_i . k_j
        _gemm(lib, qkv, q_off, (3 * C, hs, T * 3 * C), qkv, k_off, (3 * C, hs, T * 3 * C), T, T, ch, heads, images, alpha, S,
              (heads * T * T, T * T, T), invariant)
        # O[img, t, head ch + c] = sum_j P[img, head, t, j] V[img, j, head, c]; V^T per head as the B operand ([img][head][c][j])
        P = torch.softmax(S, -1)
        vt =torch.stack([qkv[:, :, v_off + h * hs: v_off + h * hs + ch] for h in range(heads)], 1).transpose(-1, -2).contiguous()
        O = torch.full((images + 1, T, C), float("nan"), device=dev)
        _gemm(lib, P, 0, (T, T * T, heads * T * T), vt, 0, (T, ch * T, heads * ch * T), T, ch, T, heads, images, 1.0, O,
              (T * C, ch, C), invariant)
    heads_of = lambda base, off: torch.stack([base[:, :, off + h * hs: off + h * hs + ch] for h in range(heads)], 1)  # noqa: E731
    tag = f"T{T} heads {heads} ch {ch} images {images} {'new' if new_order else 'legacy'} order{' invariant' if invariant else ''} {knobs}"
    assert not torch.isnan(S).any(), f"QK^T {tag}: unwritten scores"
    _gemm_check(S, heads_of(qkv, q_off), heads_of(qkv, k_off), alpha, f"QK^T {tag}")
    assert not torch.isnan(O[:images]).any(), f"PV {tag}: {int(torch.isnan(O[:images]).sum())} columns of some head unwritten"
    assert torch.isnan(O[images:]).all(), f"PV {tag}: stores past the [T][C] output"
    got = O[:images].view(images, T, heads, ch).permute(0, 2, 1, 3)
    _gemm_check(got, P, vt, 1.0, f"PV {tag}")
