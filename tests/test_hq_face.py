"""hq_demo's face256 configuration: the unconditional denoiser and the keep-mask degradations inpainting / mask_color_sr.
CPU: the oracle (oracle/hq_face.py) against the reference's own p_sample_loop results in tests/golden/hq_face.npz
(oracle/gen_hq_face_golden.py), and the host gating of ddnm_b200.hq.restore.  GPU: the engine against the same fixtures, the seeded
and batch-invariant forms, and the fused per-image-mask step / canvas kernels against an fp64 restatement."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import _golden
from oracle import hq as HQO
from oracle import hq_face as HQF
from oracle import unet_openai as UO

from helpers import assert_close

JUMP = dict(t_T=6, n_sample=1, jump_length=2, jump_n_sample=2)
WSEED = 4321
SEED = 0xFACE256
# key, deg, scale, sigma_y, resize_y, input (h, w), conf name: the cases of oracle/gen_hq_face_golden.py
CASES = [("inpaint", "inpainting", 1, 0.0, False, (256, 256), "face256"),
         ("mcsr2", "mask_color_sr", 2, 0.0, False, (256, 256), "face256"),
         ("mcsr4_noisy", "mask_color_sr", 4, 0.1, False, (256, 256), "face256"),
         ("sr4", "sr_averagepooling", 4, 0.0, False, (256, 256), "face256"),
         ("sr4_w320", "sr_averagepooling", 4, 0.0, True, (64, 80), "inet256")]


@pytest.fixture(scope="module")
def face_gold():
    return _golden("hq_face")


def face_cfg():
    return UO.OpenAIUNetConfig(image_size=256, model_channels=64, num_res_blocks=1, channel_mult=(1, 1, 2, 2, 4, 4),
                               attention_resolutions=(32, 16, 8), num_head_channels=64, out_channels=6, num_classes=None)


def face_inputs(g, i, case):
    key, deg, scale, sy, resize_y, (h, w), name = case
    gen = torch.Generator().manual_seed(int(g[key + "_seed"][0]))
    assert int(g[key + "_seed"][0]) == 900 + i
    gt = torch.rand(2, 3, h, w, generator=gen) * 2 - 1
    H, W = (h * scale, w * scale) if resize_y else (h, w)
    return gt, [torch.randn(2, 3, 256, 256, generator=gen) for _ in range(HQO.count_draws(H, W, JUMP))]


def face_model(class_cond=False, channels=64):
    from ddnm_b200.model import create_model
    return create_model(image_size=256, num_channels=channels, num_res_blocks=1, learn_sigma=True, class_cond=class_cond,
                        attention_resolutions="32,16,8", num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True,
                        use_fp16=False)


def test_fixture_masks_are_a_binary_and_a_fractional_keep_mask(face_gold):
    m = face_gold["masks"]
    assert m.shape == (2, 3, 256, 256) and m.dtype == np.float32
    assert set(np.unique(m[0])) == {0.0, 1.0} and 0 < (m[0] == 0).mean() < 0.5          # mask_mouth.png
    assert ((m[1] > 0) & (m[1] < 1)).any() and not np.array_equal(m[1, 0], m[1, 2])      # fractional edges, channel 2 differs
    assert any(b > a for a, b in zip(HQO.get_schedule_jump(**JUMP)[:-1], HQO.get_schedule_jump(**JUMP)[1:]))   # time travel


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_hq_face_matches_reference(face_gold, i):
    case = CASES[i]
    key, deg, scale, sy, resize_y, hw, name = case
    cfg = face_cfg()
    sd = UO.init_state_dict(cfg, WSEED)
    gt, tape = face_inputs(face_gold, i, case)
    masks = torch.from_numpy(face_gold["masks"])
    # the reference ran mask_color_sr image by image (its color2gray folds a batch into channels): so does the oracle here, which
    # keeps the CPU convolutions at the reference's batch size
    rows = [slice(0, 2)] if deg != "mask_color_sr" else [slice(0, 1), slice(1, 2)]
    with torch.no_grad():
        out = torch.cat([HQF.restore(lambda a, b, c: UO.forward(sd, a, b.float(), cfg), gt[r], None, [z[r] for z in tape], deg=deg,
                                     scale=scale, sigma_y=sy, resize_y=resize_y, respacing=6, jump=JUMP, gt_keep_mask=masks[r],
                                     conf_name=name) for r in rows])
    ref = face_gold[key + "_out_s2"]
    assert out.shape[:2] == (2, 3) and out[:, :, ::2, ::2].shape == ref.shape
    assert np.abs(out[:, :, ::2, ::2].numpy() - ref).max() <= 1e-5


# ------------------------------------------------------------------------------------------------ host gating (no GPU needed)
def _refused(model, exc, match, gt=None, **kw):
    from ddnm_b200 import hq as HQ
    gt = torch.zeros(1, 3, 256, 256) if gt is None else gt
    with pytest.raises(exc, match=match):
        HQ.restore(model, gt, **kw)


def test_an_unconditional_model_is_accepted_and_a_conditional_one_needs_classes():
    uncond, cond = face_model(False, 32), face_model(True, 32)
    # both get past the model check and stop at the (later) mask check
    mask_kw = dict(deg="inpainting", conf_name="face256")
    _refused(uncond, ValueError, "needs gt_keep_mask", **mask_kw)
    _refused(cond, ValueError, "needs gt_keep_mask", classes=torch.tensor([1]), **mask_kw)
    _refused(cond, ValueError, "needs classes", **mask_kw)


def test_other_models_are_refused():
    from ddnm_b200.model import create_model
    _refused(create_model(image_size=256, num_channels=32, num_res_blocks=1, learn_sigma=False, attention_resolutions="32,16,8",
                          num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True), TypeError, "learn_sigma")
    _refused(face_model(False, 32), ValueError, "conf_name", conf_name="celeba")


@pytest.mark.parametrize("deg", ["inpainting", "mask_color_sr"])
def test_masked_degradations_need_face256_and_a_mask(deg):
    m = face_model(False, 32)
    mask = torch.ones(1, 3, 256, 256)
    _refused(m, NotImplementedError, "not supported", deg=deg, scale=2, gt_keep_mask=mask)                 # inet256 (default)
    _refused(m, NotImplementedError, "not supported", deg=deg, scale=2, gt_keep_mask=mask, conf_name="inet256")
    _refused(m, ValueError, "needs gt_keep_mask", deg=deg, scale=2, conf_name="face256")


def test_face256_needs_a_256_high_input_before_resize_y():
    m = face_model(False, 32)
    _refused(m, ValueError, "Only support output size 256x256", gt=torch.zeros(1, 3, 64, 64), deg="sr_averagepooling", scale=4,
             resize_y=True, conf_name="face256")
    _refused(m, ValueError, "Only support output size 256x256", gt=torch.zeros(1, 3, 128, 256), deg="inpainting",
             gt_keep_mask=torch.ones(1, 3, 256, 256), conf_name="face256")


@pytest.mark.parametrize("deg", ["inpainting", "mask_color_sr"])
def test_resize_y_with_a_keep_mask_is_refused(deg):
    _refused(face_model(False, 32), ValueError, "resize_y", deg=deg, scale=4, resize_y=True, gt_keep_mask=torch.ones(1, 3, 256, 256),
             conf_name="face256")


# ------------------------------------------------------------------------------------------------ GPU
def _engine_model(batch_invariant=False):
    m = face_model(False, 64)
    m.load_state_dict(UO.init_state_dict(face_cfg(), WSEED))
    m.batch_invariant = batch_invariant
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_engine_hq_face_vs_reference(face_gold, i):
    from ddnm_b200 import hq as HQ
    case = CASES[i]
    key, deg, scale, sy, resize_y, hw, name = case
    gt, tape = face_inputs(face_gold, i, case)
    out = HQ.restore(_engine_model(), gt.cuda(), None, deg=deg, scale=scale, sigma_y=sy, resize_y=resize_y, timestep_respacing=6,
                     schedule_jump_params=JUMP, noise=torch.stack(tape).cuda(), gt_keep_mask=torch.from_numpy(face_gold["masks"]).cuda(),
                     conf_name=name)
    ref = face_gold[key + "_out_s2"]
    assert not out.is_cuda and out[:, :, ::2, ::2].shape == ref.shape
    assert_close(out[:, :, ::2, ::2], ref, 1e-3, 1e-4 * max(1.0, float(np.abs(ref).max())), f"hq face {key} vs hq_demo")
    sums = face_gold[key + "_sums"]
    assert abs(out.double().sum().item() - sums[0]) <= 1e-3 * sums[1]


@pytest.mark.gpu
@pytest.mark.parametrize("deg,scale", [("inpainting", 1), ("mask_color_sr", 4)])
def test_seeded_face_restore_repeats_bit_for_bit(face_gold, deg, scale):
    from ddnm_b200 import hq as HQ
    m = _engine_model()
    g = torch.Generator().manual_seed(5)
    gt = (torch.rand(2, 3, 256, 256, generator=g) * 2 - 1).cuda()
    kw = dict(deg=deg, scale=scale, sigma_y=0.05, timestep_respacing=6, schedule_jump_params=JUMP, seed=SEED,
              gt_keep_mask=torch.from_numpy(face_gold["masks"]).cuda(), conf_name="face256")
    a, b = HQ.restore(m, gt, None, **kw), HQ.restore(m, gt, None, **kw)
    assert torch.isfinite(a).all() and torch.equal(a, b)
    assert not torch.equal(a[0], a[1])


@pytest.mark.gpu
@pytest.mark.parametrize("deg,scale", [("inpainting", 1), ("mask_color_sr", 2)])
def test_batch_invariant_row_0_is_identical_alone_and_in_a_batch(face_gold, deg, scale):
    from ddnm_b200 import hq as HQ
    m = _engine_model(batch_invariant=True)
    g = torch.Generator().manual_seed(6)
    gt = (torch.rand(2, 3, 256, 256, generator=g) * 2 - 1).cuda()
    masks = torch.from_numpy(face_gold["masks"]).cuda()
    kw = dict(deg=deg, scale=scale, timestep_respacing=6, schedule_jump_params=JUMP, seed=SEED, conf_name="face256")
    one = HQ.restore(m, gt[:1], None, gt_keep_mask=masks[:1], **kw)
    two = HQ.restore(m, gt, None, gt_keep_mask=masks, **kw)
    assert torch.equal(one[0], two[0])


def _ref_ApA(z, m, deg, scale):
    """fp64 Ap(A(z)) of the keep-mask degradations, image by image"""
    if deg == "inpainting":
        return z * m * m
    g = (z * m).mean(1, keepdim=True)                               # color2gray: (z0 + z1 + z2) / 3
    p = torch.nn.functional.avg_pool2d(g, scale)
    return p.repeat_interleave(scale, 2).repeat_interleave(scale, 3).expand(-1, 3, -1, -1) * m   # gray2color(v) = v


@pytest.mark.gpu
@pytest.mark.parametrize("deg,scale,seeded", [("inpainting", 1, False), ("mask_color_sr", 2, False), ("mask_color_sr", 4, True),
                                              ("inpainting", 1, True)])
def test_fused_masked_step_vs_fp64(face_gold, deg, scale, seeded):
    """one ddnm_hq_step / ddnm_hq_step_seeded with a per-image mask (rows 0 and 1 use different masks) against an fp64 restatement
    of x0_t, the masked projection, the posterior mean and the re-noising; also ddnm_hq_canvas_masked"""
    from ddnm_b200 import _lib
    from ddnm_b200.noise import TAG_HQ, randn
    L = _lib.lib()
    B, D = 2, 256
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, 3, D, D, generator=g).cuda()
    mo = torch.randn(B, 6, D, D, generator=g).cuda()
    gt = (torch.rand(B, 3, D, D, generator=g) * 2 - 1).cuda()
    grad = (torch.randn(B, 3, D, D, generator=g) * 0.1).cuda()
    mask = torch.from_numpy(face_gold["masks"]).cuda()
    assert not torch.equal(mask[0], mask[1])
    d = _lib.SimpleDeg()
    d.use_mask, d.use_gray, d.scale, d.img_dim, d.channels, d.mask = 0, 1 if deg == "mask_color_sr" else 0, scale, D, 3, None
    d.image_mask = mask.data_ptr()
    scratch = torch.full((3 * B * 3 * D * D,), float("nan"), device="cuda")
    apy = torch.empty_like(gt)
    _lib.check(L.ddnm_hq_canvas_masked(C.byref(d), _lib.ptr(gt), B, _lib.ptr(apy), _lib.ptr(scratch), _lib.cur_stream()))
    m64 = mask.double()
    assert_close(apy, _ref_ApA(gt.double(), m64, deg, scale), 1e-6, 1e-6, "canvas")

    s = _lib.HqScalars()
    s.c_recip, s.c_recipm1, s.coef1, s.coef2, s.lambda_t, s.gamma_t, s.nonzero, s.clip = 1.7, 1.3, 0.6, 0.35, 0.8, 0.02, 1.0, 1
    rects = (C.c_int * 12)(*([0] * 12))
    x0_hat, x_next = torch.empty_like(x), torch.empty_like(x)
    if seeded:
        ns = _lib.noise_seed(SEED)
        _lib.check(L.ddnm_hq_step_seeded(C.byref(d), _lib.ptr(x), _lib.ptr(mo), 6, _lib.ptr(apy), _lib.ptr(apy), D, D, rects,
                                         _lib.ptr(grad), C.byref(ns), 7, C.byref(s), B, _lib.ptr(x0_hat), _lib.ptr(x_next),
                                         _lib.ptr(scratch), _lib.cur_stream()))
        z = randn(SEED, (B, 3, D, D), TAG_HQ, draw=7)
    else:
        z = torch.randn(B, 3, D, D, generator=g).cuda()
        _lib.check(L.ddnm_hq_step(C.byref(d), _lib.ptr(x), _lib.ptr(mo), 6, _lib.ptr(apy), _lib.ptr(apy), D, D, rects, _lib.ptr(grad),
                                  _lib.ptr(z), C.byref(s), B, _lib.ptr(x0_hat), _lib.ptr(x_next), _lib.ptr(scratch), _lib.cur_stream()))
    f = lambda v: float(np.float32(v))      # noqa: E731  the scalars as the kernel sees them
    x0 = (f(s.c_recip) * x.double() - f(s.c_recipm1) * mo[:, :3].double()).clamp(-1, 1)
    lam = f(s.lambda_t)
    want_x0h = lam * apy.double() + x0 - lam * _ref_ApA(x0, m64, deg, scale)
    mean = f(s.coef1) * want_x0h + f(s.coef2) * x.double() + f(s.gamma_t) * grad.double()
    want_next = mean + np.sqrt(f(s.gamma_t)) * z.double()
    for b in range(B):          # row by row: a kernel that read row 0's mask for row 1 fails here
        assert_close(x0_hat[b], want_x0h[b], 1e-5, 1e-5, f"x0_hat row {b}")
        assert_close(x_next[b], want_next[b], 1e-5, 1e-5, f"x_next row {b}")
