"""GPU: the library's seeded noise.  The materialised fill against the numpy contract; the in-register generation of every
step kernel against the tape form fed with that fill (which carries the existing parity evidence over to the seeded mode); the
engine against an oracle run stored in tests/golden/seeded_tiny.npz; invariance to batch split and padding; no noise memory."""
import numpy as np
import pytest
import torch

from oracle import noise as N
from oracle import operators as O
from oracle import schedule as SCH
from oracle import unet_simple as U

from helpers import assert_close, engine_op, gauss_kernel, model_config, oracle_ops, sampler_config
from test_seeded_noise import check_standard_normal

pytestmark = pytest.mark.gpu
dev = "cuda"
SEED = 0xC0FFEE0123456789
DIM = 32


def _engine_model(cfg):
    from ddnm_b200.model import Model
    m = Model(model_config(cfg))
    m.load_state_dict(U.init_state_dict(cfg, 1234))
    return m


def _tape(seed, n_pairs, shape, row_offset=0):
    from ddnm_b200 import noise
    return torch.stack([noise.randn(seed, shape, noise.TAG_LOOP, draw=k, row_offset=row_offset) for k in range(n_pairs)])


@pytest.mark.parametrize("tag,draw,row_offset", [(0, 0, 0), (1, 0, 4), (0, 495, 1 << 20), (3, 7, 63)])
def test_fill_matches_the_numpy_contract(tag, draw, row_offset):
    from ddnm_b200 import noise
    shape = (16, 3, 256, 256)
    z = noise.randn(SEED, shape, tag, draw=draw, row_offset=row_offset).cpu().numpy()
    ref = N.randn(SEED, shape, tag, draw=draw, row_offset=row_offset)
    # libm's fp32 logf / sincospif against float64 numpy rounded once
    assert (np.abs(z - ref) <= 4e-6 * np.maximum(1.0, np.abs(ref))).all(), float(np.abs(z - ref).max())
    check_standard_normal(z.reshape(-1)[: 1 << 21])
    # a row is a function of its global index; an image length that is no multiple of 4 takes the leading values
    assert torch.equal(noise.randn(SEED, (4,) + shape[1:], tag, draw=draw, row_offset=row_offset + 8).cpu(), torch.from_numpy(z[8:12]))
    odd = noise.randn(SEED, (3, 10), tag, draw=draw, row_offset=row_offset).cpu().numpy()
    assert np.array_equal(odd, z.reshape(16, -1)[:3, :10])


def _engine_ops():
    """Every operator kind at 32 x 32, built by the shims' own constructors: name -> (operator, has a Lambda)."""
    from ddnm_b200 import operators as E
    g = torch.Generator().manual_seed(11)
    missing = torch.nonzero(torch.rand(DIM * DIM, generator=g) < 0.4).long().reshape(-1) * 3
    uniform = torch.Tensor([1 / 9] * 9)
    k2 = torch.Tensor([0.1, 0.2, 0.4, 0.2, 0.1])
    return {
        "sr2": (E.SuperResolution(3, DIM, 2, dev), True), "sr4": (E.SuperResolution(3, DIM, 4, dev), True),
        "sr8": (E.SuperResolution(3, DIM, 8, dev), True), "sr16": (E.SuperResolution(3, DIM, 16, dev), True),
        "color": (E.Colorization(DIM, dev), True),
        "inpaint": (E.Inpainting(3, DIM, torch.cat([missing, missing + 1, missing + 2]), dev), True),
        "denoise": (E.Denoising(3, DIM, dev), True),
        "wh": (E.WalshHadamardCS(3, DIM, 4, torch.randperm(DIM * DIM, generator=g), dev), True),
        "deblur_gauss": (E.Deblurring(gauss_kernel().to(dev), 3, DIM, dev), True),
        "deblur_uni": (E.Deblurring(uniform.to(dev), 3, DIM, dev), True),
        "deblur2d": (E.Deblurring2D(gauss_kernel().to(dev), k2.to(dev), 3, DIM, dev), False),
        "bicubic": (E.SRConv(O.SRConv.bicubic_kernel(4).to(dev), 3, DIM, dev, stride=4), False),
        "cs": (E.CS(3, DIM, 0.25, dev), False),
        "general": (E.GeneralA(torch.randn(64, 3 * DIM * DIM, generator=g).to(dev)), False),
    }


def test_in_register_generation_equals_the_tape_form_for_every_operator():
    from ddnm_b200.sampler import ddnm_diffusion, ddnm_plus_diffusion
    m = _engine_model(U.SimpleUNetConfig.tiny())
    betas = SCH.linear_betas().to(dev)
    conf = sampler_config(6, 2, 2)
    pairs = SCH.time_pairs(1000, 6, 2, 2)
    assert any(j > i for i, j in pairs), "the schedule must contain travel-back pairs"
    torch.manual_seed(5)
    x_T, x = torch.randn(2, 3, DIM, DIM, device=dev), torch.rand(2, 3, DIM, DIM, device=dev) * 2 - 1
    tape = _tape(SEED, len(pairs), x_T.shape, row_offset=3)
    for name, (op, has_lambda) in _engine_ops().items():
        y = op.A(x)
        a = ddnm_diffusion(x_T, m, betas, 0.85, op, y, config=conf, seed=SEED, row_offset=3)
        b = ddnm_diffusion(x_T, m, betas, 0.85, op, y, config=conf, noise=tape)
        assert torch.isfinite(a[0][0]).all(), name
        assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[1][0], b[1][0]), f"{name}: DDNM seeded != tape"
        if has_lambda:
            a = ddnm_plus_diffusion(x_T, m, betas, 0.85, op, y, 0.1, config=conf, seed=SEED, row_offset=3)
            b = ddnm_plus_diffusion(x_T, m, betas, 0.85, op, y, 0.1, config=conf, noise=tape)
            assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[1][0], b[1][0]), f"{name}: DDNM+ seeded != tape"


@pytest.mark.parametrize("deg,scale", [("denoising", 1), ("mask_color_sr", 2), ("sr_averagepooling", 4), ("sr_averagepooling", 8),
                                       ("sr_averagepooling", 16)])
def test_simplified_in_register_generation_equals_the_tape_form(deg, scale):
    from ddnm_b200.sampler import SimplifiedDegradation, simplified_ddnm_plus
    m = _engine_model(U.SimpleUNetConfig.tiny())
    mask = (torch.rand(DIM, DIM, generator=torch.Generator().manual_seed(2)) < 0.7).float()
    D = SimplifiedDegradation(deg, scale, mask, DIM)
    torch.manual_seed(6)
    x_T, x = torch.randn(2, 3, DIM, DIM, device=dev), torch.rand(2, 3, DIM, DIM, device=dev) * 2 - 1
    conf = sampler_config(6, 2, 2)
    n_pairs = len(SCH.time_pairs(1000, 6, 2, 2))
    y = D.A(x)
    betas = SCH.linear_betas().to(dev)
    a = simplified_ddnm_plus(x_T, m, betas, 0.85, D, y, 0.2, config=conf, seed=SEED, row_offset=5)
    b = simplified_ddnm_plus(x_T, m, betas, 0.85, D, y, 0.2, config=conf, noise=_tape(SEED, n_pairs, x_T.shape, row_offset=5))
    assert torch.isfinite(a[0][0]).all()
    assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[1][0], b[1][0])


def test_hq_restore_in_register_generation_equals_the_tape_form(gold):
    from ddnm_b200 import hq as HQ
    from ddnm_b200 import noise
    from ddnm_b200.model import create_model
    from oracle import unet_openai as UO
    from test_hq import CASES, JUMP, hq_cfg, hq_inputs
    key, hw, sy = CASES[0]
    m = create_model(image_size=256, num_channels=64, num_res_blocks=1, learn_sigma=True, class_cond=True, attention_resolutions="32,16,8",
                     num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True, use_fp16=False)
    m.load_state_dict(UO.init_state_dict(hq_cfg(), 1234))
    y_img, tape = hq_inputs(gold["hq"], key, hw)
    kw = dict(deg="sr_averagepooling", scale=4, sigma_y=sy, resize_y=True, timestep_respacing=6, schedule_jump_params=JUMP)
    a = HQ.restore(m, y_img.cuda(), torch.tensor([950]), seed=SEED, **kw)
    drawn = torch.stack([noise.randn(SEED, (1, 3, 256, 256), noise.TAG_HQ, draw=k) for k in range(len(tape))])
    b = HQ.restore(m, y_img.cuda(), torch.tensor([950]), noise=drawn, **kw)
    assert torch.isfinite(a).all() and torch.equal(a, b)


@pytest.mark.parametrize("case", [("sr4", 10, 3, 2, 0.0), ("inpaint", 10, 2, 2, 0.1)], ids=lambda c: c[0])
def test_engine_vs_seeded_oracle_golden(gold, case):
    """tests/golden/seeded_tiny.npz: the oracle samplers driven by oracle/noise.py (oracle/gen_seeded_golden.py)."""
    from conftest import _golden
    from ddnm_b200.sampler import ddnm_diffusion, ddnm_plus_diffusion
    name, T, tl, tr, sy = case
    g, gs = gold["sampler_tiny"], _golden("seeded_tiny")
    key = f"{name}_T{T}_l{tl}_r{tr}_s{sy}"
    seed = int(gs["seed"][0])
    oop = oracle_ops(gold["operators"], 32)[name]
    eop = engine_op(name, oop, 32)
    m = _engine_model(U.SimpleUNetConfig.tiny())
    betas = torch.from_numpy(g["betas"]).to(dev)
    x_T, y = torch.from_numpy(g["x_T"]).to(dev), torch.from_numpy(g[key + "_y"]).to(dev)
    conf = sampler_config(T, tl, tr)
    if sy == 0.0:
        xs, x0s = ddnm_diffusion(x_T, m, betas, 0.85, eop, y, config=conf, seed=seed)
    else:
        xs, x0s = ddnm_plus_diffusion(x_T, m, betas, 0.85, eop, y, sy, config=conf, seed=seed)
    # same bounds as the tape-driven comparison of this network (test_gpu_parity.py::test_sampler_vs_oracle_and_golden): the
    # random-init net amplifies per-step rounding (and here the ~1e-7 libm-vs-numpy difference of the draws) over the trajectory
    assert_close(xs[0], gs[key + "_x0"], 1e-3, 3e-3, f"seeded {key} x_0 vs oracle")
    assert_close(x0s[0], gs[key + "_x0pred"], 1e-3, 3e-3, f"seeded {key} x0_pred vs oracle")


def test_result_does_not_depend_on_batch_split_or_padding(gold):
    from ddnm_b200.sampler import ddnm_plus_diffusion, sample_device
    cfg = U.SimpleUNetConfig.tiny()
    oop = oracle_ops(gold["operators"], 32)["sr4"]
    eop = engine_op("sr4", oop, 32)
    torch.manual_seed(9)
    x_T, x = torch.randn(8, 3, DIM, DIM, device=dev), torch.rand(8, 3, DIM, DIM, device=dev) * 2 - 1
    y = eop.A(x)
    conf = sampler_config(5, 2, 2)
    betas = SCH.linear_betas().to(dev)

    def run(model, lo, hi, seed=SEED):
        xs, x0s = ddnm_plus_diffusion(x_T[lo:hi], model, betas, 0.85, eop, y[lo:hi], 0.1, config=conf, seed=seed, row_offset=lo)
        return torch.cat([xs[0], x0s[0]], dim=1)
    whole = run(_engine_model(cfg), 0, 8)
    four = _engine_model(cfg)
    halves = torch.cat([run(four, 0, 4), run(four, 4, 8)])
    assert torch.equal(whole, halves), "B = 8 in one call != two calls of 4"
    padded = run(four, 4, 7)                                   # three rows ride on the 4-row engine, padded
    assert list(four._engines) == [4] and torch.equal(padded, whole[4:7])
    assert torch.equal(run(four, 0, 4), whole[:4]), "the same seed twice"
    assert not torch.equal(run(four, 0, 4, seed=SEED + 1), whole[:4]), "another seed"
    dx0, _ = sample_device(x_T[:4], four, betas, 0.85, eop, y[:4], 0.1, True, conf, seed=SEED)
    assert dx0.is_cuda and torch.equal(dx0.cpu(), whole[:4, :3])


def test_seeded_run_allocates_no_noise_buffers(gold, monkeypatch):
    from ddnm_b200 import sampler
    cfg = U.SimpleUNetConfig.tiny()
    eop = engine_op("sr4", oracle_ops(gold["operators"], 32)["sr4"], 32)
    m = _engine_model(cfg)
    torch.manual_seed(1)
    x_T = torch.randn(4, 3, DIM, DIM, device=dev)
    y = eop.A(torch.rand(4, 3, DIM, DIM, device=dev))
    conf = sampler_config(20, 1, 1)
    betas = SCH.linear_betas().to(dev)
    state = x_T.numel() * 4
    monkeypatch.setattr(sampler, "NOISE_CHUNK_BYTES", 4 * state)          # 20 pairs: the torch-drawn mode needs both chunk buffers

    def rise(**kw):
        sampler.sample_device(x_T, m, betas, 0.85, eop, y, 0.0, False, conf, **kw)      # engine, scratch and result buffers exist
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        sampler.sample_device(x_T, m, betas, 0.85, eop, y, 0.0, False, conf, **kw)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - before
    assert rise() >= 8 * state, "the torch-drawn arm of this comparison no longer holds two chunk buffers"
    assert rise(seed=SEED) < 4 * state
