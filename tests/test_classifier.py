"""The classifier of guided sampling (EncoderUNetModel, unet.py:684-895) and its cond_fn gradient (diffusion.py:183-189) run by
libddnm_b200.so.  CPU: the torch restatement (oracle/classifier.py) against the reference's logits and autograd gradients
(tests/golden/classifier.npz, written by oracle/gen_classifier_golden.py).  GPU: the engine against the fixture and the fp64
restatement, determinism, error paths and the guided sampling loop with the native gradient."""
import os

import numpy as np
import pytest
import torch

from oracle import classifier as OC
from oracle import sampler as S
from oracle import schedule as SCH
from oracle import unet_openai as UO
from oracle.gen_classifier_golden import cases, inputs

from helpers import engine_op, openai_model_kwargs, oracle_ops, sampler_config
from test_oracle_golden import sampler_inputs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEEDS = (11, 12)
CASES = {c[0]: c for c in cases()}   # fixture key -> (key, config, batch, input seed, t, labels, scale)


@pytest.fixture(scope="module")
def cgold():
    """classifier.npz merged with its part files (the full-size gradient lives in classifier.part1.npz)"""
    import glob
    g = dict(np.load(os.path.join(GOLD, "classifier.npz")))
    for part in sorted(glob.glob(os.path.join(GOLD, "classifier.part*.npz"))):
        g.update(np.load(part))
    return g


def _shape(cfg):
    class Shape:
        model_channels, channel_mult, in_channels, num_res_blocks = cfg.model_channels, cfg.channel_mult, 3, cfg.num_res_blocks
        attention_resolutions, pool, image_size, out_channels = cfg.attention_resolutions, cfg.pool, cfg.image_size, cfg.out_channels
    return Shape


def _sd(cfg, seed=1234):
    from ddnm_b200.weights import random_state_dict_classifier
    return random_state_dict_classifier(_shape(cfg), seed)


def _case(g, seed):
    return _fixture(g, f"s{seed}")[1:]


def _fixture(g, key):
    """(config, x, t, labels, scale, reference logits, reference gradient) of fixture case `key`"""
    _, cfg, B, seed, _, _, _ = CASES[key]
    return (cfg, inputs(B, seed, cfg.image_size), torch.from_numpy(g[key + "_t"]), torch.from_numpy(g[key + "_labels"]),
            float(g[key + "_scale"]), g[key + "_logits"], g[key + "_grad"])


def _grad_close(got, ref, what):
    """|d| <= 1e-3 |g_ref| + 1e-4 max |g_ref| elementwise"""
    got, ref = torch.as_tensor(got).double().cpu(), torch.as_tensor(ref).double().cpu()
    tol = 1e-3 * ref.abs() + 1e-4 * ref.abs().max()
    err = (got - ref).abs()
    assert (err <= tol).all(), f"{what}: worst excess {(err - tol).max().item():.3e} (max |ref| {ref.abs().max().item():.3e})"


def _logits_close(got, ref, what):
    got, ref = torch.as_tensor(got).double().cpu(), torch.as_tensor(ref).double().cpu()
    assert ((got - ref).abs() <= 1e-4 + 1e-3 * ref.abs()).all(), f"{what}: max |d| {(got - ref).abs().max().item():.3e}"


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("key", list(CASES))
def test_oracle_classifier_matches_reference(cgold, key):
    """tiny (two t / label sets), tiny with the adaptive pool, and the imagenet_256_cc.yml classifier at B = 1"""
    cfg, x, t, y, scale, ref_logits, ref_grad = _fixture(cgold, key)
    sd = {k: v.double() for k, v in _sd(cfg).items()}
    with torch.no_grad():
        logits = OC.forward(sd, x.double(), t.double(), cfg)
    np.testing.assert_allclose(logits.numpy(), ref_logits, rtol=1e-5, atol=1e-6)
    g = OC.cond_fn(sd, cfg, scale)(x.double(), t.double(), y)
    _grad_close(g, ref_grad, "oracle gradient")


def test_create_classifier_refuses_unbuilt_variants():
    from ddnm_b200.model import EncoderUNetModel, create_classifier
    kw = OC.ClassifierConfig.tiny().kwargs()
    for bad in (dict(pool="spatial"), dict(pool="spatial_v2"), dict(resblock_updown=False), dict(use_scale_shift_norm=False),
                dict(use_new_attention_order=True)):
        with pytest.raises(NotImplementedError):
            EncoderUNetModel(**{**kw, **bad})
    with pytest.raises(NotImplementedError):
        create_classifier(512, False, 128, 2, "32,16,8", True, True, "attention")     # fractional channel_mult
    with pytest.raises(ValueError):
        create_classifier(100, False, 128, 2, "32,16,8", True, True, "attention")
    m = create_classifier(256, True, 128, 2, "32,16,8", True, True, "attention")
    assert m.channel_mult == (1, 1, 2, 2, 4, 4) and m.attention_resolutions == (8, 16, 32) and m.out_channels == 1000
    assert m.convert_to_fp16() is None


def test_random_classifier_weights_have_the_reference_keys():
    cfg = OC.ClassifierConfig.tiny()
    sd = _sd(cfg)
    assert sd["out.2.positional_embedding"].shape == (128, 65)
    assert sd["out.2.qkv_proj.weight"].shape == (384, 128, 1)
    assert sd["input_blocks.3.0.skip_connection.weight"].shape == (128, 64, 1, 1)
    assert all(sd[k].abs().max() > 0 for k in sd if k.endswith("out_layers.3.weight") or k.endswith("proj_out.weight"))


# ------------------------------------------------------------------------------------------------ GPU
def _engine(cfg, precision="fp32"):
    from ddnm_b200.model import EncoderUNetModel
    m = EncoderUNetModel(**cfg.kwargs())
    m.precision = precision
    m.load_state_dict({"module." + k: v for k, v in _sd(cfg).items()})
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(CASES))
def test_classifier_engine_vs_reference(cgold, key):
    """every fixture case, the full-size imagenet_256_cc.yml classifier at B = 1 included (split-K data-gradient convolutions at 8x8,
    C = 256 / 512 GroupNorm backward, T = 1024 four-head attention backward, 8-head T = 65 pool)"""
    cfg, x, t, y, scale, ref_logits, ref_grad = _fixture(cgold, key)
    m = _engine(cfg)
    logits = m(x.cuda(), t.cuda())
    _logits_close(logits, ref_logits, "logits")
    g, l2 = m.grad(x.cuda(), t.cuda(), y.cuda(), scale, return_logits=True)
    assert torch.equal(l2, logits)
    _grad_close(g, ref_grad, "gradient")
    sd = {k: v.double() for k, v in _sd(cfg).items()}
    _grad_close(g, OC.cond_fn(sd, cfg, scale)(x.double(), t.double(), y), "gradient vs fp64")


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("pool", ["attention", "adaptive"])
def test_classifier_engine_vs_fp64_oracle(B, pool):
    cfg = OC.ClassifierConfig.tiny()
    cfg.pool = pool
    m = _engine(cfg)
    sd = {k: v.double() for k, v in _sd(cfg).items()}
    x = inputs(B, 20 + B)
    t = torch.tensor([37.0, 420.0, 999.0][:B])
    y = torch.tensor([5, 951, 17][:B])
    ref = OC.cond_fn(sd, cfg, 3.0)(x.double(), t.double(), y)
    with torch.no_grad():
        ref_logits = OC.forward(sd, x.double(), t.double(), cfg)
    g, logits = m.grad(x.cuda(), t.cuda(), y.cuda(), 3.0, return_logits=True)
    _logits_close(logits, ref_logits, f"{pool} B={B} logits")
    _grad_close(g, ref, f"{pool} B={B} gradient")


@pytest.mark.gpu
def test_classifier_gradient_is_deterministic_and_follows_labels_and_t(cgold):
    m = _engine(OC.ClassifierConfig.tiny())
    x, t, y, scale, _, _ = _case(cgold, 11)
    x, t, y = x.cuda(), t.cuda(), y.cuda()
    g = m.grad(x, t, y, scale)
    assert torch.equal(m.grad(x, t, y, scale), g), "graph replay must be bit-identical"
    g_y = m.grad(x, t, torch.tensor([7, 8], device="cuda"), scale)
    g_t = m.grad(x, t + 100, y, scale)
    assert (g_y - g).abs().max() > 1e-3 * g.abs().max() and (g_t - g).abs().max() > 1e-3 * g.abs().max()
    assert torch.equal(m.grad(x, t, y, scale), g)
    assert torch.equal(m.grad(x, t, y, 2 * scale), 2 * g)


@pytest.mark.gpu
def test_classifier_fast_mode(cgold):
    m = _engine(OC.ClassifierConfig.tiny(), precision="fp16")
    x, t, y, scale, ref_logits, ref_grad = _case(cgold, 11)
    g = m.grad(x.cuda(), t.cuda(), y.cuda(), scale).cpu().double()
    ref = torch.from_numpy(ref_grad).double()
    assert torch.isfinite(g).all()
    assert (g - ref).norm() <= 0.05 * ref.norm()


@pytest.mark.gpu
def test_classifier_errors_leave_the_engine_usable(cgold):
    from ddnm_b200._lib import DDNMError
    m = _engine(OC.ClassifierConfig.tiny())
    x, t, y, scale, _, ref_grad = _case(cgold, 11)
    x, t = x.cuda(), t.cuda()
    with pytest.raises(DDNMError, match="label"):
        m.grad(x, t, torch.tensor([0, 1000], device="cuda"), scale)
    with pytest.raises(DDNMError, match="label"):
        m.grad(x, t, torch.tensor([-1, 3], device="cuda"), scale)
    with pytest.raises(DDNMError):
        m.grad(torch.zeros(2, 3, 64, 64, device="cuda"), t, y.cuda(), scale)
    with pytest.raises(DDNMError):
        m.grad(x.cpu(), t, y.cuda(), scale)
    with pytest.raises(NotImplementedError):
        from ddnm_b200.model import EncoderUNetModel
        EncoderUNetModel(**{**OC.ClassifierConfig.tiny().kwargs(), "pool": "spatial"})
    _grad_close(m.grad(x, t, y.cuda(), scale), ref_grad, "gradient after errors")


GUIDED = [("sr4", 6, 0.0), ("inpaint", 6, 0.1)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GUIDED, ids=lambda c: f"{c[0]}-T{c[1]}-s{c[2]}")
def test_guided_loop_native_gradient_matches_callback(gold, case, monkeypatch):
    """ddnm_diffusion / ddnm_plus_diffusion with cls_fn=make_cond_fn(classifier) run the classifier inside the library; the result
    matches the Python-callback path with the fp64 restatement's autograd cond_fn on the same weights."""
    from ddnm_b200.guidance import ClassifierCondFn, make_cond_fn
    from ddnm_b200.model import create_model
    from ddnm_b200.sampler import ddnm_diffusion, ddnm_plus_diffusion
    name, T, sy = case
    ucfg = UO.OpenAIUNetConfig.tiny_class_cond()
    kw = openai_model_kwargs(ucfg)
    kw["class_cond"] = True
    unet = create_model(**kw)
    unet.load_state_dict(UO.init_state_dict(ucfg, 1234))
    ccfg = OC.ClassifierConfig.tiny()
    clf = _engine(ccfg)
    sd64 = {k: v.double().cuda() for k, v in _sd(ccfg).items()}
    oracle_fn = OC.cond_fn(sd64, ccfg, 2.0)
    g = gold["guided_tiny"]
    npairs = len(SCH.time_pairs(1000, T, 1, 1))
    x_T, y, tape = sampler_inputs(g, f"{name}_T{T}_s{sy}", npairs)
    oop = oracle_ops(gold["operators"], 32)[name]
    eop = engine_op(name, oop, 32)
    conf = sampler_config(T, 1, 1)
    betas, noise = SCH.linear_betas().cuda(), torch.stack(tape).cuda()

    def run(cls_fn):
        if sy == 0.0:
            return ddnm_diffusion(x_T.cuda(), unet, betas, 0.85, eop, y.cuda(), cls_fn=cls_fn, config=conf, noise=noise)
        return ddnm_plus_diffusion(x_T.cuda(), unet, betas, 0.85, eop, y.cuda(), sy, cls_fn=cls_fn, config=conf, noise=noise)
    calls = []

    def callback(x, t, classes):
        calls.append(int(classes[0]))
        return oracle_fn(x.double(), t.double(), classes).float()
    ref_x, ref_x0 = run(callback)
    assert len(calls) == npairs and set(calls) == {S.CLASS_NUM}
    cond = make_cond_fn(clf, 2.0)

    def never(*a, **k):
        raise AssertionError("the native guidance path called back into Python")
    monkeypatch.setattr(ClassifierCondFn, "__call__", never)
    xs, x0s = run(cond)
    monkeypatch.undo()
    np.testing.assert_allclose(xs[0].numpy(), ref_x[0].numpy(), rtol=1e-3, atol=3e-3)
    np.testing.assert_allclose(x0s[0].numpy(), ref_x0[0].numpy(), rtol=1e-3, atol=3e-3)
    # the guidance term matters: the same loop guided by a classifier with other weights ends elsewhere
    other = _engine(ccfg)
    other.load_state_dict(_sd(ccfg, 99))
    xo, _ = run(make_cond_fn(other, 2.0))
    assert (xo[0] - xs[0]).abs().max() > 1e-3
    # called from Python, the same object is a drop-in cond_fn returning a CUDA tensor
    xg = x_T.cuda()
    tt = torch.full((2,), 500.0, device="cuda")
    cl = torch.full((2,), S.CLASS_NUM, device="cuda")
    got = cond(xg, tt, cl)
    assert got.is_cuda
    _grad_close(got, oracle_fn(xg.double(), tt.double(), cl), "cond_fn called from Python")
