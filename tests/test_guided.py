"""SURVEY §8 f4 (class-conditional path): the class-conditional UNetModel (imagenet_256_cc.yml) and the classifier-guided branches of
ddnm_diffusion / ddnm_plus_diffusion (svd_ddnm.py:48-52, :109-113), pinned by tests/golden/guided_tiny.npz (the reference executed
with a toy differentiable classifier, oracle/guidance.py).  CPU: oracle vs golden.  GPU: engine vs golden and oracle."""
import numpy as np
import pytest
import torch

from oracle import sampler as S
from oracle import schedule as SCH
from oracle import unet_openai as UO
from oracle.guidance import make_toy_cond_fn

from helpers import assert_close, engine_op, openai_model_kwargs, oracle_ops, sampler_config
from test_oracle_golden import sampler_inputs

CASES = [("sr4", 6, 0.0), ("inpaint", 6, 0.1)]


def _cfg():
    return UO.OpenAIUNetConfig.tiny_class_cond()


# ------------------------------------------------------------------------------------------------ CPU: oracle vs reference
def test_oracle_class_conditional_unet_matches_reference(gold):
    g = gold["guided_tiny"]
    cfg = _cfg()
    sd = UO.init_state_dict(cfg, 1234)
    assert sd["label_emb.weight"].shape == (1000, 4 * cfg.model_channels)
    x, t, labels = torch.from_numpy(g["unet_x"]), torch.from_numpy(g["unet_t"]), torch.from_numpy(g["unet_labels"])
    with torch.no_grad():
        o = UO.forward(sd, x, t, cfg, y=labels)
    assert_close(o, g["unet_out"], 1e-5, 1e-6, "class-conditional unet")
    with pytest.raises(AssertionError):           # unet.py:644-646
        UO.forward(sd, x, t, cfg)
    assert_close(make_toy_cond_fn(cfg.image_size, cfg.num_classes, scale=2.0)(x, t, labels), g["cond_grad"], 1e-5, 1e-7, "toy cond_fn")


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-T{c[1]}-s{c[2]}")
def test_oracle_guided_sampler_matches_reference(gold, case):
    name, T, sy = case
    g = gold["guided_tiny"]
    cfg = _cfg()
    sd = UO.init_state_dict(cfg, 1234)
    key = f"{name}_T{T}_s{sy}"
    npairs = len(SCH.time_pairs(1000, T, 1, 1))
    x_T, y, tape = sampler_inputs(g, key, npairs)
    oop = oracle_ops(gold["operators"], 32)[name]
    cond_fn = make_toy_cond_fn(cfg.image_size, cfg.num_classes, scale=2.0)
    with torch.no_grad():
        ox, ox0 = S.ddnm_sample(x_T, lambda a, b, c: UO.forward(sd, a, b, cfg, y=c), SCH.linear_betas(), 0.85, oop, y, tape,
                                t_sampling=T, travel_length=1, travel_repeat=1, sigma_y=sy, cls_fn=cond_fn)
    assert_close(ox, g[key + "_x0"], 1e-3, 5e-4, f"guided sampler {key}")
    assert_close(ox0, g[key + "_x0pred"], 1e-3, 5e-4, f"guided sampler {key} x0_pred")
    # the guidance term matters: without it the result moves by far more than the tolerance
    with torch.no_grad():
        plain, _ = S.ddnm_sample(x_T, lambda a, b: UO.forward(sd, a, b, cfg, y=torch.ones(a.shape[0], dtype=torch.long) * S.CLASS_NUM),
                                 SCH.linear_betas(), 0.85, oop, y, tape, t_sampling=T, travel_length=1, travel_repeat=1, sigma_y=sy)
    assert (plain - ox).abs().max() > 1e-2


# ------------------------------------------------------------------------------------------------ GPU: engine vs golden
def _engine_model(cfg):
    from ddnm_b200.model import create_model
    kw = openai_model_kwargs(cfg)
    kw["class_cond"] = True
    m = create_model(**kw)
    m.load_state_dict(UO.init_state_dict(cfg, 1234))
    return m


@pytest.mark.gpu
def test_class_conditional_unet_engine_vs_reference_golden(gold):
    g = gold["guided_tiny"]
    cfg = _cfg()
    m = _engine_model(cfg)
    assert m.num_classes == 1000
    x, t = torch.from_numpy(g["unet_x"]).cuda(), torch.from_numpy(g["unet_t"]).cuda()
    labels = torch.from_numpy(g["unet_labels"]).cuda()
    out = m(x, t, labels)
    assert_close(out, g["unet_out"], 1e-3, 1e-4, "class-conditional unet (engine)")
    # other labels give another answer; the same labels the same answer (CUDA-graph replay reads the label buffer each time)
    out2 = m(x, t, torch.tensor([3, 3], device="cuda"))
    assert (out2 - out).abs().max() > 1e-3
    assert torch.equal(m(x, t, labels), out), "replay with the first labels must be bit-identical (fixed-point GroupNorm sums)"
    with pytest.raises(AssertionError):           # unet.py:644-646: y iff class-conditional
        m(x, t)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-T{c[1]}-s{c[2]}")
def test_guided_sampler_engine_vs_reference_golden(gold, case):
    from ddnm_b200.sampler import ddnm_diffusion, ddnm_plus_diffusion
    name, T, sy = case
    g = gold["guided_tiny"]
    cfg = _cfg()
    key = f"{name}_T{T}_s{sy}"
    npairs = len(SCH.time_pairs(1000, T, 1, 1))
    x_T, y, tape = sampler_inputs(g, key, npairs)
    oop = oracle_ops(gold["operators"], 32)[name]
    eop = engine_op(name, oop, 32)
    m = _engine_model(cfg)
    cond_fn = make_toy_cond_fn(cfg.image_size, cfg.num_classes, scale=2.0)
    calls = []

    def counting(x, t, classes):
        calls.append((float(t[0]), int(classes[0]), x.data_ptr()))
        return cond_fn(x, t, classes)
    betas = SCH.linear_betas().cuda()
    noise = torch.stack(tape).cuda()
    conf = sampler_config(T, 1, 1)
    xin = x_T.cuda()
    if sy == 0.0:
        xs, x0s = ddnm_diffusion(xin, m, betas, 0.85, eop, y.cuda(), cls_fn=counting, classes=torch.tensor([1, 2]), config=conf, noise=noise)
    else:
        xs, x0s = ddnm_plus_diffusion(xin, m, betas, 0.85, eop, y.cuda(), sy, cls_fn=counting, classes=torch.tensor([1, 2]), config=conf,
                                      noise=noise)
    assert len(calls) == npairs and all(c[1] == S.CLASS_NUM for c in calls)          # label override (svd_ddnm.py:49)
    assert len({c[2] for c in calls}) == 1                                           # always evaluated at the INPUT x (the quirk)
    assert [c[0] for c in calls] == [float(i) for i, _ in SCH.time_pairs(1000, T, 1, 1)]
    assert_close(xs[0], g[key + "_x0"], 1e-3, 3e-3, f"guided sampler {key} vs reference")
    assert_close(x0s[0], g[key + "_x0pred"], 1e-3, 3e-3, f"guided sampler {key} x0_pred vs reference")


@pytest.mark.gpu
def test_guided_sampler_error_paths(gold):
    from ddnm_b200.sampler import ddnm_diffusion
    g = gold["guided_tiny"]
    cfg = _cfg()
    npairs = len(SCH.time_pairs(1000, 6, 1, 1))
    x_T, y, tape = sampler_inputs(g, "sr4_T6_s0.0", npairs)
    oop = oracle_ops(gold["operators"], 32)["sr4"]
    eop = engine_op("sr4", oop, 32)
    m = _engine_model(cfg)
    conf = sampler_config(6, 1, 1)

    def broken(x, t, classes):
        raise RuntimeError("classifier exploded")
    with pytest.raises(RuntimeError, match="classifier exploded"):       # the callable's exception reaches the caller
        ddnm_diffusion(x_T.cuda(), m, SCH.linear_betas().cuda(), 0.85, eop, y.cuda(), cls_fn=broken, config=conf, noise=torch.stack(tape).cuda())
    # an unconditional denoiser with cls_fn fails like the reference's UNetModel.forward assertion (unet.py:644-646)
    from ddnm_b200.model import create_model
    kw = openai_model_kwargs(UO.OpenAIUNetConfig.tiny())
    mu = create_model(**kw)
    mu.load_state_dict(UO.init_state_dict(UO.OpenAIUNetConfig.tiny(), 1234))
    with pytest.raises(AssertionError):
        ddnm_diffusion(x_T.cuda(), mu, SCH.linear_betas().cuda(), 0.85, eop, y.cuda(), cls_fn=broken, config=conf, noise=torch.stack(tape).cuda())
    # and the engine still works afterwards
    xs, _ = ddnm_diffusion(x_T.cuda(), mu, SCH.linear_betas().cuda(), 0.85, eop, y.cuda(), config=conf, noise=torch.stack(tape).cuda())
    assert torch.isfinite(xs[0]).all()


@pytest.mark.gpu
def test_simplified_ddnm_plus_refuses_a_class_conditional_denoiser():
    """The simplified loop passes no labels, so a class-conditional denoiser is refused before the first step, as the reference's
    model(xt, t) asserts for one (unet.py:644-646); a tape shorter than the schedule is refused before the library reads it."""
    from ddnm_b200._lib import DDNMError
    from ddnm_b200.sampler import SimplifiedDegradation, simplified_ddnm_plus
    cfg = _cfg()
    m = _engine_model(cfg)
    R = cfg.image_size
    D = SimplifiedDegradation("colorization", image_size=R)
    x_T = torch.randn(2, 3, R, R, device="cuda")
    y = D.A(torch.rand(2, 3, R, R, device="cuda") * 2 - 1)
    betas = SCH.linear_betas().cuda()
    conf = sampler_config(4, 1, 1)
    npairs = len(SCH.time_pairs(1000, 4, 1, 1))
    with pytest.raises(DDNMError, match="class-conditional"):
        simplified_ddnm_plus(x_T, m, betas, 0.85, D, y, 0.1, config=conf, noise=torch.randn(npairs, *x_T.shape, device="cuda"))
    with pytest.raises(DDNMError, match="class-conditional"):
        simplified_ddnm_plus(x_T, m, betas, 0.85, D, y, 0.1, config=conf, seed=3)
    with pytest.raises(AssertionError):
        simplified_ddnm_plus(x_T, m, betas, 0.85, D, y, 0.1, config=conf, noise=torch.randn(npairs - 1, *x_T.shape, device="cuda"))
