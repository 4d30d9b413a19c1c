"""guided-diffusion's ImageNet UNet family run by libddnm_b200.so: QKVAttention (use_new_attention_order), a fixed head count per
block (num_heads / num_heads_upsample with num_head_channels = -1) and head widths that are not a multiple of 64 on the tensor
cores.  Fixtures: tests/golden/zoo.npz (reduced-width nets, one per variant, and the 64 / 128 classifiers) and
tests/golden/zoo_published*.npz (the 64 and 128 base models and the 64 -> 256 and 128 -> 512 upsamplers at full width), written by
oracle/gen_zoo_golden.py from the reference modules."""
import os

import numpy as np
import pytest
import torch

from oracle import gen_zoo_golden as G
from oracle import unet_zoo as Z

from helpers import assert_close, sampler_config

HERE = os.path.dirname(os.path.abspath(__file__))
REDUCED = {c[0]: c for c in G.reduced_cases()}       # key -> (key, config, batch, input seed, t, labels)
PUBLISHED = {c[0]: c for c in G.published_cases()}
CLASSIFIERS = {c[0]: c for c in G.classifier_cases()}
dev = "cuda"


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(HERE, "golden", "zoo.npz")))


@pytest.fixture(scope="module")
def gold_pub():
    return G.load_published(os.path.join(HERE, "golden"))


def _case(cases, g, key):
    _, cfg, B, seed, _, labels = cases[key]
    x, low = G.inputs(cfg, B, seed)
    y = None if labels is None else torch.from_numpy(g[key + "_labels"])
    return cfg, x, torch.from_numpy(g[key + "_t"]), low, y, g[key + "_out"]


def _native(cfg, graph=True, sd=None):
    from ddnm_b200.model import SuperResModel, UNetModel
    kw = cfg.reference_kwargs()
    m = SuperResModel(**kw, small_size=cfg.small_size) if cfg.small_size else UNetModel(**kw)
    m.use_cuda_graph = graph
    m.load_state_dict(G.state_dict(cfg) if sd is None else sd)
    return m


def _call(m, x, t, y, low):
    args = (x.to(dev), t.to(dev)) + (() if y is None else (y.to(dev),))
    return m(*args, low_res=low.to(dev)) if low is not None else m(*args)


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("key", list(REDUCED))
def test_oracle_zoo_matches_reference_fixture(gold, key):
    """the torch restatement with QKVAttention and the head-count rule reproduces the reference UNetModel's outputs"""
    cfg, x, t, low, y, ref = _case(REDUCED, gold, key)
    with torch.no_grad():
        out = Z.forward(G.state_dict(cfg), x, t, cfg, y=y, low_res=low)
    np.testing.assert_allclose(out.numpy(), ref, rtol=1e-4, atol=1e-5)


def test_oracle_published_64_base_matches_reference_fixture(gold_pub):
    cfg, x, t, low, y, ref = _case(PUBLISHED, gold_pub, "base64")
    with torch.no_grad():
        out = Z.forward(G.state_dict(cfg), x, t, cfg, y=y, low_res=low)
    np.testing.assert_allclose(out.numpy(), ref, rtol=1e-4, atol=1e-5)


def test_head_count_rule():
    """unet.py:277-283, 452-453: num_head_channels wins; else num_heads in the input / middle blocks and num_heads_upsample
    (-1: num_heads) in the output blocks"""
    c = REDUCED["h40"][1]
    assert Z.attention_blocks(c) == [("in.3", 16, 320, 8), ("out.0", 16, 320, 4)]   # out.1 ends in its upsampling ResBlock
    assert PUBLISHED["up256"][1].heads(384, False) == 4 and PUBLISHED["up256"][1].heads(384, True) == 4
    assert PUBLISHED["base64"][1].heads(576, True) == 9


PUBLISHED_FLAGS = {   # the flag sets the guided-diffusion ImageNet checkpoints are published with
    "base64": dict(image_size=64, num_channels=192, num_res_blocks=3, learn_sigma=True, class_cond=True, attention_resolutions="32,16,8",
                   num_head_channels=64, use_new_attention_order=True, use_scale_shift_norm=True, resblock_updown=True, dropout=0.1,
                   use_fp16=True),
    "base128": dict(image_size=128, num_channels=256, num_res_blocks=2, learn_sigma=True, class_cond=True, attention_resolutions="32,16,8",
                    num_heads=4, use_scale_shift_norm=True, resblock_updown=True, use_fp16=True),
}
SR_FLAGS = {
    "up256": dict(large_size=256, small_size=64, num_channels=192, num_res_blocks=2, learn_sigma=True, class_cond=True,
                  use_checkpoint=False, attention_resolutions="32,16,8", num_heads=4, num_head_channels=-1, num_heads_upsample=-1,
                  use_scale_shift_norm=True, dropout=0.0, resblock_updown=True, use_fp16=True),
    "up512": dict(large_size=512, small_size=128, num_channels=192, num_res_blocks=2, learn_sigma=True, class_cond=True,
                  use_checkpoint=False, attention_resolutions="32,16", num_heads=4, num_head_channels=64, num_heads_upsample=-1,
                  use_scale_shift_norm=True, dropout=0.0, resblock_updown=True, use_fp16=True),
}


def _published_model(key):
    from ddnm_b200.model import create_model, sr_create_model
    return create_model(**PUBLISHED_FLAGS[key]) if key in PUBLISHED_FLAGS else sr_create_model(**SR_FLAGS[key])


@pytest.mark.parametrize("key", list(PUBLISHED))
def test_published_flag_sets_are_accepted(key):
    """create_model / sr_create_model build the published networks instead of raising; their shape is the fixture's"""
    m = _published_model(key)
    cfg = PUBLISHED[key][1]
    assert (m.resolution, m.model_channels, m.num_res_blocks, m.channel_mult) == (cfg.image_size, cfg.model_channels,
                                                                                  cfg.num_res_blocks, cfg.channel_mult)
    assert set(m.attention_resolutions) == set(cfg.attention_ds)
    assert (m.num_head_channels, m.use_new_attention_order) == (cfg.num_head_channels, cfg.use_new_attention_order)
    if cfg.num_head_channels == -1:
        assert (m.num_heads, m.num_heads_upsample) == (cfg.num_heads, cfg.num_heads)
    assert m.num_classes == 1000 and m.out_ch == 6


def test_other_refusals_are_kept():
    from ddnm_b200.model import UNetModel
    base = dict(image_size=32, in_channels=3, model_channels=64, out_channels=6, num_res_blocks=1, attention_resolutions=(2,),
                channel_mult=(1, 2), num_heads=2, use_scale_shift_norm=True, resblock_updown=True)
    UNetModel(**base)
    with pytest.raises(NotImplementedError):
        UNetModel(**{**base, "use_scale_shift_norm": False})
    with pytest.raises(NotImplementedError):
        UNetModel(**{**base, "resblock_updown": False})
    with pytest.raises(NotImplementedError):
        UNetModel(**{**base, "channel_mult": (0.5, 1)})
    with pytest.raises(ValueError):
        UNetModel(**{**base, "num_heads": 0})
    with pytest.raises(ValueError):
        UNetModel(**{**base, "num_head_channels": 0})


def test_openai_cfg_appends_the_attention_fields():
    """ddnm_openai_cfg gains num_heads, num_heads_upsample, new_attention_order at its end (the earlier layout is a prefix)"""
    from ddnm_b200 import _lib
    names = [f[0] for f in _lib.OpenAICfg._fields_]
    assert names[-4:] == ["low_res", "num_heads", "num_heads_upsample", "new_attention_order"]
    hdr = open(os.path.join(HERE, "..", "include", "ddnm_b200.h")).read()
    body = hdr[hdr.index("int low_res;"):hdr.index("} ddnm_openai_cfg;")]
    assert body.index("int num_heads;") < body.index("int num_heads_upsample;") < body.index("int new_attention_order;")


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("key", list(REDUCED))
def test_zoo_forward_vs_reference_golden(gold, key):
    cfg, x, t, low, y, ref = _case(REDUCED, gold, key)
    m = _native(cfg)
    a = _call(m, x, t, y, low)
    assert a.shape == ref.shape
    assert_close(a, ref, what=f"{key} vs reference")
    b = _call(m, x, t, y, low)
    assert torch.equal(a, b), "graph replays differ"
    e = _call(_native(cfg, graph=False), x, t, y, low)
    assert torch.equal(a, e), "eager and graph forwards differ"


# (fixture key, attention order): widths 96 / 48 (h96), 40 / 80 (h40), 128 / 192 (wide), each in both orders
TAP_CASES = [(k, new) for k in ("h96", "h40", "wide_new") for new in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("key,new_order", TAP_CASES)
def test_attention_block_taps_vs_fp64_oracle(gold, key, new_order):
    import dataclasses
    cfg0, x, t, low, y, _ = _case(REDUCED, gold, key)
    cfg = dataclasses.replace(cfg0, use_new_attention_order=new_order)
    sd = G.state_dict(cfg)
    taps = {}
    with torch.no_grad():
        Z.forward(sd, x.double().to(dev), t.double().to(dev), cfg, taps=taps, y=None if y is None else y.to(dev))
    m = _native(cfg, sd=sd)
    _call(m, x, t, y, low)
    blocks = Z.attention_blocks(cfg)
    widths = {c // h for _, r, c, h in blocks if r * r % 128 == 0}
    assert widths, "no tensor-core attention block in the case"
    for name, r, c, heads in blocks:
        got = m.read_tap(x.shape[0], name, (x.shape[0], c, r, r))
        ref = taps[name]
        assert_close(got, ref, 1e-3, 1e-4 * max(1.0, ref.abs().max().item()),
                     f"{key} order={'new' if new_order else 'legacy'} {name}: {heads} heads of {c // heads} at {r}x{r}")


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(PUBLISHED))
def test_published_shapes_vs_reference_golden(gold_pub, key):
    cfg, x, t, low, y, ref = _case(PUBLISHED, gold_pub, key)
    m = _published_model(key)
    m.load_state_dict(G.state_dict(cfg))
    out = _call(m, x, t, y, low)
    if key == "up512":
        out = out[G.CROP]
    assert out.shape == ref.shape
    assert_close(out, ref, what=f"published {key} vs reference")
    del m


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(CLASSIFIERS))
def test_published_classifiers_vs_reference_golden(gold, key):
    from ddnm_b200.model import EncoderUNetModel
    from ddnm_b200.weights import random_state_dict_classifier
    from oracle.gen_classifier_golden import shape
    _, cfg, B, seed, _ = CLASSIFIERS[key]
    m = EncoderUNetModel(**cfg.kwargs())
    m.load_state_dict(random_state_dict_classifier(shape(cfg), 1234))
    x = torch.randn(B, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(seed))
    logits = m(x.to(dev), torch.from_numpy(gold[key + "_t"]).to(dev))
    assert_close(logits, gold[key + "_logits"], what=f"{key} logits vs reference")


@pytest.mark.gpu
def test_guided_64_to_256_pipeline():
    """the published 64x64 base guided by the 64x64 classifier, then the 64 -> 256 upsampler guided by the imagenet_256_cc.yml
    classifier: seeded runs repeat bit for bit, and the 256 x 256 result pools back to the 64 x 64 sample"""
    from ddnm_b200.guidance import make_cond_fn
    from ddnm_b200.model import EncoderUNetModel
    from ddnm_b200.operators import SuperResolution
    from ddnm_b200.superres import sample_then_upsample
    from ddnm_b200.weights import random_state_dict_classifier
    from oracle import operators as O
    from oracle import schedule as SCH
    from oracle.classifier import ClassifierConfig
    from oracle.gen_classifier_golden import shape

    def classifier(cfg, scale):
        c = EncoderUNetModel(**cfg.kwargs())
        c.load_state_dict(random_state_dict_classifier(shape(cfg), 1234))
        return make_cond_fn(c, scale)

    base = _published_model("base64")
    base.load_state_dict(G.state_dict(PUBLISHED["base64"][1]))
    sr = _published_model("up256")
    sr.load_state_dict(G.state_dict(PUBLISHED["up256"][1]))
    cls_fn = classifier(CLASSIFIERS["cls64"][1], 1.0)
    sr_cls_fn = classifier(ClassifierConfig.imagenet_256(), 1.0)
    g = torch.Generator().manual_seed(29)
    x_orig = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
    oop = O.SuperResolution.make(3, 64, 4)
    A = SuperResolution(3, 64, 4, dev, artefacts=(oop.U_small, oop.singulars_small, oop.V_small))
    y = A.A(x_orig.to(dev))
    x_T, x_T_sr = torch.randn(2, 3, 64, 64, generator=g).to(dev), torch.randn(2, 3, 256, 256, generator=g).to(dev)
    betas = SCH.linear_betas().to(dev)
    run = lambda: sample_then_upsample(x_T, base, betas, 0.85, A, y, sr, x_T_sr, config=sampler_config(3, 1, 1),  # noqa: E731
                                       cls_fn=cls_fn, sr_cls_fn=sr_cls_fn, seed=11)
    lo, hi = run()
    lo2, hi2 = run()
    assert lo.shape == (2, 3, 64, 64) and hi.shape == (2, 3, 256, 256)
    assert torch.isfinite(hi).all()
    assert torch.equal(lo, lo2) and torch.equal(hi, hi2)
    P = SuperResolution(3, 256, 4, dev)
    assert_close(P.A(hi), P.A(lo.repeat_interleave(4, dim=2).repeat_interleave(4, dim=3)), 1e-3, 1e-4,
                 "4x4 average pool of the upsampled image vs the base sample")
