"""Batch-invariant mode (`_EngineModel.batch_invariant`, `ddnm_unet_set_batch_invariant`): with it on, a row's forward, the
classifier's input gradient and a seeded restoration are bit-identical at any engine batch, row position, padding and SM count.
Every equality here is torch.equal.  The ABI / attribute checks run without a GPU."""
import os

import numpy as np
import pytest
import torch

from oracle import classifier as OC
from oracle import operators as O
from oracle import schedule as SCH
from oracle import unet_openai as UO
from oracle import unet_simple as U

from helpers import engine_op, model_config, openai_model_kwargs, sampler_config

dev = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x5EED0123


# ------------------------------------------------------------------------------------------------ CPU
def test_the_c_abi_declares_the_mode_and_the_sm_count_hook():
    from ddnm_b200 import _lib
    with open(os.path.join(ROOT, "include", "ddnm_b200.h")) as f:
        hdr = f.read()
    assert "int ddnm_unet_set_batch_invariant(void* handle, int on);" in hdr
    assert "int ddnm_tc_debug_sm_count(int n);" in hdr
    assert _lib._SIGS["ddnm_unet_set_batch_invariant"][1] == [_lib._P, _lib._I]
    assert _lib._SIGS["ddnm_tc_debug_sm_count"][1] == [_lib._I]


def test_the_attribute_is_off_by_default_and_changing_it_drops_the_engines():
    from ddnm_b200.model import EncoderUNetModel, Model, SuperResModel, UNetModel, _EngineModel
    for cls in (Model, UNetModel, SuperResModel, EncoderUNetModel):
        assert issubclass(cls, _EngineModel)
    m = object.__new__(Model)
    dropped = []
    m._destroy = lambda: dropped.append(1)
    assert m.batch_invariant is False
    m.batch_invariant = True
    assert m.batch_invariant is True and dropped == [1]
    m.batch_invariant = True          # unchanged: the engines stay
    assert dropped == [1]
    m.batch_invariant = False
    assert m.batch_invariant is False and dropped == [1, 1]


# ------------------------------------------------------------------------------------------------ GPU
def _lib():
    from ddnm_b200 import _lib as L
    return L.lib()


def _celeba():
    from ddnm_b200.model import Model
    from ddnm_b200.weights import random_state_dict
    mcfg = model_config(U.SimpleUNetConfig.celeba_hq())
    m = Model(mcfg)
    m.load_state_dict(random_state_dict(mcfg, 1234))
    return m


def _inputs(n, res=256, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, res, res, generator=g)
    t = torch.randint(0, 1000, (n,), generator=g).float()
    return x.to(dev), t.to(dev)


def _splitk_layers(prof):
    return sorted(op["name"] for op in prof if op["name"].endswith(".splitk_reduce"))


@pytest.fixture
def sm_count():
    yield lambda n: _lib().ddnm_tc_debug_sm_count(n)
    _lib().ddnm_tc_debug_sm_count(0)


@pytest.mark.gpu
def test_celeba_rows_do_not_depend_on_batch_position_padding_or_sm_count(sm_count):
    m = _celeba()
    x, t = _inputs(16)
    # the default policy really differs between the batches compared below, so equality under the mode is not for free
    assert _splitk_layers(m.profile(x[:1], t[:1])) != _splitk_layers(m.profile(x, t))
    m.batch_invariant = True
    assert not m._engines
    with torch.no_grad():
        one = {i: m(x[i:i + 1], t[i:i + 1]) for i in (0, 7, 15)}        # engine batch 1
        two = m(x[3:5], t[3:5])                                          # engine batch 2
        order = [15, 0, 7, 3, 4]
        five = m(x[order], t[order])                                     # engine batch 5, rows at other positions
        ragged = m(x[[4, 15, 0]], t[[4, 15, 0]])                         # 3 rows padded onto the 5-row engine
        assert sorted(m._engines) == [1, 2, 5]
        full = m(x, t)                                                   # engine batch 16
    for i, o in one.items():
        assert torch.equal(o[0], full[i]), f"row {i}: B = 1 vs B = 16"
    assert torch.equal(two, full[3:5]), "B = 2 vs B = 16"
    assert torch.equal(five, full[order]), "B = 5 (permuted rows) vs B = 16"
    assert torch.equal(ragged, full[[4, 15, 0]]), "ragged batch padded onto a bigger engine"
    for n in (66, 114):
        sm_count(n)
        ms = _celeba()
        ms.batch_invariant = True
        with torch.no_grad():
            assert torch.equal(ms(x, t), full), f"{n} SMs vs the device's count"
        del ms


@pytest.mark.gpu
def test_bn_64_and_128_round_every_element_alike():
    """Forcing the N tile to 64 or 128 on the celeba shapes under the mode gives the same bits, so BN stays a free launch choice"""
    L = _lib()
    x, t = _inputs(4, seed=5)
    outs = []
    try:
        for bn in (64, 128):
            L.ddnm_tc_debug_force_bn(bn)
            m = _celeba()
            m.batch_invariant = True
            with torch.no_grad():
                outs.append(m(x, t))
            del m
    finally:
        L.ddnm_tc_debug_force_bn(0)
    assert torch.equal(outs[0], outs[1]), f"BN = 64 vs 128: max |diff| {(outs[0] - outs[1]).abs().max().item():.3e}"


def _imagenet(class_cond):
    from ddnm_b200.model import create_model
    from ddnm_b200.weights import random_state_dict_openai
    kw = openai_model_kwargs(UO.OpenAIUNetConfig.imagenet_256())
    kw["class_cond"] = class_cond
    m = create_model(**kw)
    sd = random_state_dict_openai(m, 1234)
    if class_cond:   # the random init draws no label embedding (nn.Embedding's N(0, 1), unet.py:478-479)
        sd["label_emb.weight"] = torch.randn(1000, 4 * m.model_channels, generator=torch.Generator().manual_seed(5))
    m.load_state_dict(sd)
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("class_cond", [False, True])
def test_imagenet_unet_rows_match_at_batch_1_2_4(class_cond):
    m = _imagenet(class_cond)
    m.batch_invariant = True
    x, t = _inputs(4, seed=7)
    y = torch.tensor([1, 500, 999, 3], device=dev) if class_cond else None
    sel = lambda idx: (x[idx], t[idx]) + ((y[idx],) if class_cond else ())   # noqa: E731
    with torch.no_grad():
        one = m(*sel([2]))
        two = m(*sel([3, 0]))
        four = m(*sel([0, 1, 2, 3]))
    assert torch.equal(one[0], four[2]), "B = 1 vs B = 4"
    assert torch.equal(two, four[[3, 0]]), "B = 2 vs B = 4"


@pytest.mark.gpu
def test_superres_rows_match_at_batch_1_and_3():
    """the published 64 -> 256 upsampler (SuperResModel, full width) with its low_res input"""
    from test_zoo import G, PUBLISHED, _published_model
    m = _published_model("up256")
    m.load_state_dict(G.state_dict(PUBLISHED["up256"][1]))
    g = torch.Generator().manual_seed(21)
    x = torch.randn(3, 3, 256, 256, generator=g).to(dev)
    low = (torch.rand(3, 3, 64, 64, generator=g) * 2 - 1).to(dev)
    t = torch.tensor([10.0, 500.0, 999.0], device=dev)
    y = torch.tensor([4, 250, 870], device=dev)
    with torch.no_grad():       # the default policy differs between B = 1 and B = 3 (the engines stage low_res first)
        m(x[1:2], t[1:2], y[1:2], low_res=low[1:2])
        m(x, t, y, low_res=low)
    assert _splitk_layers(m.profile(x[1:2], t[1:2])) != _splitk_layers(m.profile(x, t))
    m.batch_invariant = True
    with torch.no_grad():
        one = m(x[1:2], t[1:2], y[1:2], low_res=low[1:2])
        three = m(x, t, y, low_res=low)
    assert torch.equal(one[0], three[1])


def _classifier():
    from ddnm_b200.model import EncoderUNetModel
    from test_classifier import _sd
    cfg = OC.ClassifierConfig.imagenet_256()
    m = EncoderUNetModel(**cfg.kwargs())
    m.load_state_dict(_sd(cfg))
    return m


@pytest.mark.gpu
def test_classifier_logits_and_gradient_rows_match_at_batch_1_3_8(sm_count):
    m = _classifier()
    m.batch_invariant = True
    x, t = _inputs(8, seed=11)
    y = torch.arange(8, device=dev) * 111
    with torch.no_grad():
        res = {}
        for idx in ([5], [2, 7, 0], list(range(8))):
            res[len(idx)] = (idx, m(x[idx], t[idx]), m.grad(x[idx], t[idx], y[idx], 3.0))
    _, l8, g8 = res[8]
    for b in (1, 3):
        idx, lb, gb = res[b]
        assert torch.equal(lb, l8[idx]), f"logits B = {b} vs 8"
        assert torch.equal(gb, g8[idx]), f"gradient B = {b} vs 8"
    sm_count(66)
    m2 = _classifier()
    m2.batch_invariant = True
    assert torch.equal(m2.grad(x, t, y, 3.0), g8), "gradient at 66 SMs"


# ---- parity with the mode on: the existing fixture comparisons, every engine built in batch-invariant mode
@pytest.fixture
def invariant_by_default(monkeypatch):
    from ddnm_b200.model import _EngineModel
    monkeypatch.setattr(_EngineModel, "_batch_invariant", True)


@pytest.mark.gpu
def test_unet_fixtures_hold_with_the_mode_on(gold, invariant_by_default):
    import test_gpu_parity as P
    P.test_unet_tiny_vs_reference_golden(gold, True)
    P.test_unet_celeba_vs_reference_golden(gold)
    P.test_openai_unet_tiny_vs_reference_golden(gold, True)
    P.test_openai_unet_imagenet_vs_reference_golden(gold)


@pytest.mark.gpu
def test_fullsize_fixture_holds_with_the_mode_on(gold, invariant_by_default, monkeypatch):
    import test_gpu_fullsize as F
    from oracle import fullsize as FS
    monkeypatch.setattr(F, "_ENG", {})
    F.test_fullsize_sampler_vs_reference(gold["fullsize"], FS.FULLSIZE_CASES[0])


@pytest.mark.gpu
def test_classifier_fixtures_hold_with_the_mode_on(invariant_by_default):
    import glob
    import test_classifier as TC
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "classifier.npz")))
    for part in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "classifier.part*.npz"))):
        g.update(np.load(part))
    for key in TC.CASES:
        TC.test_classifier_engine_vs_reference(g, key)


# ---- end to end, seeded, full-size networks
def _sr4():
    return engine_op("sr4", O.SuperResolution.make(3, 256, 4), 256)


@pytest.mark.gpu
@pytest.mark.parametrize("plus", [False, True])
def test_seeded_restoration_is_identical_however_it_is_batched(plus):
    from ddnm_b200.sampler import ddnm_diffusion, ddnm_plus_diffusion
    m = _celeba()
    m.batch_invariant = True
    eop = _sr4()
    g = torch.Generator().manual_seed(2)
    x_T = torch.randn(6, 3, 256, 256, generator=g).to(dev)
    y = eop.A((torch.rand(6, 3, 256, 256, generator=g) * 2 - 1).to(dev))
    conf = sampler_config(4, 2, 2)
    betas = SCH.linear_betas().to(dev)

    def run(lo, hi):
        if plus:
            xs, x0s = ddnm_plus_diffusion(x_T[lo:hi], m, betas, 0.85, eop, y[lo:hi], 0.1, config=conf, seed=SEED, row_offset=lo)
        else:
            xs, x0s = ddnm_diffusion(x_T[lo:hi], m, betas, 0.85, eop, y[lo:hi], config=conf, seed=SEED, row_offset=lo)
        return torch.cat([xs[0], x0s[0]], dim=1)
    singles = torch.cat([run(i, i + 1) for i in range(6)])      # engine batch 1
    split = torch.cat([run(0, 4), run(4, 6)])                    # engines 4 and (padded onto 4) 2
    whole = run(0, 6)                                            # engine batch 6
    assert torch.equal(whole, split), "6 in one call vs 4 + 2"
    assert torch.equal(whole, singles), "6 in one call vs six calls of 1"


@pytest.mark.gpu
def test_seeded_guided_loop_is_identical_however_it_is_batched():
    from ddnm_b200.guidance import make_cond_fn
    from ddnm_b200.sampler import ddnm_diffusion
    unet = _imagenet(True)
    unet.batch_invariant = True
    clf = _classifier()
    clf.batch_invariant = True
    cond = make_cond_fn(clf, 2.0)
    eop = _sr4()
    g = torch.Generator().manual_seed(4)
    x_T = torch.randn(3, 3, 256, 256, generator=g).to(dev)
    y = eop.A((torch.rand(3, 3, 256, 256, generator=g) * 2 - 1).to(dev))
    conf = sampler_config(3, 1, 1)
    betas = SCH.linear_betas().to(dev)

    def run(lo, hi):
        xs, x0s = ddnm_diffusion(x_T[lo:hi], unet, betas, 0.85, eop, y[lo:hi], cls_fn=cond, config=conf, seed=SEED,
                                 row_offset=lo)
        return torch.cat([xs[0], x0s[0]], dim=1)
    one = run(2, 3)
    whole = run(0, 3)
    assert torch.equal(whole[2:3], one)


@pytest.mark.gpu
def test_seeded_simplified_ddnm_plus_is_identical_however_it_is_batched():
    from ddnm_b200.sampler import SimplifiedDegradation, simplified_ddnm_plus
    m = _celeba()
    m.batch_invariant = True
    deg = SimplifiedDegradation("sr_averagepooling", 4, image_size=256)
    g = torch.Generator().manual_seed(6)
    x_T = torch.randn(3, 3, 256, 256, generator=g).to(dev)
    y = deg.A((torch.rand(3, 3, 256, 256, generator=g) * 2 - 1).to(dev))
    conf = sampler_config(4, 2, 2)
    betas = SCH.linear_betas().to(dev)

    def run(lo, hi):
        xs, x0s = simplified_ddnm_plus(x_T[lo:hi], m, betas, 0.85, deg, y[lo:hi], 0.05, config=conf, seed=SEED, row_offset=lo)
        return torch.cat([xs[0], x0s[0]], dim=1)
    one = run(1, 2)
    whole = run(0, 3)
    assert torch.equal(whole[1:2], one)


@pytest.mark.gpu
def test_seeded_hq_restore_row_0_is_identical_alone_and_in_a_batch():
    """hq.restore keys an image's draws by its row within the call (it has no row_offset), so the comparable rows are those that
    keep their index: image 0 restored alone and as row 0 of a batch of 2"""
    from ddnm_b200 import hq as HQ
    m = _imagenet(True)
    m.batch_invariant = True
    g = torch.Generator().manual_seed(8)
    gt = (torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).to(dev)
    kw = dict(deg="sr_averagepooling", scale=4, resize_y=True, timestep_respacing=6,
              schedule_jump_params=dict(t_T=6, n_sample=1, jump_length=2, jump_n_sample=2), seed=SEED)
    one = HQ.restore(m, gt[:1], torch.tensor([950]), **kw)          # engine batch 1 (built first, so nothing rides padded)
    two = HQ.restore(m, gt, torch.tensor([950, 3]), **kw)
    assert two.shape == (2, 3, 256, 256)
    assert torch.equal(one[0], two[0])


@pytest.mark.gpu
def test_seeded_restore_batch_writes_the_same_files_at_batch_size_3_and_1(tmp_path):
    """runner.restore_batch(seed=...): a dataset slice restored as one batch of 3 and as three batches of 1 (idx_so_far = the
    images' dataset index) writes byte-identical PNGs and reports the same PSNR; DDNM+ with a noisy y exercises every seeded draw"""
    from ddnm_b200 import runner as R
    from test_runner_io import _cfg
    m = _celeba()
    m.batch_invariant = True
    eop = _sr4()
    conf = sampler_config(4, 2, 2)
    conf.data = _cfg(True, False, channels=3, size=256).data
    betas = SCH.linear_betas().to(dev)
    x01 = torch.rand(3, 3, 256, 256, generator=torch.Generator().manual_seed(12))
    idx0 = 10

    def run(folder, lo, hi):
        return R.restore_batch(conf, m, eop, "sr_averagepooling", x01[lo:hi], betas, 0.85, sigma_y=0.1, add_noise=True,
                               image_folder=str(folder), idx_so_far=idx0 + lo, seed=SEED)
    singles = [run(tmp_path / "b1", i, i + 1) for i in range(3)]   # engine batch 1 (built first, so nothing rides padded)
    whole = run(tmp_path / "b3", 0, 3)
    assert torch.equal(whole["psnr"], torch.cat([o["psnr"] for o in singles]))
    names = sorted(p.relative_to(tmp_path / "b3") for p in (tmp_path / "b3").rglob("*.png"))
    assert len(names) == 9 and names == sorted(p.relative_to(tmp_path / "b1") for p in (tmp_path / "b1").rglob("*.png"))
    for n in names:
        assert (tmp_path / "b3" / n).read_bytes() == (tmp_path / "b1" / n).read_bytes(), str(n)
