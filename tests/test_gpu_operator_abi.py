"""The operator C ABI below the Python shims: the refusals ddnm_operator_create and the Lambda entries return themselves (the
shims raise some of them before the library sees the call), and scratch reuse across batch sizes on one handle."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import schedule as SCH
from oracle import unet_simple as U

from helpers import engine_op, model_config, oracle_ops, sampler_config

dev = "cuda"
DIM = 32
SEED = 0x5EED


def _create(kind, channels=3, img_dim=DIM, ratio=0, **arrays):
    """ddnm_operator_create on a raw descriptor: (return code, handle, last error)."""
    from ddnm_b200 import _lib
    d = _lib.OperatorDesc()
    d.kind, d.channels, d.img_dim, d.ratio = kind, channels, img_dim, ratio
    for name, arr in arrays.items():
        setattr(d, name, arr.ctypes.data)
    h = C.c_void_p()
    rc = _lib.lib().ddnm_operator_create(C.byref(d), C.byref(h))
    return rc, h, _lib.lib().ddnm_last_error().decode()


def _sr_basis(r):
    return dict(v_small=np.eye(r * r, dtype=np.float32), u_small=np.ones((1, 1), np.float32), singulars=np.ones(1, np.float32))


# these refusals happen before any device memory is touched, so they also run without a GPU
@pytest.mark.parametrize("case", [
    ("unknown kind", dict(kind=42), "unknown operator kind"),
    ("sr ratio", dict(kind=0, ratio=3, **_sr_basis(3)), "img_dim % ratio"),
    ("wh not a power of two", dict(kind=3, img_dim=48, ratio=4, perm=np.arange(48 * 48, dtype=np.int64)),
     "WalshHadamardCS: img_dim must be a power of two"),
    ("wh perm", dict(kind=3, ratio=4, perm=np.r_[0, np.arange(DIM * DIM - 1)].astype(np.int64)), "perm is not a permutation"),
    ("general channels", dict(kind=9, channels=3, img_dim=64, ratio=8, v_small=np.eye(64, dtype=np.float32),
                              u_small=np.eye(8, dtype=np.float32), singulars=np.ones(8, np.float32)), "GeneralA: pass channels = 1"),
], ids=lambda c: c[0])
def test_create_refuses_a_malformed_descriptor(case):
    _, kw, text = case
    rc, h, err = _create(**kw)
    assert rc != 0 and not h.value
    assert text in err, err


@pytest.mark.gpu
@pytest.mark.parametrize("name,cls", [("bicubic", "SRConv"), ("deblur2d", "Deblurring2D"), ("cs", "CS"), ("general", "GeneralA")])
def test_lambda_entries_refuse_where_the_reference_defines_none(gold, name, cls):
    from ddnm_b200 import _lib
    op = _builders(gold)[name]()
    v = torch.randn(2, op.x_dim, device=dev)
    out = torch.empty_like(v)
    L = _lib.lib()
    rc = L.ddnm_operator_lambda(op._h, _lib.ptr(v), 2, 0.9, 0.1, 0.3, 0.85, _lib.ptr(out), _lib.cur_stream())
    err = L.ddnm_last_error().decode()
    assert rc != 0 and f"{cls} defines no Lambda (" in err and "sigma_y > 0 is unsupported" in err, err
    rc = L.ddnm_operator_lambda_noise(op._h, _lib.ptr(v), _lib.ptr(v), 2, 0.9, 0.1, 0.3, 0.85, _lib.ptr(out), _lib.cur_stream())
    err = L.ddnm_last_error().decode()
    assert rc != 0 and f"{cls} defines no Lambda_noise (" in err, err


def _builders(gold):
    """name -> a function that builds a fresh handle of that operator from fixed artefacts."""
    from ddnm_b200 import operators as E
    ops = oracle_ops(gold["operators"], DIM)
    sr = E.SuperResolution(3, DIM, 16, dev)
    ga = E.GeneralA(torch.randn(64, 3 * DIM * DIM, generator=torch.Generator().manual_seed(3)).to(dev))
    b = {name: (lambda name=name: engine_op(name, ops[name], DIM)) for name in ("wh", "deblur", "bicubic", "deblur2d", "cs")}
    b["sr16"] = lambda: E.SuperResolution(3, DIM, 16, dev, artefacts=(sr.U_small, sr.singulars_small, sr.V_small))
    b["general"] = lambda: E.GeneralA(None, artefacts=(ga._U, ga._singulars, ga._V))
    return b


def _engine_model():
    from ddnm_b200.model import Model
    cfg = U.SimpleUNetConfig.tiny()
    m = Model(model_config(cfg))
    m.load_state_dict(U.init_state_dict(cfg, 1234))
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("name,has_lambda", [("wh", True), ("deblur", True), ("sr16", True), ("bicubic", False), ("cs", False),
                                             ("general", False)])
def test_scratch_grown_on_one_handle_equals_a_fresh_handle(gold, monkeypatch, name, has_lambda):
    from ddnm_b200 import sampler as ES
    monkeypatch.setattr(ES, "time_pairs", lambda *a, **k: [(500, 400)])
    make = _builders(gold)[name]
    m = _engine_model()
    betas = SCH.linear_betas().to(dev)
    conf = sampler_config(1000, 1, 1)
    g = torch.Generator().manual_seed(17)
    x, x_T, v, e = (torch.randn(4, 3, DIM, DIM, generator=g).to(dev) for _ in range(4))
    tape = torch.randn(1, 4, 3, DIM, DIM, generator=g).to(dev)

    def run(op, B):
        y = op.A(x[:B])
        out = [op.project(x_T[:B], y)]
        if has_lambda:
            out.append(op.Lambda_noise(v[:B].reshape(B, -1), 0.9, 0.1, 0.3, 0.85, e[:B].reshape(B, -1)))
        for kw in (dict(noise=tape[:, :B]), dict(seed=SEED)):
            if has_lambda:
                xs, x0s = ES.ddnm_plus_diffusion(x_T[:B], m, betas, 0.85, op, y, 0.1, config=conf, **kw)
            else:
                xs, x0s = ES.ddnm_diffusion(x_T[:B], m, betas, 0.85, op, y, config=conf, **kw)
            out += [xs[0], x0s[0]]
        return [t.cpu() for t in out]

    grown = make()
    run(grown, 1)
    a, b = run(grown, 4), run(make(), 4)
    for i, (p, q) in enumerate(zip(a, b)):
        assert torch.equal(p, q), f"{name}: output {i} of a handle grown from B = 1 differs from a fresh one"
