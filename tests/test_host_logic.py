"""CPU: host-side logic of the product package and the C-ABI surface (no GPU compute)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import schedule as OS
from oracle import unet_simple as U

from helpers import model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_schedule_matches_oracle_and_reference_counts():
    from ddnm_b200 import schedule as ES
    for T, tl, tr in ((20, 1, 1), (100, 1, 1), (100, 3, 3), (100, 2, 2), (250, 1, 1), (10, 3, 2), (7, 2, 3)):
        assert ES.get_schedule_jump(T, tl, tr) == OS.jump_schedule(T, tl, tr)
        assert ES.time_pairs(1000, T, tl, tr) == OS.time_pairs(1000, T, tl, tr)
    # UNet evaluations per image measured on the reference (SURVEY.md section 3.2)
    pairs = ES.time_pairs(1000, 100, 3, 3)
    assert len(pairs) == 496 and sum(1 for i, j in pairs if j < i) == 298
    assert len(ES.time_pairs(1000, 100, 1, 1)) == 100
    pairs = ES.time_pairs(1000, 100, 2, 2)
    assert sum(1 for i, j in pairs if j < i) == 198 and sum(1 for i, j in pairs if j > i) == 98
    assert ES.time_pairs(1000, 20, 1, 1)[-1] == (0, -1)


def test_alpha_bar_table_is_compute_alpha():
    from ddnm_b200 import schedule as ES
    b = OS.linear_betas()
    tab = ES.alpha_bar_table(b)
    assert torch.equal(tab, OS.alpha_bar_table(b))
    # compute_alpha(beta, t) of svd_ddnm.py:10-13
    for t in (-1, 0, 17, 999):
        beta = torch.cat([torch.zeros(1), b], dim=0)
        a = (1 - beta).cumprod(dim=0).index_select(0, torch.tensor([t]) + 1)
        assert tab[t + 1] == a[0]
    assert tab[0] == 1.0


def test_random_state_dict_equals_oracle_init():
    from ddnm_b200.weights import random_state_dict
    cfg = U.SimpleUNetConfig.tiny()
    a, b = U.init_state_dict(cfg, 1234), random_state_dict(model_config(cfg), 1234)
    assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)


def test_shard_rows_partition():
    from ddnm_b200.parallel import shard_rows
    for n in (1, 7, 16, 64, 128, 129):
        for w in (1, 2, 3, 4, 8):
            spans = [shard_rows(n, r, w) for r in range(w)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(spans[i][1] == spans[i + 1][0] for i in range(w - 1))
            sizes = [h - l for l, h in spans]
            assert max(sizes) - min(sizes) <= 1


def _declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "ddnm_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(ddnm_[a-z_0-9A-Z]+)\s*\(", hdr)))


def test_library_loads_and_exports_every_declared_symbol():
    from ddnm_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "build the library first: python -c 'import __graft_entry__ as g; g.build()'"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    declared = _declared_symbols()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/ddnm_b200.h but not exported"
    # and the ctypes table covers the header
    assert set(declared) == set(_lib.EXPORTS)
    assert _lib.lib().ddnm_version() >= 100


def _ctype_of(decl):
    """ctypes type the binding should use for one C parameter declaration of the header"""
    t = re.sub(r"\bconst\b", "", decl).strip()
    t = re.sub(r"\s+\w+$", "", t) if not t.endswith("*") else t   # drop the parameter name
    t = re.sub(r"\s+", " ", t).replace(" *", "*").strip()
    scalar = {"int": ctypes.c_int, "long long": ctypes.c_longlong, "float": ctypes.c_float, "double": ctypes.c_double,
              "unsigned": ctypes.c_uint, "void*": ctypes.c_void_p, "char*": ctypes.c_char_p}
    if t in scalar:
        return scalar[t]
    if t in ("double*", "int*", "long long*", "float*"):
        return ("ptr", t[:-1])   # an out-parameter the binding types, or a device buffer passed as void*
    return None


def test_new_op_entry_signatures_match_the_header():
    """the ctypes argument lists of the op-level test entries agree with their prototypes, parameter by parameter"""
    from ddnm_b200 import _lib
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ddnm_b200.h")).read(), flags=re.S)
    for name in ("ddnm_conv_tc_ex", "ddnm_gemm_tc", "ddnm_conv_tc"):
        params = re.search(name + r"\s*\(([^)]*)\)", hdr).group(1).split(",")
        res, args = _lib._SIGS[name]
        assert res is ctypes.c_int and len(args) == len(params), name
        for decl, got in zip(params, args):
            want = _ctype_of(decl)
            if isinstance(want, tuple):
                base = {"double": ctypes.c_double, "int": ctypes.c_int, "long long": ctypes.c_longlong, "float": ctypes.c_float}[want[1]]
                assert got in (ctypes.c_void_p, ctypes.POINTER(base)), f"{name}: {decl.strip()} bound as {got}"
            else:
                assert want is not None and got is want, f"{name}: {decl.strip()} bound as {got}"


def test_fails_loudly_without_gpu_or_library(monkeypatch, tmp_path):
    from ddnm_b200 import _lib
    from ddnm_b200.model import Model
    if not torch.cuda.is_available():
        cfg = U.SimpleUNetConfig.tiny()
        m = Model(model_config(cfg))
        m.load_state_dict(U.init_state_dict(cfg, 1234))
        with pytest.raises((_lib.DDNMError, AssertionError)):
            m(torch.zeros(1, 3, 32, 32), torch.zeros(1))
        with pytest.raises(_lib.DDNMError):
            m.engine(1)                      # no CUDA device -> error status from the C ABI, never a CPU fallback
    # a missing shared library is an error at import-of-use time
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.DDNMError):
        _lib.lib()


def test_product_package_does_not_import_oracle():
    pkg = os.path.join(ROOT, "ddnm_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), f"{fn} imports the oracle"


def test_operator_constructor_artefacts_match_oracle():
    """The shims' init-time arithmetic (host torch) equals the oracle's / reference's constructors."""
    from oracle import operators as O
    A = torch.Tensor([[1 / 16] * 16])
    U_, S_, V_ = torch.svd(A, some=False)
    o = O.SuperResolution.make(3, 32, 4)
    assert torch.equal(o.V_small, V_) and torch.equal(o.singulars_small, S_)
    k = O.SRConv.bicubic_kernel(4)
    assert abs(k.sum().item() - 1) < 1e-6 and k.numel() == 16
