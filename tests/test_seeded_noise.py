"""CPU: the seeded-noise contract (oracle/noise.py restates it), its C-ABI surface and the host plumbing around it."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import scipy.stats
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import noise as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0x1234ABCD5678EF01


def _hex(words):
    return " ".join("%08x" % int(w) for w in words)


def test_philox_known_answers():
    """Random123's known-answer rows for Philox4x32-10."""
    assert _hex(N.philox4x32_10((0, 0, 0, 0), (0, 0))) == "6627e8d5 e169c58d bc57ac4c 9b00dbd8"
    assert _hex(N.philox4x32_10((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2)) == "408f276d 41c83b0e a20bc7c6 6d5451fd"
    assert _hex(N.philox4x32_10((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0))) == \
        "d16cfe09 94fdcceb 5001e420 24126ea1"


def test_uniform_is_strictly_inside_the_unit_interval():
    lo, hi = N.uniform(0), N.uniform(0xFFFFFFFF)
    assert lo.dtype == np.float32 and 0.0 < lo < hi < 1.0
    assert float(lo) == 2.0 ** -24 and float(hi) == 1.0 - 2.0 ** -24          # both exact in fp32


def check_standard_normal(z):
    z = np.asarray(z, dtype=np.float64).reshape(-1)
    assert np.isfinite(z).all()
    assert abs(z.mean()) < 5e-3 and abs(z.var() - 1.0) < 5e-3
    assert scipy.stats.kstest(z, "norm").pvalue > 1e-3


def test_oracle_normals_are_standard_and_streams_are_independent():
    n = 1 << 20
    base = N.normal(SEED, 0, 0, 0, n)
    check_standard_normal(base)
    others = {"seed": N.normal(SEED + 1, 0, 0, 0, n), "tag": N.normal(SEED, 1, 0, 0, n), "draw": N.normal(SEED, 0, 1, 0, n),
              "row": N.normal(SEED, 0, 0, 1, n), "seed high word": N.normal(SEED ^ (1 << 40), 0, 0, 0, n)}
    for what, z in others.items():
        assert not np.array_equal(z, base), what
        assert abs(np.corrcoef(z.astype(np.float64), base.astype(np.float64))[0, 1]) < 0.01, what


def test_rows_depend_on_the_global_index_only():
    shape = (3, 8, 8)
    whole = N.tape(SEED, 3, (8,) + shape)
    part = N.tape(SEED, 3, (4,) + shape, row_offset=4)
    assert np.array_equal(whole[:, 4:], part)
    # an image whose length is not a multiple of 4 takes the leading values of its last quad
    assert np.array_equal(N.normal(SEED, 2, 5, 9, 10), N.normal(SEED, 2, 5, 9, 12)[:10])


SEEDED_SYMBOLS = ["ddnm_noise_fill", "ddnm_sample_range_seeded", "ddnm_sample_seeded", "ddnm_sample_simplified_range_seeded",
                  "ddnm_hq_step_seeded", "ddnm_hq_undo_seeded"]


def test_seeded_entries_are_declared_exported_and_bound():
    from ddnm_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "ddnm_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in SEEDED_SYMBOLS:
        m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\);", hdr)
        assert m, f"{name} not declared"
        assert hasattr(lib, name), f"{name} not exported"
        res, args = _lib._SIGS[name]
        assert res is ctypes.c_int and len(args) == len(m.group(1).split(",")), f"{name}: ctypes arity differs from the header"
        seed_pos = [i for i, a in enumerate(m.group(1).split(",")) if "ddnm_noise_seed" in a]
        assert len(seed_pos) == 1 and args[seed_pos[0]] is ctypes.POINTER(_lib.NoiseSeed), name
    assert re.search(r"typedef\s+struct\s*\{\s*unsigned long long seed;\s*long long row_offset;\s*\}\s*ddnm_noise_seed;", hdr)
    assert ctypes.sizeof(_lib.NoiseSeed) == 16
    # argument checks come back as a status + message, before any device work
    L = _lib.lib()
    assert L.ddnm_noise_fill(None, 0, 0, None, 1, 4, None) != 0 and b"noise" in L.ddnm_last_error()
    bad = _lib.NoiseSeed(1, -1)
    buf = (ctypes.c_float * 4)()
    assert L.ddnm_noise_fill(ctypes.byref(bad), 0, 0, ctypes.cast(buf, ctypes.c_void_p), 1, 4, None) != 0
    assert b"row" in L.ddnm_last_error()


def test_seed_and_tape_together_are_rejected():
    from ddnm_b200 import hq, runner, sampler
    x, nz = torch.zeros(1, 3, 8, 8), torch.zeros(2, 1, 3, 8, 8)
    with pytest.raises(ValueError, match="seed"):
        sampler.ddnm_diffusion(x, None, None, 0.85, None, None, noise=nz, seed=1)
    with pytest.raises(ValueError, match="seed"):
        sampler.ddnm_plus_diffusion(x, None, None, 0.85, None, None, 0.1, noise=nz, seed=1)
    with pytest.raises(ValueError, match="seed"):
        sampler.sample_device(x, None, None, 0.85, None, None, 0.0, False, None, noise=nz, seed=1)
    with pytest.raises(ValueError, match="seed"):
        sampler.simplified_ddnm_plus(x, None, None, 0.85, None, None, 0.1, noise=nz, seed=1)
    with pytest.raises(ValueError, match="seed"):
        hq.restore(None, x, [0], noise=nz, seed=1)
    with pytest.raises(ValueError, match="row_offset"):
        sampler.ddnm_diffusion(x, None, None, 0.85, None, None, row_offset=4)
    with pytest.raises(ValueError):
        sampler.ddnm_diffusion(x, None, None, 0.85, None, None, seed=-1)
    assert "seed" in runner.restore_batch.__code__.co_varnames


# ---------------------------------------------------------------------------------------------------- sharding (gloo, 2 ranks)
def _fake_seeded_sampler(x, y, seed, row_offset=0):
    # any row-independent map of (x, y, the row's own draws) stands in for the per-image trajectory
    acc = x.clone()
    nz = torch.from_numpy(N.tape(seed, 4, tuple(x.shape), row_offset=row_offset))
    for k in range(nz.shape[0]):
        acc = acc * 0.9 + nz[k] * 0.1 + y.mean(dim=1).reshape(-1, 1, 1, 1)
    return acc, acc * 2


def _worker(rank, world, port, B, q):
    sys.path.insert(0, ROOT)
    from ddnm_b200.parallel import sharded_sample_seeded
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 3, 8, 8, generator=g)
    y = torch.randn(B, 12, generator=g)
    a, b = sharded_sample_seeded(_fake_seeded_sampler, x, y, SEED)
    ra, rb = _fake_seeded_sampler(x, y, SEED)
    q.put((rank, torch.equal(a, ra) and torch.equal(b, rb), tuple(a.shape)))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("B,port", [(8, 29551), (7, 29552)], ids=["even", "ragged"])
def test_sharded_seeded_equals_unsharded(B, port):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_worker, args=(r, world, port, B, q)) for r in range(world)]
    [p.start() for p in ps]
    res = [q.get(timeout=120) for _ in range(world)]
    [p.join(timeout=60) for p in ps]
    assert all(p.exitcode == 0 for p in ps)
    assert all(ok for _, ok, _ in res), res
    assert all(shape[0] == B for _, _, shape in res)


def test_sharded_seeded_single_rank_passthrough():
    from ddnm_b200.parallel import sharded_sample_seeded
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(3, 3, 8, 8, generator=g), torch.randn(3, 12, generator=g)
    a, b = sharded_sample_seeded(_fake_seeded_sampler, x, y, SEED)
    ra, rb = _fake_seeded_sampler(x, y, SEED)
    assert torch.equal(a, ra) and torch.equal(b, rb)


def test_noise_bench_fails_without_a_gpu_and_parses_arguments():
    import subprocess
    tool = os.path.join(ROOT, "tools", "noise_bench.py")
    r = subprocess.run([sys.executable, tool, "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--repeats" in r.stdout
    if not torch.cuda.is_available():
        r = subprocess.run([sys.executable, tool, "--steps", "2"], capture_output=True, text=True)
        assert r.returncode != 0 and "CUDA" in (r.stderr + r.stdout)
