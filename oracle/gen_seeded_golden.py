"""tests/golden/seeded_tiny.npz: the oracle DDNM and DDNM+ samplers driven by the seeded generator of oracle/noise.py.

Inputs (x_T, y, betas, operator artefacts) are those of the existing sampler_tiny / operators fixtures and the tiny denoiser
with init seed 1234; only the noise tape differs: pair k of image row b uses draw k of stream 0 of ``SEED``.  Runs on the CPU:
    python -m oracle.gen_seeded_golden
"""
import os
import sys

import numpy as np
import torch

from oracle import noise as N
from oracle import sampler as S
from oracle import schedule as SCH
from oracle import unet_simple as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SEED = 0x5EED0123456789AB
CASES = [("sr4", 10, 3, 2, 0.0), ("inpaint", 10, 2, 2, 0.1)]   # operator, T_sampling, travel_length, travel_repeat, sigma_y


def load(name):
    """A golden file, re-joined from its .partN.npz pieces when it was split."""
    out = dict(np.load(os.path.join(GOLD, name + ".npz")))
    i = 1
    while os.path.exists(os.path.join(GOLD, f"{name}.part{i}.npz")):
        out.update(np.load(os.path.join(GOLD, f"{name}.part{i}.npz")))
        i += 1
    return out


def run_case(g, ops, case, seed=SEED):
    name, T, tl, tr, sy = case
    cfg = U.SimpleUNetConfig.tiny()
    sd = U.init_state_dict(cfg, 1234)
    key = f"{name}_T{T}_l{tl}_r{tr}_s{sy}"
    x_T, y = torch.from_numpy(g["x_T"]), torch.from_numpy(g[key + "_y"])
    npairs = len(SCH.time_pairs(1000, T, tl, tr))
    tape = [torch.from_numpy(t) for t in N.tape(seed, npairs, tuple(x_T.shape))]
    with torch.no_grad():
        return key, S.ddnm_sample(x_T, lambda a, b: U.forward(sd, a, b, cfg), torch.from_numpy(g["betas"]), 0.85, ops[name], y, tape,
                                  t_sampling=T, travel_length=tl, travel_repeat=tr, sigma_y=sy)


def main():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from helpers import oracle_ops
    g, ops = load("sampler_tiny"), oracle_ops(load("operators"), 32)
    out = {"seed": np.array([SEED], dtype=np.uint64)}
    for case in CASES:
        key, (x0, x0p) = run_case(g, ops, case)
        out[key + "_x0"], out[key + "_x0pred"] = x0.numpy(), x0p.numpy()
        print(key, float(x0.abs().max()))
    np.savez_compressed(os.path.join(GOLD, "seeded_tiny.npz"), **out)


if __name__ == "__main__":
    main()
