"""numpy restatement of the library's seeded Gaussian draws (ddnm_b200/csrc/noise.cuh, include/ddnm_b200.h "Seeded noise").

One value is a pure function of (seed, tag, draw, global image row, element index):
  Philox4x32-10 (Random123 constants), key = (seed low 32 bits, seed high 32 bits), counter = (q, draw, row, tag) with
  q = element index inside one image // 4; the four outputs x0..x3 give elements 4q .. 4q+3;
  u = ((x >> 9) + 0.5) * 2^-23 in fp32; Box-Muller on (x0, x1) and (x2, x3):
  r = sqrt(-2 log u_a), values r * cos(2 pi u_b), r * sin(2 pi u_b).
The transcendental functions are evaluated in float64 from the fp32 uniforms and rounded once, so this is the value the
fp32 library functions approximate.
"""
import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF

TAG_LOOP, TAG_XT, TAG_Y, TAG_HQ, TAG_DEQUANT = 0, 1, 2, 3, 4


def philox4x32_10(counter, key):
    """counter: four arrays (or ints) of 32-bit words, key: two 32-bit ints -> four uint64 arrays holding 32-bit words."""
    c = [np.asarray(v, dtype=np.uint64) & np.uint64(MASK) for v in counter]
    c = list(np.broadcast_arrays(*c))
    k0, k1 = int(key[0]) & MASK, int(key[1]) & MASK
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & np.uint64(MASK),
             (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & np.uint64(MASK)]
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return c


def uniform(x):
    """32 random bits -> fp32 uniform strictly inside (0, 1)."""
    x = np.asarray(x, dtype=np.uint64)
    return ((x >> np.uint64(9)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)


def _box_muller(xa, xb):
    ua, ub = uniform(xa).astype(np.float64), uniform(xb).astype(np.float64)
    r = np.sqrt(-2.0 * np.log(ua))
    return (r * np.cos(2.0 * np.pi * ub)).astype(np.float32), (r * np.sin(2.0 * np.pi * ub)).astype(np.float32)


def normal(seed, tag, draw, row, n):
    """The n values of image ``row`` (global index) of draw ``draw`` of stream ``tag``: float32 (n,)."""
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    x = philox4x32_10((q, draw, row, tag), (seed & MASK, (seed >> 32) & MASK))
    z0, z1 = _box_muller(x[0], x[1])
    z2, z3 = _box_muller(x[2], x[3])
    return np.stack([z0, z1, z2, z3], axis=1).reshape(-1)[:n]


def randn(seed, shape, tag, draw=0, row_offset=0):
    """(B, ...) array: row b holds the draws of global image row ``row_offset + b``."""
    per = int(np.prod(shape[1:], dtype=np.int64))
    return np.stack([normal(seed, tag, draw, row_offset + b, per) for b in range(shape[0])]).reshape(shape)


def tape(seed, n_pairs, shape, row_offset=0, tag=TAG_LOOP):
    """(n_pairs, B, ...) array: the loop's draws, pair k = draw k."""
    return np.stack([randn(seed, shape, tag, k, row_offset) for k in range(n_pairs)])
