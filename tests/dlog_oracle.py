"""Exact MSM answers from bases with known discrete logs (TEST INFRASTRUCTURE ONLY).

`Net.generate_g1/g2(seed, n)` and `cref.g1/g2_generate(seed, n)` both make P_i = k_i G with
k_i = splitmix64(seed + i) | 1 (csrc/msm.cu, k_generate_points).  For scalars given as Montgomery limbs v_i,

    MSM(P, s) = e G,   e = R^-1 sum_i k_i v_i  (mod r),   R = 2^256,

which is plain integer arithmetic: no curve arithmetic, no bucket, window or reduction code is involved.  The dot
product splits k_i into four and v_i into sixteen 16-bit limbs, so every partial sum stays below 2^32 * n < 2^63 for
n < 2^31, and runs as torch int64 matrix products (no code shared with the library or the CPU twin).  One scalar
multiplication in oracle/bn254.py then gives the expected point.

Also here: a Python restatement of glv_decompose (csrc/glv.cuh) and the scalar families the exact MSM tests use."""
from __future__ import annotations

import os
import re

import numpy as np

from oracle import bn254 as o, layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASK64 = (1 << 64) - 1
RINV = pow(1 << 256, -1, o.R)


# ---- bases with known logs --------------------------------------------------------------------------------------
def splitmix64(x: np.ndarray) -> np.ndarray:
    """splitmix64 finaliser on uint64 arrays (wrapping arithmetic, as in k_generate_points)."""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def base_logs(seed: int, n: int, start: int = 0) -> np.ndarray:
    """k_i = splitmix64(seed + i) | 1 for i in [start, start + n): the discrete logs of the generated bases."""
    idx = np.arange(start, start + n, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = np.uint64(seed & MASK64) + idx
    return splitmix64(x) | np.uint64(1)


def _chunks(n: int, step: int = 1 << 20):
    for lo in range(0, n, step):
        yield lo, min(n, lo + step)


def exact_dot(logs, scalars) -> int:
    """sum_i logs[i] * v_i as a Python int; logs: (n,) uint64, scalars: (n, 4) uint64 limbs (any 256-bit values)."""
    import torch
    logs = np.ascontiguousarray(logs, dtype=np.uint64).reshape(-1)
    scalars = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
    n = logs.shape[0]
    assert scalars.shape[0] == n and n < (1 << 31)
    acc = torch.zeros((4, 16), dtype=torch.int64)
    for lo, hi in _chunks(n):
        k16 = torch.from_numpy(logs[lo:hi].view(np.uint16).reshape(-1, 4).astype(np.int64))
        v16 = torch.from_numpy(scalars[lo:hi].view(np.uint16).reshape(-1, 16).astype(np.int64))
        acc += k16.T @ v16                                  # every entry < 2^32 * n < 2^63
    d = acc.numpy()
    return sum(int(d[a, b]) << (16 * (a + b)) for a in range(4) for b in range(16))


def exponent(logs, scalars) -> int:
    """e with MSM(P, s) = e G for bases P_i = logs[i] G and Montgomery scalars."""
    return exact_dot(logs, scalars) % o.R * RINV % o.R


def point_from_exponent(e: int, g2: bool):
    """(affine limbs as in b200zk.h, infinity flag) of e G."""
    e %= o.R
    curve, gen = (o.G2, o.G2_GEN) if g2 else (o.G1, o.G1_GEN)
    pt = curve.mul(gen, e) if e else None
    arr = (layout.g2_to_arr if g2 else layout.g1_to_arr)([pt])[0]
    return arr, pt is None


def expected_msm(seed: int, scalars, g2: bool = False):
    """Expected MSM of the generated bases (seed, n = len(scalars)) with `scalars` (Montgomery limbs)."""
    scalars = np.asarray(scalars, dtype=np.uint64).reshape(-1, 4)
    return point_from_exponent(exponent(base_logs(seed, scalars.shape[0]), scalars), g2)


def expected_from_logs(logs, scalars, g2: bool = False):
    """Expected MSM for bases with designed logs (Python ints, any sign) and Montgomery scalars."""
    vals = layout.arr_to_fr(scalars)
    return point_from_exponent(sum((int(a) % o.R) * v for a, v in zip(logs, vals)), g2)


# ---- GLV split (restatement of csrc/glv.cuh) -------------------------------------------------------------------
def _inc_constants() -> dict:
    """GlvParams as the device code sees them (csrc/bn254_constants.inc), as Python ints."""
    src = open(os.path.join(ROOT, "distributed_groth16_b200", "csrc", "bn254_constants.inc")).read()
    body = src[src.index("struct GlvParams"):]
    body = body[:body.index("\n};")]
    out = {}
    for name, limbs in re.findall(r"uint32_t (\w+)\(int i\) \{\s*constexpr uint32_t t\[\d+\] = \{([^}]*)\}", body):
        vals = [int(v.strip().rstrip("u"), 16) for v in limbs.split(",")]
        out[name] = sum(v << (32 * i) for i, v in enumerate(vals))
    return out


GLV = _inc_constants()
LAMBDA = o.fr_unmont(GLV["lambda_mont"])


def glv_decompose(k: int):
    """(k1, k2) as signed ints with k = k1 + k2 lambda (mod r): the device's rounding, step for step."""
    assert 0 <= k < o.R
    c1 = (k * GLV["g1"] + (1 << 255)) >> 256
    c2 = (k * GLV["g2"] + (1 << 255)) >> 256
    k1 = k - c1 * GLV["a1"] - c2 * GLV["a2"]
    k2 = c1 * GLV["nb1"] - c2 * GLV["b2"]
    return k1, k2


def glv_compose(k1: int, k2: int) -> int:
    return (k1 + k2 * LAMBDA) % o.R


# ---- scalar families -------------------------------------------------------------------------------------------
def repeat_digit(d: int, c: int, bits: int) -> int:
    """d in every c-bit window whose top bit lies below `bits` (the value stays < 2^bits)."""
    v, w = 0, 0
    while c * w + c <= bits:
        v |= d << (c * w)
        w += 1
    return v


# Largest |k1|, |k2| the split produces is about 2^126.1: designed halves up to 125 bits are split back unchanged
GLV_HALF_BITS = 125


def digit_families(c: int, glv: bool) -> dict:
    """name -> list of canonical scalars: the digit patterns B, B + 1 (a negative digit and a carry) and 2^c - 1 (a carry
    through every window) on k itself (plain path) or on both GLV halves, in every sign combination."""
    B = 1 << (c - 1)
    pats = {"digit_B": B, "digit_B+1": B + 1, "digit_all_ones": (1 << c) - 1}
    fams = {}
    for name, d in pats.items():
        if glv:
            h = repeat_digit(d, c, GLV_HALF_BITS)
            fams[name] = [glv_compose(s1 * h, s2 * h) for s1 in (1, -1) for s2 in (1, -1)] + [glv_compose(h, 0), glv_compose(0, h)]
        else:
            fams[name] = [repeat_digit(d, c, 253), repeat_digit(d, c, 254) % o.R]
    fams["edges"] = [o.R - 1, 1 << 253, 1, 0]
    return fams


def glv_designed_halves(extremes=()) -> list:
    """(k1, k2) pairs: zero halves, every sign combination, and the given extreme splits."""
    a, b = (1 << 124) + 12345, (1 << 123) + 678
    pairs = [(0, 0), (a, 0), (-a, 0), (0, b), (0, -b), (a, b), (a, -b), (-a, b), (-a, -b)]
    return pairs + list(extremes)


def glv_extremes(count: int = 1 << 16, seed: int = 5):
    """The k among `count` random scalars whose split has the largest |k1|, and the one with the largest |k2|."""
    rng = np.random.default_rng(seed)
    best1, best2 = (0, 0), (0, 0)
    for _ in range(count):
        k = int.from_bytes(rng.bytes(32), "little") % o.R
        k1, k2 = glv_decompose(k)
        if abs(k1) > best1[0]:
            best1 = (abs(k1), k)
        if abs(k2) > best2[0]:
            best2 = (abs(k2), k)
    return best1[1], best2[1]
