"""Exact Groth16 proofs from discrete logs (TEST INFRASTRUCTURE ONLY).

When every point of a proving key is generated as in `Net.generate_g1/g2(seed, n)` (P_i = k_i G, tests/dlog_oracle.py),
each proof element is e G for an exponent e made of integer dot products.  With the formulas of csrc/prove.cu:

    e_A  = alpha + aq_0 + sum_{i>=1} aq_i z_i + r delta_1
    e_B  = beta_2 + b2_0 + sum_{i>=1} b2_i z_i + s delta_2
    e_B1 = beta_1 + b1_0 + sum_{i>=1} b1_i z_i + s delta_1
    e_C  = sum_j l_j z_{n_inputs + j} + sum_j hq_j h_j + s e_A + r e_B1 - r s delta_1

No curve MSM runs at any size: the dot products are exact integer arithmetic (dlog_oracle.exponent), and the expected
128 bytes cost three scalar multiplications in oracle/bn254.py.  Rows zeroed to infinity have log 0.

A key is described by `KeySpec`: the seeds of the five query vectors and of the vk points (alpha_1, beta_1, delta_1 from
one G1 seed; beta_2, delta_2 from one G2 seed), the shape, and the rows set to infinity."""
from __future__ import annotations

import os
from dataclasses import dataclass, field

import numpy as np

from oracle import bn254 as o, layout

import dlog_oracle as dl

QUERIES = ("a", "b1", "b2", "l", "h")
G2_QUERIES = ("b2",)


@dataclass
class KeySpec:
    m: int
    n_vars: int
    n_inputs: int
    seed: int                                         # query k uses seed + index of k in QUERIES; vk1 seed + 5, vk2 seed + 6
    inf: dict = field(default_factory=dict)           # query name -> row indices at infinity

    def seed_of(self, name: str) -> int:
        return self.seed + (QUERIES + ("vk1", "vk2")).index(name)

    def length(self, name: str) -> int:
        return {"a": self.n_vars, "b1": self.n_vars, "b2": self.n_vars, "l": self.n_vars - self.n_inputs, "h": self.m,
                "vk1": 3, "vk2": 2}[name]

    def inf_rows(self, name: str) -> np.ndarray:
        rows = np.asarray(self.inf.get(name, ()), dtype=np.int64).reshape(-1)
        assert rows.size == 0 or (rows.min() >= 0 and rows.max() < self.length(name)), name
        return rows

    def logs(self, name: str) -> np.ndarray:
        """discrete logs of query `name` (uint64), 0 on the rows at infinity"""
        k = dl.base_logs(self.seed_of(name), self.length(name))
        k[self.inf_rows(name)] = 0
        return k

    def vk_logs(self):
        """(alpha_1, beta_1, delta_1), (beta_2, delta_2) as Python ints"""
        return [int(v) for v in self.logs("vk1")], [int(v) for v in self.logs("vk2")]

    # -- the same key as points --------------------------------------------------------------------------------------
    def host_points(self, cref) -> dict:
        """the key as host arrays from the CPU twin's generator (same points as Net.generate_*)"""
        out = {}
        for name in QUERIES + ("vk1", "vk2"):
            gen = cref.g2_generate if name in G2_QUERIES + ("vk2",) else cref.g1_generate
            arr = gen(self.seed_of(name), self.length(name))
            arr[self.inf_rows(name)] = 0
            out[name] = arr
        return out

    def device_points(self, net) -> dict:
        """the key as CUDA int64 tensors made by Net.generate_g1/g2; vk1 / vk2 come back as host arrays"""
        import torch
        out = {}
        for name in QUERIES:
            n = self.length(name)
            if n == 0:
                out[name] = torch.empty((0, 16 if name in G2_QUERIES else 8), dtype=torch.int64, device=net._dev())
                continue
            t = net.generate_g2(self.seed_of(name), n) if name in G2_QUERIES else net.generate_g1(self.seed_of(name), n)
            rows = self.inf_rows(name)
            if rows.size:
                t[torch.from_numpy(rows).to(t.device)] = 0
            out[name] = t
        out["vk1"] = net.generate_g1(self.seed_of("vk1"), 3).cpu().numpy().view(np.uint64)
        out["vk2"] = net.generate_g2(self.seed_of("vk2"), 2).cpu().numpy().view(np.uint64)
        return out


def vk_array(pts: dict) -> np.ndarray:
    """the 56 vk limbs as b200zk_pk_upload and orc_groth16_prove take them"""
    return np.concatenate([np.asarray(pts["vk1"], dtype=np.uint64).reshape(-1), np.asarray(pts["vk2"], dtype=np.uint64).reshape(-1)])


@dataclass
class Exponents:
    """the parts of e_A, e_B, e_B1, e_C that do not depend on (r, s)"""
    a: int            # alpha + aq_0 + sum aq_i z_i
    b: int            # beta_2 + b2_0 + sum b2_i z_i
    b1: int           # beta_1 + b1_0 + sum b1_i z_i
    lh: int           # sum l_j z_{n_inputs + j} + sum hq_j h_j
    delta1: int
    delta2: int


def exponents(spec: KeySpec, z, h) -> Exponents:
    """z: (n_vars, 4) and h: (m, 4) Montgomery limbs"""
    z = np.ascontiguousarray(z, dtype=np.uint64).reshape(-1, 4)
    h = np.ascontiguousarray(h, dtype=np.uint64).reshape(-1, 4)
    assert z.shape[0] == spec.n_vars and h.shape[0] == spec.m
    (alpha, beta1, delta1), (beta2, delta2) = spec.vk_logs()
    R = o.R

    def dot(name, sc):
        return dl.exponent(spec.logs(name)[1:] if name in ("a", "b1", "b2") else spec.logs(name), sc)

    def first(name):
        return int(spec.logs(name)[0])

    zr = z[1:]
    return Exponents(a=(alpha + first("a") + dot("a", zr)) % R, b=(beta2 + first("b2") + dot("b2", zr)) % R,
                     b1=(beta1 + first("b1") + dot("b1", zr)) % R,
                     lh=(dot("l", z[spec.n_inputs:]) + dot("h", h)) % R, delta1=delta1 % R, delta2=delta2 % R)


def proof_exponents(e: Exponents, r: int, s: int):
    """(e_A, e_B, e_C) for canonical r, s"""
    R = o.R
    eA = (e.a + r * e.delta1) % R
    eB = (e.b + s * e.delta2) % R
    eB1 = (e.b1 + s * e.delta1) % R
    eC = (e.lh + s * eA + r * eB1 - r * s % R * e.delta1) % R
    return eA, eB, eC


def proof_bytes(e: Exponents, r: int, s: int) -> bytes:
    """o.proof_compress(e_A G1, e_B G2, e_C G1), None (flag 0x40) for a zero exponent"""
    eA, eB, eC = proof_exponents(e, r, s)
    mul = lambda curve, gen, k: curve.mul(gen, k) if k else None
    return o.proof_compress(mul(o.G1, o.G1_GEN, eA), mul(o.G2, o.G2_GEN, eB), mul(o.G1, o.G1_GEN, eC))


def expected_proof(spec: KeySpec, z, h, r, s) -> bytes:
    """r, s as Montgomery limbs (4,)"""
    rr, ss = (layout.arr_to_fr(np.asarray(v, dtype=np.uint64).reshape(1, 4))[0] for v in (r, s))
    return proof_bytes(exponents(spec, z, h), rr, ss)


# ---- randomisers designed to put a proof element at infinity ---------------------------------------------------------
def _div(a: int, b: int) -> int:
    assert b % o.R, "no randomiser solves this: the divisor is 0 mod r"
    return (-a) * pow(b, -1, o.R) % o.R


def r_for_a_at_infinity(e: Exponents) -> int:
    """r with e_A = 0 (any s)"""
    return _div(e.a, e.delta1)


def s_for_b_at_infinity(e: Exponents) -> int:
    """s with e_B = 0 (any r)"""
    return _div(e.b, e.delta2)


def r_for_c_at_infinity(e: Exponents) -> int:
    """r with e_C = 0 at s = 0: e_C = lh + r e_B1"""
    return _div(e.lh, e.b1)


def designed_cases(e: Exponents, s_other: int = 0x5EED) -> dict:
    """name -> (r, s) canonical, and the element each puts at infinity"""
    return {"A_inf": (r_for_a_at_infinity(e), s_other), "B_inf": (0x1234, s_for_b_at_infinity(e)),
            "C_inf_s0": (r_for_c_at_infinity(e), 0)}


# ---- witnesses and h ---------------------------------------------------------------------------------------------------
ONE = layout.fr_to_arr([1])[0]


def sha256_like_witness(n: int, seed: int, random_rows: int = 0) -> np.ndarray:
    """z[0] = 1, then 99.99 % of the entries 0 or 1 (the giant-bucket case of a real sha256 witness) and a few random"""
    rng = np.random.default_rng(seed)
    z = np.zeros((n, 4), dtype=np.uint64)
    z[rng.random(n) < 0.5] = ONE
    k = random_rows or max(1, n // 10000)
    idx = rng.choice(n, size=min(k, n), replace=False)
    z[idx] = layout.fr_to_arr([int.from_bytes(rng.bytes(32), "little") for _ in idx])
    z[0] = ONE
    return z


def expected_h(cref, a, b, c) -> np.ndarray:
    return cref.h_circom(a, b, c, nthreads=os.cpu_count() or 0)
