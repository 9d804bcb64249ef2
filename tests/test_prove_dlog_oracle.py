"""tests/prove_dlog_oracle.py against the CPU twin: the log-based proof must equal cref.groth16_prove byte for byte
on keys made by cref.g1_generate / g2_generate (the points Net.generate_* makes), for every key shape, row-at-infinity
pattern, mirror_bg1 setting and (r, s) family the GPU prover tests use.  This is what makes their expectations
trustworthy.  Shapes whose MSMs are empty are also checked against the pure-Python prover of oracle/bn254.py."""
import numpy as np
import pytest

from oracle import bn254 as o, layout

import prove_dlog_oracle as po

R = o.R


def _rs_families(e):
    fams = {"0,0": (0, 0), "r,s": (0x1234567, 0x89ABCDEF), "r,0": (0x77, 0), "0,s": (0, 0x99),
            "ord-1,ord-1": (R - 1, R - 1)}
    fams.update(po.designed_cases(e))
    return fams


def _shapes(m):
    out = []
    for nv in (1, 40, m, 3 * m + 7):
        for ni in sorted({1, 2, 17, nv}):
            if ni <= nv:
                out.append((nv, ni))
    return out


def _inf_patterns(spec):
    nv, nl = spec.n_vars, spec.n_vars - spec.n_inputs
    half = list(range(0, nv, 2))
    return {"none": {}, "index0": {"a": [0], "b1": [0], "b2": [0], "l": [0] if nl else [], "h": [0]},
            "half_b": {"b1": half, "b2": half[::-1]}, "all_l": {"l": list(range(nl))}}


def _check(cref, spec, z, h, cases, mirror_values=(False, True)):
    pts = spec.host_points(cref)
    vk = po.vk_array(pts)
    e = po.exponents(spec, z, h)
    for name, (r, s) in cases(e).items():
        rr, ss = layout.fr_to_arr([r])[0], layout.fr_to_arr([s])[0]
        want = po.proof_bytes(e, r, s)
        for mirror in mirror_values:
            got = cref.groth16_prove(pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], vk, spec.n_inputs, z, h, rr, ss,
                                     mirror_bg1=mirror)
            assert got == want, "m=%d n_vars=%d n_inputs=%d inf=%s rs=%s mirror=%s" % (
                spec.m, spec.n_vars, spec.n_inputs, sorted(spec.inf), name, mirror)
    return e


@pytest.mark.parametrize("log_m", [4, 8, 11])
def test_rs_families_and_mirror(cref, log_m):
    m = 1 << log_m
    spec = po.KeySpec(m, m, 2, 0x51000 + log_m)
    z = cref.fr_generate(0x52000 + log_m, m)
    z[0] = po.ONE
    a, b, c = (cref.fr_generate(0x53000 + 10 * log_m + k, m) for k in range(3))
    h = po.expected_h(cref, a, b, c)
    e = _check(cref, spec, z, h, _rs_families)
    # the designed randomisers do what they say: each puts its element at infinity (compressed flag 0x40)
    for name, (r, s) in po.designed_cases(e).items():
        pf = po.proof_bytes(e, r, s)
        off = {"A_inf": 0, "B_inf": 32, "C_inf_s0": 96}[name]
        ln = 64 if name == "B_inf" else 32
        assert pf[off:off + ln] == bytes(ln - 1) + b"\x40", name
    # a sha256-like witness (0 / 1 almost everywhere)
    _check(cref, spec, po.sha256_like_witness(m, log_m, random_rows=3), h, lambda e: {"r,s": (5, 7)})


@pytest.mark.parametrize("log_m", [4, 8, 11])
def test_key_shapes_and_infinity_rows(cref, log_m):
    m = 1 << log_m
    a, b, c = (cref.fr_generate(0x54000 + 10 * log_m + k, m) for k in range(3))
    h = po.expected_h(cref, a, b, c)
    for nv, ni in _shapes(m):
        z = cref.fr_generate(0x55000 + nv, nv)
        z[0] = po.ONE
        base = po.KeySpec(m, nv, ni, 0x56000 + nv + ni)
        for pname, inf in _inf_patterns(base).items():
            spec = po.KeySpec(m, nv, ni, base.seed, inf)
            _check(cref, spec, z, h, lambda e: {"0,0": (0, 0), "r,s": (0xABC, 0xDEF)}, mirror_values=(False,))


def test_empty_msm_shapes_against_the_python_prover(cref):
    """n_vars = 1 (A, B, B1 MSMs empty) and n_inputs = n_vars (L MSM empty), m = 2^4: the pure-Python prover agrees"""
    m = 16
    a, b, c = (cref.fr_generate(0x57000 + k, m) for k in range(3))
    h = po.expected_h(cref, a, b, c)
    for nv, ni in ((1, 1), (5, 5), (40, 1), (40, 40)):
        spec = po.KeySpec(m, nv, ni, 0x58000 + nv + ni, {"a": [0], "b2": [0]})
        pts = spec.host_points(cref)
        z = cref.fr_generate(0x59000 + nv, nv)
        z[0] = po.ONE
        pk = o.ProvingKey()
        pk.n_public = ni - 1
        pk.a_query, pk.b_g1_query, pk.l_query, pk.h_query = (layout.arr_to_g1(pts[k]) for k in ("a", "b1", "l", "h"))
        pk.b_g2_query = layout.arr_to_g2(pts["b2"])
        pk.alpha_g1, pk.beta_g1, pk.delta_g1 = layout.arr_to_g1(pts["vk1"])
        pk.beta_g2, pk.delta_g2 = layout.arr_to_g2(pts["vk2"])
        e = po.exponents(spec, z, h)
        for r, s in ((0, 0), (3, 0), (0, 4), (0x1111, 0x2222)):
            A, B, C = o.groth16_prove(pk, layout.arr_to_fr(z), layout.arr_to_fr(h), r, s)
            assert o.proof_compress(A, B, C) == po.proof_bytes(e, r, s), (nv, ni, r, s)
