"""The operand corpus of tests/arith_oracle.py holds every branch class it is built for, in both fields, and its branch models
agree with direct arithmetic.  A change to the generator cannot quietly lose a class."""
import collections
import random

import pytest

from oracle import bn254 as o

import arith_oracle as A
import dlog_oracle as dl

P, R, MONT = A.P, A.R, A.MONT


def _classes(name):
    return collections.Counter(c for c, _ in A.corpus()[name])


def _pairs(name):
    return [(c, A.num(r[0:4]), A.num(r[4:8])) for c, r in A.corpus()[name]]


def test_every_op_has_a_unique_code_and_a_corpus():
    """(The record sizes are checked against selftest.cu's own table in tests/test_host_arith.py.)"""
    codes = [op.code for op in A.OPS.values()]
    assert len(set(codes)) == len(codes)
    assert set(A.corpus()) == set(A.OPS)
    for name, op in A.OPS.items():
        assert len(A.corpus()[name]) >= 2, name
    # device-only ops: the root of unity and the four quad_ops entries of each group
    assert sorted(n for n, op in A.OPS.items() if op.device_only) == sorted(
        ["fr_root_of_unity"] + ["%s_quad_%s%s" % (g, s, w) for g in ("g1", "g2") for s in ("add", "dbl") for w in ("", "_fullwarp")])


@pytest.mark.parametrize("g", ["g1", "g2"])
def test_point_views_reject_noncanonical_coordinates(g):
    """The group-law comparison is exact about representation: a coordinate left in [p, 2p) (a skipped final subtraction)
    is congruent to the right one but must not read as correct, in XYZZ and in affine outputs, in every Fq component."""
    G = A.G1 if g == "g1" else A.G2
    pt = G.c.mul(G.gen, 12345)
    z = 7 if g == "g1" else (7, 3)
    good_x, good_a = G.xyzz_w(pt, z), G.aff_w(pt)
    assert G.xyzz_view(good_x) == G.pt_view(pt) == G.aff_view(good_a)
    for ws, view in ((good_x, G.xyzz_view), (good_a, G.aff_view)):
        for k in range(0, len(ws), 4):
            bad = list(ws)
            v = A.num(bad[k:k + 4]) + P
            assert v < MONT
            bad[k:k + 4] = A.words(v)
            assert view(bad)[0] == "noncanonical", k


@pytest.mark.parametrize("f,p", [("fq", P), ("fr", R)])
def test_montgomery_product_classes(f, p):
    """T = (a b + M p) / 2^256 is congruent to a b R^-1, below 2p; the corpus reaches T >= p, results 1, 2, 3 after the
    subtraction and T = p - 1 without it."""
    ri = pow(MONT, -1, p)
    seen = collections.Counter()
    for c, a, b in _pairs(f + "_mul"):
        t = A.mont_pre(a * b, p)
        assert t % p == a * b * ri % p and t < 2 * p
        seen["final_sub"] += t >= p
        for v in (1, 2, 3):
            seen["result_%d_after_sub" % v] += t == p + v
        seen["T_p_minus_1"] += t == p - 1
        if c in ("final_sub",):
            assert t >= p
        if c.startswith("result_"):
            assert t == p + int(c.split("_")[1])
        if c == "T_p_minus_1":
            assert t == p - 1
    assert seen["final_sub"] >= 24
    for v in (1, 2, 3):
        assert seen["result_%d_after_sub" % v] >= 2
    assert seen["T_p_minus_1"] >= 2
    sq = [A.num(r) for c, r in A.corpus()[f + "_sqr"]]
    assert sum(A.mont_pre(a * a, p) >= p for a in sq) >= 8
    # b >= p (the contract inv relies on): T < 2p still
    for c, a, b in _pairs(f + "_mul_any"):
        assert a < p and b < MONT and A.mont_pre(a * b, p) < 2 * p
    assert sum(b >= p for _, _, b in _pairs(f + "_mul_any")) >= 16


@pytest.mark.parametrize("f,p", [("fq", P), ("fr", R)])
def test_redc2_classes(f, p):
    ri = pow(MONT, -1, p)
    cls = collections.Counter()
    for c, r in A.corpus()[f + "_redc2"]:
        t = A.num(r)
        assert t < 2 * p * MONT
        pre = A.mont_pre(t, p)
        assert pre % p == t * ri % p and pre < 3 * p
        cls[pre // p] += 1
    assert cls[0] >= 8 and cls[1] >= 8 and cls[2] >= 8


def test_fq2_mul_classes():
    """c0's t0 reaches [0, p), [p, 2p) and [2p, 3p) before redc<2>'s subtractions; c1's t2 reaches [0, p) and [p, 2p) and
    cannot reach 2p: t2 < 2 p^2, so T < (2 p^2 + 2^256 p) / 2^256 < 1.38 p."""
    assert (2 * P * P + MONT * P) / MONT < 1.38 * P
    c0, c1 = collections.Counter(), collections.Counter()
    pm1 = 0
    for c, r in A.corpus()["fq2_mul"]:
        a0, a1, b0, b1 = (A.num(r[4 * i:4 * i + 4]) for i in range(4))
        t0 = a0 * b0 - a1 * b1 + P * MONT
        t2 = a0 * b1 + a1 * b0
        assert 0 <= t0 < 2 * P * MONT and t2 < 2 * P * MONT
        c0[A.mont_pre(t0, P) // P] += 1
        c1[A.mont_pre(t2, P) // P] += 1
        pm1 += c == "pm1_combo"
    assert c0[0] >= 8 and c0[1] >= 8 and c0[2] >= 8
    assert c1[0] >= 8 and c1[1] >= 8 and c1[2] == 0
    assert pm1 == 16 and _classes("fq2_mul")["zero_coeff"] >= 2


@pytest.mark.parametrize("f,p", [("fq", P), ("fr", R)])
def test_inverse_reaches_every_iteration_count(f, p):
    """Fp::inv's k = 254..507: every doubling count of the j = 512 - k >= 256 tail and every multiplier 2^j, j <= 255.
    k = 508 is reached by none of the candidates (and not asserted)."""
    ks = set()
    for c, r in A.corpus()[f + "_inv"]:
        a = A.num(r)
        if c.startswith("iter_"):
            k = A.kaliski_k(a, p)
            assert k == int(c[5:])
            ks.add(k)
    assert ks >= set(range(254, 508))
    assert 508 not in ks


@pytest.mark.parametrize("f,p", [("fq", P), ("fr", R)])
def test_add_sub_classes(f, p):
    cls = _classes(f + "_add")
    for c, n in (("sum_p", 5), ("sum_p_minus_1", 5), ("sum_2p_minus_2", 1), ("diff_minus_1", 5), ("carry_ripple", 7),
                 ("borrow_ripple", 7)):
        assert cls[c] >= n, c
    for c, a, b in _pairs(f + "_add"):
        assert a < p and b < p
        if c == "sum_p":
            assert a + b == p
        if c == "sum_p_minus_1":
            assert a + b == p - 1
        if c == "sum_2p_minus_2":
            assert a + b == 2 * p - 2
        if c == "diff_minus_1":
            assert a - b == -1
    ripples = sorted((a ^ (a + b)).bit_length() for c, a, b in _pairs(f + "_add") if c == "carry_ripple")
    assert ripples == [32 * i + 1 for i in range(1, 8)]          # the carry crosses 1..7 limb boundaries


def test_sqrt_and_larger_classes():
    for c, r in A.corpus()["fq_sqrt"]:
        v = A.fq_v(r)
        s = pow(v, (P + 1) // 4, P)
        if c == "residue":
            assert s * s % P == v
        if c in ("non_residue", "minus_one"):
            assert s * s % P != v
    for c, r in A.corpus()["fq2_sqrt"]:
        a = A.fq2_v(r)
        s = o.fq2_sqrt(a)
        if c == "non_square":
            assert s is None
        else:
            assert s is not None and o.fq2_sqr(s) == a                  # every root the reference expects squares back
        if c.startswith("c1_zero"):
            assert a[1] == 0 and a[0] != 0
            assert (pow(a[0], (P - 1) // 2, P) == 1) == (c == "c1_zero_residue")
    cls = _classes("fq2_sqrt")
    for c in ("c1_zero_residue", "c1_zero_non_residue", "c0_zero", "zero", "non_square", "square"):
        assert cls[c] >= 1, c
    vals = {A.fq_v(r) for _, r in A.corpus()["fq_is_larger"]}
    assert {(P - 1) // 2, (P + 1) // 2} <= vals
    l2 = [A.fq2_v(r) for _, r in A.corpus()["fq2_is_larger"]]
    assert any(a[1] == 0 and a[0] > (P - 1) // 2 for a in l2) and any(a[1] == 0 and 0 < a[0] <= (P - 1) // 2 for a in l2)
    half = [A.num(r) for c, r in A.corpus()["fq_half"] if c == "noncanonical_odd_carry"]
    assert half and all(a % 2 and a + P >= MONT for a in half)               # the carry into the ninth word
    fb = _classes("fq_from_bytes")
    assert fb["ge_p"] >= 4 and fb["lt_p"] >= 4


def test_tower_and_pairing_classes():
    for name in ("fq6_inv", "fq12_inv", "fq12_frob2"):
        cls = _classes(name)
        for c in ("one", "fq_subfield", "fq2_subfield", "b_zero", "a_zero", "c_zero", "random"):
            assert cls[c] >= 1, (name, c)
    for c in ("c1_zero", "c0_zero", "line"):
        assert _classes("fq12_inv")[c] >= 1
    # the sparsity patterns are what their names say (Fq2 blocks a, b, c of the first Fq6: words 0-7, 8-15, 16-23)
    blocks = lambda r: tuple(any(r[i:i + 8]) for i in (0, 8, 16))
    want = {"b_zero": (True, False, True), "a_zero": (False, True, True), "c_zero": (True, True, False),
            "fq2_subfield": (True, False, False)}
    for c, r in A.corpus()["fq6_inv"]:
        if c in want:
            assert blocks(r) == want[c], c
    # the tower map is the inverse of the reader
    f = tuple(range(1, 13))
    assert A.fq12_v(A.fq12_w(f)) == f and o.fq12_mul(f, A.fq12_inv(f)) == o.FQ12_ONE
    cls = _classes("pairing")
    assert set(cls) >= {"P=O", "Q=O", "-P", "-Q", "random", "generators"}


def test_glv_corpus_and_reference():
    ks = [A.num(r) for _, r in A.corpus()["glv_decompose"]]
    lam = dl.LAMBDA
    assert {0, 1, lam, R - 1, R - lam} <= set(ks)
    for k in ks:
        k1, k2 = dl.glv_decompose(k)
        assert (k1 + lam * k2 - k) % R == 0 and abs(k1) < 1 << 127 and abs(k2) < 1 << 127
    assert len(_classes("glv_decompose")) >= 4


@pytest.mark.parametrize("g", ["g1", "g2"])
def test_group_law_relations(g):
    for name in ("add", "add_ilp", "quad_add"):
        cls = _classes("%s_%s" % (g, name))
        for c in ("Q=P", "Q=-P", "Q=O", "P=O", "Q=2P", "random"):
            assert cls[c] >= 1, (name, c)
    # quad_ops: every warp's eight quads hold eight different relations
    recs = A.corpus()[g + "_quad_add"]
    assert len(recs) % 8 == 0
    for w in range(0, len(recs), 8):
        assert len({c for c, _ in recs[w:w + 8]}) == 8
    madd = _classes(g + "_madd")
    for c in ("acc=p", "acc=-p", "acc=p_negated", "acc=-p_negated", "acc=O", "p=O"):
        assert madd[c] >= 1
    ks = _classes(g + "_mul_scalar")
    for c in ("k=0", "k=1", "k=r-1", "k=r", "k=2^256-1"):
        assert ks[c] >= 1
    # z values: raw limbs 1, p - 1 and 2^64 - 1 among the lifted points' ZZ^(1/2)
    G = A.G1 if g == "g1" else A.G2
    zs = A._z_values(G, random.Random(1))
    raws = {A.to_raw(z if g == "g1" else z[0]) for z in zs}
    assert {1, P - 1, (1 << 64) - 1} <= raws
