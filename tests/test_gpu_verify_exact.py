"""The accept / reject decisions of the verifier and of the ceremony checks, and the phase-2 point kernels, against exact
answers from known discrete logs.

If every point is a known multiple of the generator (alpha = al G1, beta = be G2, ..., A = a G1, B = b G2, C = c G1,
IC_i = ic_i G1), the Groth16 equation e(A, B) = e(alpha, beta) e(S, gamma) e(C, delta), S = IC_0 + sum_i x_i IC_{i+1},
holds iff

    a b = al be + ga s + c de  (mod r),    s = ic_0 + sum_i x_i ic_{i+1},

so any number of valid and invalid proofs can be built and judged with Python integers, without a pairing on the host.
Points with known logs come from fixed_base_mul_dev (exact-tested in test_gpu_qap_setup_exact.py; a few are checked here
against dlog_oracle.point_from_exponent) and Net.generate_g1/g2 (logs dlog_oracle.base_logs).  Covered here:
  - k_groth16_verify through verify.verify_proof (limb tuples and the 128-byte form) on keys with n_public = 0, 1, 2, 17
    and 1000: public inputs 0, 1 and r - 1, an IC_i at infinity, inputs that make S = O with IC_0 != O, an IC sum whose
    first addition doubles; valid proofs with A = O, B = O or C = O; every public input (a sample at 1000) moved by 1,
    A, B, C and every vk element replaced, A and C swapped; 200 random (key, proof, flip) cases at n_public = 2..17; the
    n_public = 17 case through circom.groth16_verify on JSON.  A moved input or a replaced IC term whose weight is zero
    (IC_i = O, x_i = 0) leaves S, and so the verdict, unchanged: the equation says so and the kernel must agree;
  - phase2._same_ratio (every ceremony check) against p1 q2 == p2 q1 (mod r), with every slot at infinity alone and in pairs;
  - snarkjs.alphabeta_12 against the oracle pairing raised to ffjavascript's multiple 2u(6u^2 + 3u + 1), alpha or beta = O;
  - points_scale_dev on G1 (GLV + width-5 NAF) at scalars on the split's edges (zero, negative and extreme halves, NAF digit
    patterns on both halves, lambda, r - lambda, 2^127, 2^128 +- 1, 2..33, k >= r), at n = 1, 63, 64, 65, a block that is
    all infinity and one with a single finite point, and 2^20 + 77 (out of place and in place); on G2 (the ladder) at n = 33;
  - points_spmv_dev on G1 and G2 at row lengths 255..258 around the MSM threshold (256), adjacent long rows, a long row
    first and last, a long row of zero coefficients, rows with a repeated or cancelling entry, and nnz = 0 with empty
    (null) idx and val; the number of rows sent to the MSM is checked through the launch profile, since both paths give the same points.
Device outputs start as all-ones words.  A failure names the kernel, the size and the case.

k_groth16_verify sums the IC terms on one thread (a 256-bit double-and-add per input).  Measured with
tools/verify_bench.py (CUDA events around one b200zk_groth16_verify call, median of 5) on an H100 80GB HBM3 at a 700 W
power limit: 56.5 ms at n_public = 1, 89.9 ms at 17, 2.00 s at 1000 and 8.03 s at 2^12, i.e. about 2 ms per public
input on top of the pairings.  This file ran in 112 s on the same card, 52 s of it in the n_public = 1000 key."""
import os
import random
import sys

import numpy as np
import pytest

from distributed_groth16_b200 import ark_serialize as ark, formats
from distributed_groth16_b200._native import c_vp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import dlog_oracle as dl  # noqa: E402
from oracle import bn254 as o, layout  # noqa: E402

pytestmark = pytest.mark.gpu
R = o.R
MASK64 = (1 << 64) - 1
U = o.BN_U
SNARKJS_M = 2 * U * (6 * U * U + 3 * U + 1)


# ---- helpers ---------------------------------------------------------------------------------------------------------
def host(t):
    return t.cpu().numpy().view(np.uint64)


def filled(net, shape):
    import torch
    return torch.full(shape, -1, dtype=torch.int64, device=net._dev())


def mont(vals) -> np.ndarray:
    """canonical ints (any sign, any size) -> (n, 4) Montgomery limbs"""
    b = b"".join((v % R * o.MONT_R % R).to_bytes(32, "little") for v in vals)
    return np.frombuffer(b, dtype=np.uint64).reshape(-1, 4).copy()


def points_dev(net, exps, g2=False):
    """e G for every e of exps (fixed_base_mul_dev), a CUDA int64 (n, 8 | 16) tensor"""
    n = len(exps)
    out = filled(net, (max(n, 1), 16 if g2 else 8))
    if n:
        sc = net.to_device(mont(exps))
        net.check(net._lib.b200zk_fixed_base_mul_dev(net._h, int(g2), c_vp(sc.data_ptr()), n, c_vp(out.data_ptr())))
    return out[:n]


def points(net, exps, g2=False) -> np.ndarray:
    return host(points_dev(net, exps, g2))


def first_rows(bad, k=6):
    import torch
    return torch.nonzero(bad).reshape(-1)[:k].tolist()


def test_fixed_base_points_are_the_known_multiples(net):
    """The expected points of this file, spot-checked against the oracle's scalar multiplication."""
    es = [0, 1, 2, R - 1, dl.LAMBDA, 0x1234567890ABCDEF << 130]
    for g2 in (False, True):
        got = points(net, es, g2)
        for e, row in zip(es, got):
            want, _ = dl.point_from_exponent(e, g2)
            assert (row == want).all(), "fixed_base_mul_dev %s: e = %#x" % ("G2" if g2 else "G1", e)


# ---- the verifier, by logs -------------------------------------------------------------------------------------------
class Case:
    """logs of one (vk, public inputs, proof) triple"""

    def __init__(self, what, alpha, beta, gamma, delta, ic, x, a, b, c):
        self.what, self.alpha, self.beta, self.gamma, self.delta = what, alpha, beta, gamma, delta
        self.ic, self.x, self.a, self.b, self.c = list(ic), list(x), a, b, c

    def s(self):
        return (self.ic[0] + sum(xi * l for xi, l in zip(self.x, self.ic[1:]))) % R

    def holds(self):
        return (self.a * self.b - self.alpha * self.beta - self.gamma * self.s() - self.c * self.delta) % R == 0

    def but(self, what, **kw):
        d = dict(alpha=self.alpha, beta=self.beta, gamma=self.gamma, delta=self.delta, ic=self.ic, x=self.x, a=self.a,
                 b=self.b, c=self.c)
        d.update(kw)
        return Case("%s, %s" % (self.what, what), **d)


def solve_c(k, a, b):
    """c with a b = al be + ga s + c de"""
    return (a * b - k.alpha * k.beta - k.gamma * k.s()) * pow(k.delta, -1, R) % R


def valid_proofs(key, rng):
    """valid (a, b, c) on key: random a, b; A = O; B = O; C = O (a b = al be + ga s)"""
    rnd = lambda: rng.randrange(1, R)
    a, b = rnd(), rnd()
    out = [key.but("valid", a=a, b=b, c=solve_c(key, a, b))]
    b = rnd()
    out.append(key.but("A = O", a=0, b=b, c=solve_c(key, 0, b)))
    a = rnd()
    out.append(key.but("B = O", a=a, b=0, c=solve_c(key, a, 0)))
    a = rnd()
    out.append(key.but("C = O", a=a, b=(key.alpha * key.beta + key.gamma * key.s()) * pow(a, -1, R) % R, c=0))
    for p in out:
        assert p.holds(), p.what
    return out


def mutations(p, rng, inputs):
    """p with one public input moved by 1 (indices `inputs`), A, B, C, every vk element replaced, A and C swapped"""
    rnd = lambda: rng.randrange(1, R)
    fixed = [p.but("A other", a=rnd()), p.but("B other", b=rnd()), p.but("C other", c=rnd()), p.but("A <-> C", a=p.c, c=p.a)]
    fixed += [p.but(name + " other", **{name: rnd()}) for name in ("alpha", "beta", "gamma", "delta")]
    for m in fixed:
        if not (p.s() == 0 and m.what.endswith("gamma other")):
            assert not m.holds(), m.what                     # A, B, C, alpha .. delta matter, gamma unless S = O
    weighted = [p.but("x[%d] + 1" % i, x=p.x[:i] + [(p.x[i] + 1) % R] + p.x[i + 1:]) for i in inputs]
    n = len(p.ic) - 1
    for j in sorted({0, n} | {j for j in range(1, n + 1) if p.ic[j] == 0 or p.x[j - 1] == 0}):
        weighted.append(p.but("IC_%d other" % j, ic=p.ic[:j] + [rnd()] + p.ic[j + 1:]))
    return fixed + weighted


def run_cases(net, cases, byte_form=False):
    """verify.verify_proof verdicts; points by two fixed_base_mul_dev calls for all cases"""
    from distributed_groth16_b200.groth16 import verify
    g1 = [e for k in cases for e in [k.alpha, k.a, k.c] + k.ic]
    g2 = [e for k in cases for e in (k.beta, k.gamma, k.delta, k.b)]
    p1, p2 = points(net, g1), points(net, g2, True)
    out, i = [], 0
    for j, k in enumerate(cases):
        alpha, a, c = p1[i:i + 3]
        ic = p1[i + 3:i + 3 + len(k.ic)]
        i += 3 + len(k.ic)
        beta, gamma, delta, b = p2[4 * j:4 * j + 4]
        vk = ark.ArkVerifyingKey(alpha, beta, gamma, delta, ic)
        x = layout.fr_to_arr(k.x)
        got = verify.verify_proof(net, vk, x, (a, b, c))
        if byte_form:
            blob = ark.serialize_proof(net, a, b, c)
            assert verify.verify_proof(net, vk, x, blob) == got, "k_groth16_verify n_public=%d %s: byte form differs" % (
                len(k.x), k.what)
        out.append(got)
    return out


def _key(what, rng, ic, x):
    rnd = lambda: rng.randrange(1, R)
    return Case(what, rnd(), rnd(), rnd(), rnd(), ic, x, 0, 0, 0)


def designed_keys(rng):
    """(key, public-input indices to move) for n_public = 0, 1, 2, 17, 1000"""
    rnd = lambda: rng.randrange(1, R)
    keys = [(_key("n_public=0", rng, [rnd()], []), [])]
    keys.append((_key("n_public=1, x = r - 1", rng, [rnd(), rnd()], [R - 1]), [0]))
    i0, i1, i2 = rnd(), rnd(), rnd()
    keys.append((_key("n_public=2, S = O", rng, [i0, i1, i2], [1, -(i0 + i1) * pow(i2, -1, R) % R]), [0, 1]))
    x0 = rnd()
    keys.append((_key("n_public=2, IC_0 = x_0 IC_1 (doubling), x_1 = 0", rng, [x0 * i1 % R, i1, i2], [x0, 0]), [0, 1]))
    ic = [rnd() for _ in range(18)]
    ic[6] = 0                                                   # IC_6 = O: x[5] has weight zero
    x = [0, 1, R - 1] + [rnd() for _ in range(14)]
    x[9] = 0
    keys.append((_key("n_public=17, IC_6 = O", rng, ic, x), list(range(17))))
    ic = [rnd() for _ in range(1001)]
    ic[500] = 0
    x = [0, 1, R - 1] + [rnd() for _ in range(997)]
    x[700] = 0
    keys.append((_key("n_public=1000, IC_500 = O", rng, ic, x), [0, 1, 2, 499, 700, 998, 999]))
    for k, _ in keys:
        assert k.s() != 0 or "S = O" in k.what
    return keys


@pytest.fixture(scope="module")
def designed():
    return designed_keys(random.Random(0x5E81F1))


@pytest.mark.parametrize("which", range(6), ids=["n0", "n1", "n2_S=O", "n2_dbl", "n17", "n1000"])
def test_verify_designed_keys_accepts_exactly_when_the_log_equation_holds(net, designed, which):
    key, inputs = designed[which]
    rng = random.Random(0x7E57 + which)
    small = len(key.x) <= 17
    cases = []
    for p in valid_proofs(key, rng):
        cases += [p] + (mutations(p, rng, inputs) if p.what.endswith("valid") else [])
    got = run_cases(net, cases, byte_form=small)
    bad = [(c.what, g) for c, g in zip(cases, got) if g != c.holds()]
    assert not bad, "k_groth16_verify n_public=%d: verdict != log equation for %s" % (len(key.x), bad)
    n_valid = sum(c.holds() for c in cases)
    assert n_valid >= 4 and len(cases) - n_valid >= 8, (n_valid, len(cases))
    if "S = O" in key.what:
        assert key.s() == 0 and key.ic[0] != 0
    if not small:                                           # the other valid proofs in the 128-byte form too
        for p, g in zip(cases[:1], run_cases(net, cases[:1], byte_form=True)):
            assert g, p.what


def test_verify_random_keys_proofs_and_flips(net):
    """200 (key, proof, flip) cases at n_public = 2..17: the verdict equals the log equation in every case."""
    rng = random.Random(0xC0FFEE)
    rnd = lambda: rng.randrange(1, R)
    special = [0, 1, R - 1]
    cases = []
    for t in range(200):
        n = rng.randint(2, 17)
        ic = [rnd() if rng.random() > 0.15 else 0 for _ in range(n + 1)]
        x = [rng.choice(special) if rng.random() < 0.25 else rnd() for _ in range(n)]
        key = _key("random #%d n_public=%d" % (t, n), rng, ic, x)
        p = rng.choice(valid_proofs(key, rng))
        flip = rng.choice(["none"] * 4 + ["x", "A", "B", "C", "alpha", "beta", "gamma", "delta", "ic", "swap"])
        if flip == "x":
            i = rng.randrange(n)
            p = p.but("x[%d] + 1" % i, x=p.x[:i] + [(p.x[i] + 1) % R] + p.x[i + 1:])
        elif flip == "ic":
            j = rng.randrange(n + 1)
            p = p.but("IC_%d other" % j, ic=p.ic[:j] + [rnd()] + p.ic[j + 1:])
        elif flip == "swap":
            p = p.but("A <-> C", a=p.c, c=p.a)
        elif flip != "none":
            name = {"A": "a", "B": "b", "C": "c"}.get(flip, flip)
            p = p.but(flip + " other", **{name: rnd()})
        cases.append(p)
    got = run_cases(net, cases)
    bad = [(c.what, g) for c, g in zip(cases, got) if g != c.holds()]
    assert not bad, "k_groth16_verify random cases: verdict != log equation for %s" % bad
    n_valid = sum(got)
    assert 50 <= n_valid <= 150, n_valid


def test_verify_n17_through_snarkjs_json(net, designed):
    """circom.groth16_verify on verification_key.json / public.json / proof.json text of the n_public = 17 key"""
    from distributed_groth16_b200.groth16 import circom, snarkjs
    key, _ = designed[4]
    rng = random.Random(0x15017)
    valid = valid_proofs(key, rng)
    p1 = points(net, [key.alpha] + key.ic)
    p2 = points(net, [key.beta, key.gamma, key.delta], True)
    g1 = lambda rows: layout.arr_to_g1(rows)
    g2 = lambda rows: layout.arr_to_g2(rows)
    ab = snarkjs.alphabeta_12(net, p1[0], p2[0])
    (beta, gamma, delta) = g2(p2)
    vk_json = formats.write_vk_json(formats.SnarkjsVerificationKey(17, g1(p1[:1])[0], beta, gamma, delta, ab, g1(p1[1:])))

    def proof_json(p):
        (a, c), (b,) = g1(points(net, [p.a, p.c])), g2(points(net, [p.b], True))
        return formats.write_proof_json(formats.SnarkjsProof(a, b, c))

    cases = valid + [valid[0].but("x[0] + 1", x=[1] + key.x[1:]), valid[0].but("x[5] + 1 (IC_6 = O)", x=key.x[:5] + [(key.x[5] + 1) % R] + key.x[6:]),
                     valid[0].but("C other", c=rng.randrange(1, R))]
    for p in cases:
        got = circom.groth16_verify(net, vk_json, formats.write_public_json(p.x), proof_json(p))
        assert got == p.holds(), "groth16_verify (JSON) n_public=17 %s: got %s" % (p.what, got)
    assert [p.holds() for p in cases] == [True] * 4 + [False, True, False]


# ---- _same_ratio ------------------------------------------------------------------------------------------------------
def test_same_ratio_is_the_log_equation_with_every_slot_at_infinity(net):
    """_same_ratio(P1, P2, Q1, Q2) == (p1 q2 == p2 q1 mod r); slots at infinity alone and in pairs, random and equal
    ratios"""
    from itertools import combinations
    from distributed_groth16_b200.groth16.phase2 import _same_ratio
    rng = random.Random(0x5A4E)
    rnd = lambda: rng.randrange(1, R)
    cases = [(rnd(), rnd(), rnd(), rnd()) for _ in range(6)]
    for _ in range(6):
        p1, q1, t = rnd(), rnd(), rnd()
        cases.append((p1, p1 * t % R, q1, q1 * t % R))                       # equal ratios
    cases.append((1, 1, 1, 1))
    cases.append((R - 1, 1, 1, R - 1))
    base = list(cases[-3])
    for k in (1, 2, 4):
        for slots in combinations(range(4), k):
            for src in (base, [rnd() for _ in range(4)]):
                cases.append(tuple(0 if i in slots else v for i, v in enumerate(src)))
    g1 = points(net, [e for c in cases for e in c[:2]])
    g2 = points(net, [e for c in cases for e in c[2:]], True)
    bad = []
    for i, (p1, p2, q1, q2) in enumerate(cases):
        want = (p1 * q2 - p2 * q1) % R == 0
        got = _same_ratio(net, g1[2 * i], g1[2 * i + 1], g2[2 * i], g2[2 * i + 1])
        if got != want:
            bad.append(((p1, p2, q1, q2), got))
    assert not bad, "same_ratio (k_groth16_verify, no inputs): %s" % bad
    wants = [(c[0] * c[3] - c[1] * c[2]) % R == 0 for c in cases]
    assert 10 <= sum(wants) <= len(cases) - 10


# ---- vk_alphabeta_12 --------------------------------------------------------------------------------------------------
def _snarkjs_nesting(f):
    """Oracle Fq12 (coefficients of w^0..w^11, u = w^6 - 9) -> snarkjs's [[c0.a, c0.b, c0.c], [c1.a, c1.b, c1.c]]"""
    out = [[None] * 3 for _ in range(2)]
    for (h, k), i in zip(((0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (1, 2)), (0, 2, 4, 1, 3, 5)):
        y = f[i + 6]
        out[h][k] = [(f[i] + 9 * y) % o.P, y]
    return out


def test_alphabeta_12_against_the_oracle_pairing(net):
    from distributed_groth16_b200.groth16 import snarkjs
    rng = random.Random(0xAB12)
    cases = [(rng.randrange(1, R), rng.randrange(1, R)) for _ in range(4)] + [(0, rng.randrange(1, R)), (rng.randrange(1, R), 0)]
    for a, b in cases:
        pa = o.G1.mul(o.G1_GEN, a) if a else None
        pb = o.G2.mul(o.G2_GEN, b) if b else None
        got = snarkjs.alphabeta_12(net, layout.g1_to_arr([pa])[0], layout.g2_to_arr([pb])[0])
        want = _snarkjs_nesting(o.fq12_pow(o.pairing(pa, pb), SNARKJS_M))
        assert got == want, "vk_alphabeta_12: alpha = %#x G1, beta = %#x G2" % (a, b)
        if not (a and b):
            assert want == _snarkjs_nesting(o.FQ12_ONE)


# ---- points_scale_dev -------------------------------------------------------------------------------------------------
def scale_scalars():
    """(name, k as a 256-bit integer) on the GLV split's edges"""
    ks = [("halves %d,%d" % (h1.bit_length() * (1 if h1 >= 0 else -1), h2.bit_length() * (1 if h2 >= 0 else -1)),
           dl.glv_compose(h1, h2)) for h1, h2 in dl.glv_designed_halves()]
    ext = dl.glv_extremes(1 << 14)
    ks += [("largest |k1|", ext[0]), ("largest |k2|", ext[1])]
    for fam, vals in dl.digit_families(5, True).items():
        ks += [("%s #%d" % (fam, i), v) for i, v in enumerate(vals)]
    lam = dl.LAMBDA
    ks += [("lambda", lam), ("r - lambda", R - lam), ("2^127", 1 << 127), ("2^128 - 1", (1 << 128) - 1), ("2^128", 1 << 128),
           ("2^128 + 1", (1 << 128) + 1)]
    ks += [("%d" % v, v) for v in range(2, 34)]
    ks += [("r", R), ("r + 1", R + 1), ("r + lambda", R + lam), ("2r - 1", 2 * R - 1), ("5r + 12345", 5 * R + 12345),
           ("2^256 - 1", (1 << 256) - 1)]
    for name, k in ks:
        assert 0 <= k < 1 << 256, name
    return ks


def scale_dev(net, pts, k, g2, in_place=False):
    out = pts if in_place else filled(net, tuple(pts.shape))
    kl = np.array([(k >> (64 * i)) & MASK64 for i in range(4)], dtype=np.uint64)
    net.check(net._lib.b200zk_points_scale_dev(net._h, 0, int(g2), c_vp(pts.data_ptr()), int(pts.shape[0]),
                                               c_vp(kl.ctypes.data), c_vp(out.data_ptr())))
    return out


def known_log_points(net, seed, n, inf_rows, g2=False):
    """generated points with some rows at infinity, and their logs as Python ints"""
    import torch
    pts = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
    logs = dl.base_logs(seed, n).tolist()
    if inf_rows:
        pts[torch.tensor(inf_rows, device=pts.device)] = 0
    for i in inf_rows:
        logs[i] = 0
    return pts, logs


SCALE_SHAPES = {"n1": (1, []), "n63": (63, [0, 62]), "n64": (64, [31]), "n65": (65, [64]),
                "n192_block_inf_and_single": (192, list(range(64, 128)) + [i for i in range(128, 192) if i != 150])}


@pytest.mark.parametrize("shape", list(SCALE_SHAPES))
def test_points_scale_g1_at_the_splits_edges(net, shape):
    import torch
    n, inf_rows = SCALE_SHAPES[shape]
    pts, logs = known_log_points(net, 0x5CA1E000 + n, n, inf_rows)
    before = pts.clone()
    ks = scale_scalars()
    want = points_dev(net, [k * l for _, k in ks for l in logs]).reshape(len(ks), n, 8)
    for j, (name, k) in enumerate(ks):
        got = scale_dev(net, pts, k, False)
        bad = (got != want[j]).any(dim=1)
        assert not bad.any(), "points_scale_dev G1 n=%d (%s) k = %s (%#x): rows %s wrong" % (n, shape, name, k, first_rows(bad))
    assert torch.equal(pts, before), "points_scale_dev G1 n=%d: the input was modified" % n


def test_points_scale_g1_at_2_20_plus_77_out_of_place_and_in_place(net):
    n = (1 << 20) + 77
    inf_rows = [0] + list(range(64 * 7, 64 * 8)) + [i for i in range(64 * 9, 64 * 10) if i != 64 * 9 + 17] + [n - 1]
    pts, logs = known_log_points(net, 0x5CA1E20, n, inf_rows)
    ext = dl.glv_extremes(1 << 14)
    a, b = (1 << 124) + 12345, (1 << 123) + 678
    ks = [("largest |k1|", ext[0]), ("largest |k2|", ext[1]), ("halves -a,-b", dl.glv_compose(-a, -b)),
          ("r - lambda", R - dl.LAMBDA), ("2^256 - 1", (1 << 256) - 1)]
    rand = random.Random(0x20).randrange(1 << 256)
    for j, (name, k) in enumerate(ks + [("random, in place", rand)]):
        km = k % R
        want = points_dev(net, [km * l for l in logs])
        got = scale_dev(net, pts, k, False, in_place=(j == len(ks)))
        bad = (got != want).any(dim=1)
        assert not bad.any(), "points_scale_dev G1 n=2^20+77 k = %s: %d rows wrong, first %s" % (name, int(bad.sum()),
                                                                                                   first_rows(bad))


def test_points_scale_g2_ladder_at_the_same_scalars(net):
    n = 33
    pts, logs = known_log_points(net, 0x5CA1E2, n, [0, 17], g2=True)
    ks = scale_scalars()
    want = points_dev(net, [k * l for _, k in ks for l in logs], True).reshape(len(ks), n, 16)
    for j, (name, k) in enumerate(ks):
        got = scale_dev(net, pts, k, True)
        bad = (got != want[j]).any(dim=1)
        assert not bad.any(), "points_scale_dev G2 n=%d k = %s (%#x): rows %s wrong" % (n, name, k, first_rows(bad))


# ---- points_spmv_dev --------------------------------------------------------------------------------------------------
SPMV_MSM_ROW = 256                     # rows longer than this take the MSM path (csrc/setup.cu)


def spmv_dev(net, ptr, idx, val_m, pts, n_rows, g2):
    out = filled(net, (n_rows, 16 if g2 else 8))
    d = lambda a: net.to_device(np.ascontiguousarray(a).view(np.int32) if a.dtype == np.uint32 else a)
    ptr_d, idx_d, val_d = d(ptr), d(idx), d(val_m)
    net.check(net._lib.b200zk_points_spmv_dev(net._h, 0, int(g2), c_vp(ptr_d.data_ptr()), c_vp(idx_d.data_ptr()),
                                              c_vp(val_d.data_ptr()), c_vp(pts.data_ptr()), n_rows, c_vp(out.data_ptr())))
    return host(out)


@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_points_spmv_row_lengths_at_the_msm_threshold(net, g2):
    """Long rows first, adjacent and last, lengths 255..258, a long row of zero coefficients, repeated and cancelling
    entries; each row against point_from_exponent(sum v log), and the MSM path taken by exactly the rows longer than 256"""
    rng = random.Random(0x5B3 + g2)
    n_pts = 600
    pts, logs = known_log_points(net, 0x5B3000 + g2, n_pts, [3, 77, 400], g2)
    rows = []                                          # (what, [(idx, canonical v)])
    full = lambda: rng.randrange(R)
    pick = lambda: rng.choice([0, 1, R - 1, rng.randrange(1, 1 << 64), full(), full(), full()])
    gen = lambda ln: [(rng.randrange(n_pts), pick()) for _ in range(ln)]
    rows.append(("long first (300)", gen(300)))
    rows.append(("long adjacent (257)", gen(257)))
    rows.append(("short (3)", gen(3)))
    for ln in (255, 256, 257, 258):
        rows.append(("length %d" % ln, gen(ln)))
    rows.append(("empty", []))
    j, v = rng.randrange(4, 70), full()
    rows.append(("repeated entry", [(j, v), (j, v)]))
    rows.append(("cancelling entry", [(j, v), (j, R - v)]))
    rows.append(("repeated, cancelling and infinity", [(j, v), (j + 1, 5), (j, v), (j + 1, R - 5), (3, v)]))
    rows.append(("256 equal products", [(j, v)] * 256))
    rows.append(("long, zero coefficients (260)", [(rng.randrange(n_pts), 0) for _ in range(260)]))
    rows.append(("long, cancelling pairs (262)", [e for a in gen(131) for e in (a, (a[0], (R - a[1]) % R))]))
    rows.append(("short (5)", gen(5)))
    rows.append(("long last (259)", gen(259)))
    lens = [len(r) for _, r in rows]
    ptr = np.zeros(len(rows) + 1, dtype=np.uint32)
    ptr[1:] = np.cumsum(lens)
    ent = [e for _, r in rows for e in r]
    idx = np.array([e[0] for e in ent], dtype=np.uint32)
    net.profile(True)
    net.profile_reset()
    try:
        got = spmv_dev(net, ptr, idx, mont([e[1] for e in ent]), pts, len(rows), g2)
        prof = net.profile_report()
    finally:
        net.profile(False)
        net.profile_reset()
    for (what, r), row in zip(rows, got):
        want, _ = dl.point_from_exponent(sum(v * logs[i] for i, v in r), g2)
        assert (row == want).all(), "points_spmv_dev %s rows=%d: row '%s' (%d entries) wrong" % (
            "G2" if g2 else "G1", len(rows), what, len(r))
    long_rows = [i for i, ln in enumerate(lens) if ln > SPMV_MSM_ROW]
    gaps = sum(1 for lo, hi in zip([0] + [int(ptr[i + 1]) for i in long_rows], [int(ptr[i]) for i in long_rows] + [int(ptr[-1])])
               if hi > lo)
    launches = {k: prof.get(k, {}).get("launches", 0) for k in ("points_gather", "xyzz_to_affine", "points_spmv_products")}
    assert launches == {"points_gather": len(long_rows), "xyzz_to_affine": len(long_rows), "points_spmv_products": gaps}, (
        "points_spmv_dev %s: rows longer than %d must take the MSM path, %s" % ("G2" if g2 else "G1", SPMV_MSM_ROW, launches))


@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_points_spmv_no_nonzeros(net, g2):
    """nnz = 0 with n_rows > 0 (a query matrix with no entries, as an empty B): the empty idx and val tensors have null
    data pointers, and every row is the point at infinity.  With nnz > 0 a null idx is refused before any launch."""
    from distributed_groth16_b200 import B200zkError
    pts, _ = known_log_points(net, 0x5B4, 8, [], g2)
    got = spmv_dev(net, np.zeros(6, dtype=np.uint32), np.zeros(0, dtype=np.uint32), np.zeros((0, 4), dtype=np.uint64), pts, 5, g2)
    assert not got.any(), "points_spmv_dev %s n_rows=5 nnz=0: rows not infinity" % ("G2" if g2 else "G1")
    ptr = net.to_device(np.array([0, 1], dtype=np.uint32).view(np.int32))
    val = net.to_device(mont([1]))
    first = net.launch_count()
    with pytest.raises(B200zkError):
        net.check(net._lib.b200zk_points_spmv_dev(net._h, 0, int(g2), c_vp(ptr.data_ptr()), None, c_vp(val.data_ptr()),
                                                  c_vp(pts.data_ptr()), 1, c_vp(pts.data_ptr())))
    assert net.launch_count() == first, "points_spmv_dev: the refusal of a null idx launched a kernel"
