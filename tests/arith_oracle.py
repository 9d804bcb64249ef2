"""Exact answers and the operand corpus for b200zk_test_arith (csrc/selftest.cu): every device primitive of fp.cuh, codec.cuh,
pairing.cuh, glv.cuh and ec.cuh against Python big integers (TEST INFRASTRUCTURE ONLY).

Records are lists of u64 words exactly as the op table in include/b200zk.h lays them out; field elements are raw Montgomery
limbs.  `OPS` names every op with its code, record sizes and reference; `corpus()` gives, per op, (class, record) pairs whose
operands were chosen with a model of the branch they are meant to reach:

- Montgomery product: the value before the final subtraction of any word-serial product is T = (t + M p) / 2^256 with
  M = -t p^-1 mod 2^256 (t = a b, or the 512-bit input of redc); the subtraction runs iff T >= p (`mont_pre`).
- Fq2::mul: c0 reduces t0 = a0 b0 - a1 b1 + p 2^256 and c1 reduces t2 = a0 b1 + a1 b0 with redc<2>; the class of each is
  mont_pre // p.  c1's T stays below 1.38 p, so its second subtraction cannot run.
- Fp::inv: the iteration count k of the binary extended Euclid (`kaliski_k`) selects the doubling tail (k <= 256) or the
  multiplier 2^(512 - k); every k in 254..507 is reached by simple raw values, k = 508 by none found.
"""
from __future__ import annotations

import functools
import random
from dataclasses import dataclass
from typing import Callable, List

from oracle import bn254 as o

import dlog_oracle as dl

P, R = o.P, o.R
MONT = 1 << 256
M64 = (1 << 64) - 1


# ---- words <-> integers, raw Montgomery <-> values -------------------------------------------------------------------
def words(x: int, n: int = 4) -> List[int]:
    return [(x >> (64 * i)) & M64 for i in range(n)]


def num(ws) -> int:
    return sum(int(w) << (64 * i) for i, w in enumerate(ws))


def mont_pre(t: int, p: int) -> int:
    """The value a Montgomery reduction of t holds before its conditional subtractions."""
    m = (-t * pow(p, -1, MONT)) % MONT
    return (t + m * p) >> 256


def kaliski_k(a: int, p: int) -> int:
    """Iterations of Fp::inv's loop on the raw value a (0 < a < p)."""
    u, v, k = p, a, 0
    while v:
        if u % 2 == 0:
            u >>= 1
        elif v % 2 == 0:
            v >>= 1
        elif u > v:
            u = (u - v) >> 1
        else:
            v = (v - u) >> 1
        k += 1
    return k


RINV = {P: pow(MONT, -1, P), R: pow(MONT, -1, R)}


def to_raw(v: int, p: int = P) -> int:
    return v % p * MONT % p


def to_val(raw: int, p: int = P) -> int:
    return raw * RINV[p] % p


def canonical(ws) -> bool:
    """Every 4-word Fq component of a record is below p."""
    return all(num(ws[i:i + 4]) < P for i in range(0, len(ws), 4))


# Fq2 / tower / points as values <-> raw words
def fq_w(v: int) -> List[int]:
    return words(to_raw(v))


def fq_v(ws) -> int:
    return to_val(num(ws))


def fq2_w(a) -> List[int]:
    return fq_w(a[0]) + fq_w(a[1])


def fq2_v(ws):
    return (fq_v(ws[0:4]), fq_v(ws[4:8]))


TOWER_ORDER = (0, 2, 4, 1, 3, 5)          # pairing.cuh's c0.a c0.b c0.c c1.a c1.b c1.c = w^0 w^2 w^4 w^1 w^3 w^5


def fq12_w(f) -> List[int]:
    """oracle Fq12 (12 coefficients in w, w^6 = 9 + u) -> the 48 words of pairing.cuh's Fq12."""
    out = []
    for i in TOWER_ORDER:
        y = f[i + 6]
        out += fq2_w(((f[i] + 9 * y) % P, y))
    return out


def fq12_v(ws):
    f = [0] * 12
    for j, i in enumerate(TOWER_ORDER[:len(ws) // 8]):
        x, y = fq2_v(ws[8 * j:8 * j + 8])
        f[i], f[i + 6] = (x - 9 * y) % P, y
    return tuple(f)


def fq6_w(f) -> List[int]:
    assert all(f[i] == 0 for i in (1, 3, 5, 7, 9, 11)), "not in Fq6"
    return fq12_w(f)[:24]


def fq12_inv(f):
    """f^-1 by solving f x = 1 over Fq (the columns of the matrix are f w^j); 0 -> 0."""
    if not any(f):
        return f
    cols = [o.fq12_mul(f, tuple(int(i == j) for i in range(12))) for j in range(12)]
    m = [[cols[j][i] for j in range(12)] + [int(i == 0)] for i in range(12)]
    for c in range(12):
        piv = next(r for r in range(c, 12) if m[r][c])
        m[c], m[piv] = m[piv], m[c]
        iv = pow(m[c][c], -1, P)
        m[c] = [x * iv % P for x in m[c]]
        for r in range(12):
            if r != c and m[r][c]:
                k = m[r][c]
                m[r] = [(x - k * y) % P for x, y in zip(m[r], m[c])]
    return tuple(m[i][12] for i in range(12))


W2 = tuple(int(i == 2) for i in range(12))          # v = w^2


# ---- points ------------------------------------------------------------------------------------------------------------
class _G:
    def __init__(self, curve, fw, fv, zero, one, gen, width):
        self.c, self.fw, self.fv, self.zero, self.one, self.gen, self.W = curve, fw, fv, zero, one, gen, width

    def aff_w(self, pt) -> List[int]:
        return [0] * (2 * self.W) if pt is None else self.fw(pt[0]) + self.fw(pt[1])

    def aff_v(self, ws):
        W = self.W
        if not any(ws):
            return None
        return (self.fv(ws[:W]), self.fv(ws[W:2 * W]))

    def xyzz_w(self, pt, z) -> List[int]:
        """pt lifted to XYZZ with z (a field value): X = x z^2, Y = y z^3, ZZ = z^2, ZZZ = z^3; None -> all zero."""
        if pt is None:
            return [0] * (4 * self.W)
        F = self.c.F
        zz = F.mul(z, z)
        zzz = F.mul(zz, z)
        return self.fw(F.mul(pt[0], zz)) + self.fw(F.mul(pt[1], zzz)) + self.fw(zz) + self.fw(zzz)

    def xyzz_view(self, ws):
        """A device XYZZ record as ('inf',), ('pt', x, y), ('bad', ...) when ZZ^3 != ZZZ^2, or ('noncanonical', words) when
        any Fq component is not below p: the group law keeps every coordinate canonical, and a skipped final subtraction
        would otherwise read as the right value modulo p."""
        if not canonical(ws):
            return ("noncanonical", tuple(ws))
        F, W = self.c.F, self.W
        X, Y, ZZ, ZZZ = (self.fv(ws[i * W:(i + 1) * W]) for i in range(4))
        if ZZ == self.zero:
            return ("inf",)
        if F.mul(F.mul(ZZ, ZZ), ZZ) != F.mul(ZZZ, ZZZ):
            return ("bad", X, Y, ZZ, ZZZ)
        return ("pt", F.mul(X, F.inv(ZZ)), F.mul(Y, F.inv(ZZZ)))

    def aff_view(self, ws):
        if not canonical(ws):
            return ("noncanonical", tuple(ws))
        pt = self.aff_v(ws)
        return ("inf",) if pt is None else ("pt",) + pt

    @staticmethod
    def pt_view(pt):
        return ("inf",) if pt is None else ("pt",) + tuple(pt)


G1 = _G(o.G1, fq_w, fq_v, 0, 1, o.G1_GEN, 4)
G2 = _G(o.G2, fq2_w, fq2_v, o.FQ2_ZERO, o.FQ2_ONE, o.G2_GEN, 8)

# phi's constants from their definition: phi(P) = lambda P with y unchanged, read off the generators (G1's x is 1)
BETA_G1 = o.G1.mul(o.G1_GEN, dl.LAMBDA)[0]
_lg2 = o.G2.mul(o.G2_GEN, dl.LAMBDA)
assert _lg2[1] == o.G2_GEN[1] and o.G1.mul(o.G1_GEN, dl.LAMBDA)[1] == o.G1_GEN[1]
BETA_G2 = o.fq2_mul(_lg2[0], o.fq2_inv(o.G2_GEN[0]))
assert BETA_G2[1] == 0
BETA_G2 = BETA_G2[0]


# ---- the op table --------------------------------------------------------------------------------------------------------
@dataclass
class Op:
    name: str
    code: int
    n_in: int
    n_out: int
    ref: Callable                           # record -> expected, in the form `view` gives the device's output
    view: Callable = list
    device_only: bool = False
    field: str = ""


OPS: dict = {}


def _op(name, code, n_in, n_out, ref, view=list, device_only=False, field=""):
    OPS[name] = Op(name, code, n_in, n_out, ref, view, device_only, field)


FP_SUB = dict(add=0, sub=1, neg=2, dbl=3, mul=4, mul_ni=5, sqr=6, mul_any=7, mul_k2=8, mul_k3=9, mul_k4=10,
              mul_wide_redc1=11, redc2=12, inv=13, inv_fermat=14, to_mont=15, from_mont=16, from_u32=17, pow_u64=18)
FIELDS = {"fq": (P, 0), "fr": (R, 32)}


def _fp_refs(p):
    ri = RINV[p]
    mul = lambda a, b: a * b * ri % p
    inv = lambda a: 0 if a % p == 0 else MONT * MONT * pow(a, -1, p) % p
    pair = lambda f: lambda r: words(f(num(r[0:4]), num(r[4:8])))
    one = lambda f: lambda r: words(f(num(r[0:4])))
    mulk = lambda K: lambda r: sum((words(mul(num(r[8 * k:8 * k + 4]), num(r[8 * k + 4:8 * k + 8]))) for k in range(K)), [])
    return dict(
        add=(8, 4, pair(lambda a, b: (a + b) % p)), sub=(8, 4, pair(lambda a, b: (a - b) % p)),
        neg=(4, 4, one(lambda a: -a % p)), dbl=(4, 4, one(lambda a: 2 * a % p)),
        mul=(8, 4, pair(mul)), mul_ni=(8, 4, pair(mul)), sqr=(4, 4, one(lambda a: mul(a, a))), mul_any=(8, 4, pair(mul)),
        mul_k2=(16, 8, mulk(2)), mul_k3=(24, 12, mulk(3)), mul_k4=(32, 16, mulk(4)),
        mul_wide_redc1=(8, 12, lambda r: words(num(r[0:4]) * num(r[4:8]), 8) + words(mul(num(r[0:4]), num(r[4:8])))),
        redc2=(8, 4, lambda r: words(num(r) * ri % p)),
        inv=(4, 4, one(inv)), inv_fermat=(4, 4, one(inv)),
        to_mont=(4, 4, one(lambda a: a * MONT % p)), from_mont=(4, 4, one(lambda a: a * ri % p)),
        from_u32=(1, 4, lambda r: words((r[0] & 0xFFFFFFFF) * MONT % p)),
        pow_u64=(5, 4, lambda r: words(pow(num(r[0:4]) * ri, r[4], p) * MONT % p)),
    )


for _f, (_p, _base) in FIELDS.items():
    for _s, (_ni, _no, _ref) in _fp_refs(_p).items():
        _op("%s_%s" % (_f, _s), _base + FP_SUB[_s], _ni, _no, _ref, field=_f)


def _root_ref(r):
    log_n, inverse = r[0] & 0xFF, (r[0] >> 8) & 1
    w = o.fr_root_of_unity(1 << log_n)
    return words(o.fr_mont(pow(w, -1, R) if inverse else w))


_op("fr_root_of_unity", 64, 1, 4, _root_ref, device_only=True, field="fr")


def _fq2_inv(a):
    return o.FQ2_ZERO if a == o.FQ2_ZERO else o.fq2_inv(a)


def _fq2_sqrt_ref(r):
    s = o.fq2_sqrt(fq2_v(r))
    return [0] * 9 if s is None else [1] + fq2_w(s)


def _fq_sqrt_ref(r):
    a = fq_v(r)
    s = pow(a, (P + 1) // 4, P)
    return [int(s * s % P == a)] + fq_w(s)


def _fq_half_ref(r):
    a = num(r)
    return words((a if a % 2 == 0 else a + P) >> 1)        # the integer contract, for any raw a < 2^256


def _from_bytes_ref(r):
    x = num(r[0:4]) & ~(0xFF << 248) | ((num(r[0:4]) >> 248) & r[4]) << 248
    return [int(x < P)] + words(x * MONT % P)


def _glv_ref(r):
    k1, k2 = dl.glv_decompose(num(r))
    return words(abs(k1), 2) + [int(k1 < 0)] + words(abs(k2), 2) + [int(k2 < 0)]


def _mulgroup(K):
    return lambda r: sum((fq2_w(o.fq2_mul(fq2_v(r[16 * k:16 * k + 8]), fq2_v(r[16 * k + 8:16 * k + 16]))) for k in range(K)), [])


_op("fq2_mul", 70, 16, 8, lambda r: fq2_w(o.fq2_mul(fq2_v(r[:8]), fq2_v(r[8:]))))
_op("fq2_sqr", 71, 8, 8, lambda r: fq2_w(o.fq2_sqr(fq2_v(r))))
_op("fq2_inv", 72, 8, 8, lambda r: fq2_w(_fq2_inv(fq2_v(r))))
for _k in range(1, 5):
    _op("fq2_mul_group%d" % _k, 72 + _k, 16 * _k, 8 * _k, _mulgroup(_k))
_op("fq2_mul_xi", 77, 8, 8, lambda r: fq2_w(o.fq2_mul(fq2_v(r), o.XI)))
_op("fq2_conj", 78, 8, 8, lambda r: fq2_w(o.fq2_conj(fq2_v(r))))
_op("glv_phi_x_g1", 79, 4, 4, lambda r: fq_w(fq_v(r) * BETA_G1))
_op("glv_phi_x_g2", 80, 8, 8, lambda r: fq2_w(o.fq2_scalar(fq2_v(r), BETA_G2)))
_op("fq_pow_p1_4", 84, 4, 4, lambda r: fq_w(pow(fq_v(r), (P + 1) // 4, P)))
_op("fq_sqrt", 85, 4, 5, _fq_sqrt_ref)
_op("fq2_sqrt", 86, 8, 9, _fq2_sqrt_ref)
_op("fq_half", 87, 4, 4, _fq_half_ref)
_op("fq_is_larger", 88, 4, 1, lambda r: [int(o._fq_is_neg(fq_v(r)))])
_op("fq2_is_larger", 89, 8, 1, lambda r: [int(o._fq2_is_neg(fq2_v(r)))])
_op("fq_from_bytes", 90, 5, 5, _from_bytes_ref)
_op("fq6_mul", 96, 48, 24, lambda r: fq6_w(o.fq12_mul(fq12_v(r[:24]), fq12_v(r[24:]))))
_op("fq6_inv", 97, 24, 24, lambda r: fq6_w(fq12_inv(fq12_v(r))))
_op("fq6_mul_v", 98, 24, 24, lambda r: fq6_w(o.fq12_mul(fq12_v(r), W2)))
_op("fq12_mul", 99, 96, 48, lambda r: fq12_w(o.fq12_mul(fq12_v(r[:48]), fq12_v(r[48:]))))
_op("fq12_inv", 100, 48, 48, lambda r: fq12_w(fq12_inv(fq12_v(r))))
_op("fq12_conj", 101, 48, 48, lambda r: fq12_w(o.fq12_pow(fq12_v(r), P ** 6)))
_op("fq12_frob2", 102, 48, 48, lambda r: fq12_w(o.fq12_pow(fq12_v(r), P ** 2)))
_op("final_exponentiation", 103, 48, 48, lambda r: fq12_w(o.final_exponentiation(fq12_v(r))))
_op("pairing", 104, 24, 48, lambda r: fq12_w(o.pairing(G1.aff_v(r[:8]), G2.aff_v(r[8:]))))
_op("g2_frobenius_twist", 105, 16, 16, lambda r: G2.aff_w(o._frob_twist(G2.aff_v(r))))
_op("glv_decompose", 108, 4, 6, _glv_ref)

EC_SUB = dict(dbl=0, add=1, dbl_ilp=2, add_ilp=3, madd=4, dbl_affine=5, to_affine=6, mul_scalar=7,
              quad_add=8, quad_dbl=9, quad_add_fullwarp=10, quad_dbl_fullwarp=11)


def _ec_ops(gname, g: _G, base):
    W, c = g.W, g.c
    X = 4 * W
    pt = lambda ws: (lambda v: None if v[0] == "inf" else v[1:])(g.xyzz_view(ws))
    add = lambda r: g.pt_view(c.add(pt(r[:X]), pt(r[X:2 * X])))
    dbl = lambda r: g.pt_view(c.add(pt(r[:X]), pt(r[:X])))

    def madd(r):
        p = g.aff_v(r[X:X + 2 * W])
        return g.pt_view(c.add(pt(r[:X]), c.neg(p) if r[X + 2 * W] else p))

    table = dict(
        dbl=(X, X, dbl), add=(2 * X, X, add), dbl_ilp=(X, X, dbl), add_ilp=(2 * X, X, add), madd=(X + 2 * W + 1, X, madd),
        dbl_affine=(2 * W, X, lambda r: g.pt_view(c.add(g.aff_v(r), g.aff_v(r)))),
        to_affine=(X, 2 * W, lambda r: g.pt_view(pt(r))),
        mul_scalar=(X + 4, X, lambda r: g.pt_view(c.mul(pt(r[:X]), num(r[X:X + 4])))),
        quad_add=(2 * X, X, add), quad_dbl=(X, X, dbl), quad_add_fullwarp=(2 * X, X, add), quad_dbl_fullwarp=(X, X, dbl),
    )
    for s, (ni, no, ref) in table.items():
        view = g.aff_view if s == "to_affine" else g.xyzz_view
        _op("%s_%s" % (gname, s), base + EC_SUB[s], ni, no, ref, view=view, device_only=s.startswith("quad"), field=gname)


_ec_ops("g1", G1, 112)
_ec_ops("g2", G2, 128)


# ---- the corpus ------------------------------------------------------------------------------------------------------------
def _edges(p):
    e = [0, 1, 2, 3, p - 1, p - 2, p - 3, (p - 1) // 2, (p + 1) // 2, MONT % p, MONT * MONT % p, (1 << 253) % p]
    e += [(1 << (32 * i)) - 1 for i in range(1, 8)] + [1 << (32 * i) for i in range(1, 8)]
    return e


def _search(rng, p, pred, tries=200000, make=None):
    for _ in range(tries):
        a, b = make() if make else (rng.randrange(p), rng.randrange(p))
        if pred(a, b):
            return a, b
    raise AssertionError("model class not reached")


def _mul_pairs(p, rng):
    """(class, a, b) for the Montgomery product: edges, random, final subtraction, small results after it, T = p - 1."""
    out = []
    ed = _edges(p)
    out += [("edges", a, b) for a in ed for b in ed[::3]]
    out += [("random", rng.randrange(p), rng.randrange(p)) for _ in range(48)]
    for _ in range(24):
        a, b = _search(rng, p, lambda a, b: mont_pre(a * b, p) >= p)
        out.append(("final_sub", a, b))
    for v in (1, 2, 3):                 # result v reached through the subtraction: T = p + v (b = v R a^-1)
        for _ in range(2):
            def mk():
                a = rng.randrange(1, p)
                return a, v * MONT * pow(a, -1, p) % p
            a, b = _search(rng, p, lambda a, b: mont_pre(a * b, p) == p + v, make=mk)
            out.append(("result_%d_after_sub" % v, a, b))
    for _ in range(2):                  # T = p - 1: the largest value that skips the subtraction
        def mk():
            a = rng.randrange(1, p)
            return a, (p - 1) * MONT * pow(a, -1, p) % p
        a, b = _search(rng, p, lambda a, b: mont_pre(a * b, p) == p - 1, make=mk)
        out.append(("T_p_minus_1", a, b))
    return out


def _add_pairs(p, rng):
    out = [("random", rng.randrange(p), rng.randrange(p)) for _ in range(32)]
    ed = _edges(p)
    out += [("edges", a, b) for a in ed for b in ed]
    for a in (1, 2, (p - 1) // 2, p - 1, rng.randrange(p)):
        out.append(("sum_p", a, p - a))
        out.append(("sum_p_minus_1", a, p - 1 - a))
        out.append(("diff_minus_1", a - 1, a))
    out.append(("sum_2p_minus_2", p - 1, p - 1))
    for i in range(1, 8):               # a carry from limb 0 through every limb boundary below 32 i / a borrow the same way
        out.append(("carry_ripple", (1 << (32 * i)) - 1, 1))
        out.append(("borrow_ripple", 1 << (32 * i), 1))
    return out


def _inv_inputs(p):
    """One raw input per iteration count k of Fp::inv (254..507), then edges."""
    cands = list(range(1, 3000)) + [p - i for i in range(1, 3000)] + [1 << i for i in range(254)]
    cands += [p - (1 << i) for i in range(254)] + [(1 << i) - 1 for i in range(2, 254)] + [(1 << i) + 1 for i in range(1, 253)]
    cands += [p // d for d in range(2, 2000)]
    by_k = {}
    for a in cands:
        if 0 < a < p:
            by_k.setdefault(kaliski_k(a, p), a)
    return [("iter_%d" % k, a) for k, a in sorted(by_k.items())] + [("edges", 0), ("edges", p - 1), ("edges", MONT % p)]


def _fq2_mul_pairs(rng):
    """(class, a, b) as Fq2 raw pairs; the class names the redc<2> branch each coefficient reaches."""
    def cls(a, b):
        t0 = a[0] * b[0] - a[1] * b[1] + P * MONT
        t2 = a[0] * b[1] + a[1] * b[0]
        return mont_pre(t0, P) // P, mont_pre(t2, P) // P
    rnd = lambda: (rng.randrange(P), rng.randrange(P))
    out = []
    for k0 in (0, 1, 2):
        for _ in range(8):
            a, b = _search(rng, P, lambda a, b: cls(a, b)[0] == k0, make=lambda: (rnd(), rnd()))
            out.append(("c0_sub%d" % k0, a, b))
    for k1 in (0, 1):
        for _ in range(8):
            a, b = _search(rng, P, lambda a, b: cls(a, b)[1] == k1, make=lambda: (rnd(), rnd()))
            out.append(("c1_sub%d" % k1, a, b))
    for m in range(16):                 # every coefficient 0 or p - 1
        v = [P - 1 if (m >> i) & 1 else 0 for i in range(4)]
        out.append(("pm1_combo", (v[0], v[1]), (v[2], v[3])))
    out += [("zero_coeff", (0, rng.randrange(P)), rnd()), ("zero_coeff", (rng.randrange(P), 0), (0, rng.randrange(P)))]
    out += [("random", rnd(), rnd()) for _ in range(16)]
    return out


def _rand_fq12(rng, mask=range(12)):
    return tuple(rng.randrange(P) if i in mask else 0 for i in range(12))


def _tower_elems(rng, fq6: bool):
    c0 = (0, 2, 4, 6, 8, 10)            # w^0 w^2 w^4 in the oracle's basis: the Fq6 part
    out = [("random", _rand_fq12(rng, c0 if fq6 else range(12))) for _ in range(4)]
    out += [("one", o.FQ12_ONE), ("fq_subfield", (rng.randrange(P),) + (0,) * 11)]
    out += [("fq2_subfield", fq12_v(fq2_w((rng.randrange(P), rng.randrange(P))) + [0] * 40))]
    out += [("b_zero", fq12_v([rng.randrange(1 << 62) for _ in range(8)] + [0] * 8 + [rng.randrange(1 << 62) for _ in range(8)]
                              + [0] * 24))]
    out += [("a_zero", fq12_v([0] * 8 + [rng.randrange(1 << 62) for _ in range(16)] + [0] * 24))]
    out += [("c_zero", fq12_v([rng.randrange(1 << 62) for _ in range(16)] + [0] * 32))]
    if not fq6:
        out += [("c1_zero", _rand_fq12(rng, c0)), ("c0_zero", _rand_fq12(rng, (1, 3, 5, 7, 9, 11)))]
        lam, xT, yT = ((rng.randrange(P), rng.randrange(P)) for _ in range(3))
        out += [("line", o._line(lam, (xT, yT), (rng.randrange(P), rng.randrange(P))))]
    # fq12_v applied to raw words only produces values; re-check they are well-formed
    return [(c, tuple(x % P for x in f)) for c, f in out]


def _z_values(g: _G, rng):
    """z values whose raw limbs sit at the edges: raw 1, raw p - 1, raw 2^(32 i) - 1, the value 1, random."""
    raws = [1, P - 1, (1 << 64) - 1, (1 << 224) - 1, MONT % P]
    vals = [to_val(x) for x in raws] + [rng.randrange(1, P)]
    if g is G2:
        return [(v, 0) for v in vals[:3]] + [(vals[3], vals[4]), (0, vals[0]), (rng.randrange(P), rng.randrange(P))]
    return vals


def _points(g: _G, rng, n):
    return [g.c.mul(g.gen, rng.randrange(1, R)) for _ in range(n)]


def _ec_corpus(g: _G, rng):
    c = g.c
    zs = _z_values(g, rng)
    pts = _points(g, rng, 4)
    P0 = pts[0]
    rel = lambda p: [("Q=P", p, p), ("Q=-P", p, c.neg(p)), ("Q=O", p, None), ("P=O", None, p), ("Q=2P", p, c.add(p, p)),
                     ("random", p, pts[3]), ("both_O", None, None), ("Q=P+G", p, c.add(p, g.gen))]
    pairs = []
    for i, z in enumerate(zs):
        z2 = zs[(i + 1) % len(zs)]
        for cls, a, b in rel(pts[i % 3]):
            pairs.append((cls, g.xyzz_w(a, z) + g.xyzz_w(b, z2)))
    singles = [("finite", g.xyzz_w(p, z)) for p in pts for z in zs] + [("O", [0] * (4 * g.W))]
    madd = []
    for i, z in enumerate(zs):
        p = pts[i % 3]
        for cls, acc, q, neg in (("acc=p", p, p, 0), ("acc=-p", p, c.neg(p), 0), ("acc=p_negated", c.neg(p), p, 1),
                                 ("acc=-p_negated", p, p, 1), ("acc=O", None, p, i & 1), ("p=O", p, None, i & 1),
                                 ("random", p, pts[3], 0), ("random_negated", p, pts[3], 1)):
            madd.append((cls, g.xyzz_w(acc, z) + g.aff_w(q) + [neg]))
    ks = [0, 1, R - 1, R, MONT - 1, rng.randrange(R)]
    scal = [("k=%s" % ("r-1" if k == R - 1 else "r" if k == R else "2^256-1" if k == MONT - 1 else k if k < 2 else "random"),
             g.xyzz_w(p, zs[j % len(zs)]) + words(k)) for j, p in enumerate(pts[:2]) for k in ks]
    # quad_ops: eight relations per warp so the quads of one warp take different early returns in one launch
    quad_add = [(cls, g.xyzz_w(a, zs[j % len(zs)]) + g.xyzz_w(b, zs[(j + 2) % len(zs)]))
                for j in range(3) for cls, a, b in rel(pts[j])]
    quad_dbl = [(cls, g.xyzz_w(p, zs[j % len(zs)])) for j in range(3)
                for cls, p in (("finite", pts[j]), ("O", None), ("finite", pts[3]), ("O", None), ("finite", c.neg(pts[j])),
                               ("finite", g.gen), ("O", None), ("finite", pts[(j + 1) % 4]))]
    return dict(dbl=singles, add=pairs, dbl_ilp=singles, add_ilp=pairs, madd=madd,
                dbl_affine=[("finite", g.aff_w(p)) for p in pts + [g.gen, c.neg(P0)]],
                to_affine=singles, mul_scalar=scal, quad_add=quad_add, quad_dbl=quad_dbl,
                quad_add_fullwarp=quad_add, quad_dbl_fullwarp=quad_dbl)


@functools.lru_cache(maxsize=None)
def corpus() -> dict:
    """op name -> [(class, record)], deterministic."""
    rng = random.Random(20261017)
    C = {}
    for f, (p, _) in FIELDS.items():
        mp = _mul_pairs(p, rng)
        ap = _add_pairs(p, rng)
        rec2 = lambda prs: [(c, words(a) + words(b)) for c, a, b in prs]
        C[f + "_add"] = C[f + "_sub"] = rec2(ap)
        singles = [(c, words(a)) for c, a, _ in ap if c != "random"] + [("random", words(rng.randrange(p))) for _ in range(16)]
        singles += [("dbl_p_minus_1", words((p - 1) // 2)), ("dbl_p_plus_1", words((p + 1) // 2))]
        C[f + "_neg"] = C[f + "_dbl"] = singles
        for s in ("mul", "mul_ni"):
            C["%s_%s" % (f, s)] = rec2(mp)
        C[f + "_mul_wide_redc1"] = rec2(mp)
        sq = [("edges", words(a)) for a in _edges(p)] + [("random", words(rng.randrange(p))) for _ in range(16)]
        for _ in range(8):
            a, _b = _search(rng, p, lambda a, b: mont_pre(a * a, p) >= p)
            sq.append(("final_sub", words(a)))
        C[f + "_sqr"] = sq
        anyb = [MONT - 1, p, p + 1, 2 * p, MONT - p, 1 << 255, (1 << 255) + 1, 1 << 254] + [rng.randrange(p, MONT) for _ in range(8)]
        C[f + "_mul_any"] = ([("b_ge_p", words(a) + words(b)) for a in (1, p - 1, rng.randrange(p), MONT % p) for b in anyb]
                             + [("b_pow2", words(rng.randrange(p)) + words(1 << j)) for j in range(256)])
        for K in (2, 3, 4):             # the product corpus in groups of K, each group mixing classes
            flat = [(c, words(a) + words(b)) for c, a, b in mp]
            C["%s_mul_k%d" % (f, K)] = [("+".join(c for c, _ in flat[i:i + K]), sum((r for _, r in flat[i:i + K]), []))
                                        for i in range(0, len(flat) - K + 1, K)] + \
                                       [("mixed", sum((flat[(i * 37 + 11 * j) % len(flat)][1] for j in range(K)), []))
                                        for i in range(16)]
        red = [("random", words(rng.randrange(2 * p * MONT), 8)) for _ in range(16)]
        red += [("edges", words(t, 8)) for t in (0, 1, 2 * p * MONT - 1, p * MONT, p * MONT - 1, (p - 1) ** 2, MONT - 1)]
        for k in (0, 1, 2):
            for _ in range(8):
                t, _b = _search(rng, p, lambda t, b: mont_pre(t, p) // p == k, make=lambda: (rng.randrange(2 * p * MONT), 0))
                red.append(("sub%d" % k, words(t, 8)))
        C[f + "_redc2"] = red
        inv = [(c, words(a)) for c, a in _inv_inputs(p)]
        C[f + "_inv"] = inv
        C[f + "_inv_fermat"] = [x for i, x in enumerate(inv) if i % 4 == 0 or x[0] == "edges"]
        tm = [("edges", words(a)) for a in _edges(p)] + [("random", words(rng.randrange(p))) for _ in range(16)]
        C[f + "_to_mont"] = C[f + "_from_mont"] = tm
        C[f + "_from_u32"] = [("edges", [v]) for v in (0, 1, 2, 3, 1 << 31, (1 << 32) - 1)] + \
                             [("random", [rng.randrange(1 << 32)]) for _ in range(8)]
        C[f + "_pow_u64"] = [("edges", words(a) + [e]) for a in (0, 1, MONT % p, p - 1, rng.randrange(p))
                             for e in (0, 1, 2, 3, 1 << 63, M64, rng.randrange(1 << 64))]
    C["fr_root_of_unity"] = [("log_n=%d" % l, [l | inv << 8]) for inv in (0, 1) for l in range(29)]

    fq2p = _fq2_mul_pairs(rng)
    C["fq2_mul"] = [(c, fq2_raw(a) + fq2_raw(b)) for c, a, b in fq2p]
    for K in range(1, 5):
        flat = C["fq2_mul"]
        C["fq2_mul_group%d" % K] = [("+".join(c for c, _ in flat[i:i + K]), sum((r for _, r in flat[i:i + K]), []))
                                    for i in range(0, len(flat) - K + 1, K)]
    f2 = [(c, fq2_raw(a)) for c, a, _ in fq2p] + [("zero", [0] * 8), ("one", fq2_w(o.FQ2_ONE))]
    f2 += [("c1_zero", fq2_raw((rng.randrange(P), 0))), ("c0_zero", fq2_raw((0, rng.randrange(P))))]
    C["fq2_sqr"] = C["fq2_inv"] = C["fq2_mul_xi"] = C["fq2_conj"] = C["glv_phi_x_g2"] = f2
    C["glv_phi_x_g1"] = [("edges", words(a)) for a in _edges(P)] + [("random", words(rng.randrange(P))) for _ in range(8)]

    # square roots: values chosen by residuosity, written raw
    sqv = []
    for _ in range(8):
        s = rng.randrange(1, P)
        sqv += [("residue", s * s % P), ("non_residue", -s * s % P)]
    sqv += [("zero", 0), ("one", 1), ("minus_one", P - 1)]
    C["fq_pow_p1_4"] = C["fq_sqrt"] = [(c, fq_w(v)) for c, v in sqv]
    f2s = []
    for _ in range(4):
        s, t = rng.randrange(1, P), rng.randrange(1, P)
        f2s += [("c1_zero_residue", (s * s % P, 0)), ("c1_zero_non_residue", (-s * s % P, 0)),
                ("c0_zero", (0, s)), ("square", o.fq2_sqr((s, t)))]
        while True:
            x = (rng.randrange(P), rng.randrange(P))
            if o.fq2_sqrt(x) is None:
                f2s.append(("non_square", x))
                break
    f2s += [("zero", (0, 0)), ("minus_one", (P - 1, 0))]
    C["fq2_sqrt"] = [(c, fq2_w(v)) for c, v in f2s]
    half = [("even", words(2 * rng.randrange(P // 2))) for _ in range(4)] + [("odd", words(2 * rng.randrange(P // 2) + 1)) for _ in range(4)]
    half += [("edges", words(a)) for a in (0, 1, P - 1, P - 2)]
    half += [("noncanonical_odd_carry", words(a)) for a in (MONT - 1, MONT - P, MONT - P + 2, (MONT - 1) - 2 * rng.randrange(P // 2))]
    C["fq_half"] = half
    lv = [("half_minus", (P - 1) // 2), ("half_plus", (P + 1) // 2), ("zero", 0), ("one", 1), ("minus_one", P - 1)]
    lv += [("random", rng.randrange(P)) for _ in range(8)]
    C["fq_is_larger"] = [(c, fq_w(v)) for c, v in lv]
    l2 = [("c1_zero_small_c0", (v, 0)) for v in (1, 5, (P - 1) // 2)] + [("c1_zero_large_c0", (v, 0)) for v in (P - 1, (P + 1) // 2)]
    l2 += [("c1_small", (rng.randrange(P), v)) for v in (1, (P - 1) // 2)] + [("c1_large", (rng.randrange(P), v)) for v in (P - 1, (P + 1) // 2)]
    l2 += [("c1_small_c0_large", (P - 1, 1)), ("c1_large_c0_small", (1, P - 1)), ("zero", (0, 0))]
    C["fq2_is_larger"] = [(c, fq2_w(v)) for c, v in l2]
    fb = []
    for x in (0, 1, P - 1, P, P + 1, (1 << 254) - 1, 1 << 254, 1 << 255, MONT - 1, rng.randrange(P)):
        for mask in (0xFF, 0x3F):
            xm = x & ~(0xFF << 248) | ((x >> 248) & mask) << 248
            fb.append(("lt_p" if xm < P else "ge_p", words(x) + [mask]))
    C["fq_from_bytes"] = fb

    e6 = _tower_elems(rng, True)
    e12 = _tower_elems(rng, False)
    C["fq6_mul"] = [(ca + "*" + cb, fq6_w(a) + fq6_w(b)) for i, (ca, a) in enumerate(e6) for cb, b in e6[i::3]]
    C["fq6_inv"] = [(c, fq6_w(a)) for c, a in e6] + [("zero", [0] * 24)]
    C["fq6_mul_v"] = [(c, fq6_w(a)) for c, a in e6]
    C["fq12_mul"] = [(ca + "*" + cb, fq12_w(a) + fq12_w(b)) for i, (ca, a) in enumerate(e12) for cb, b in e12[i::4]]
    C["fq12_inv"] = [(c, fq12_w(a)) for c, a in e12]
    C["fq12_conj"] = [(c, fq12_w(a)) for c, a in e12[:6]]
    C["fq12_frob2"] = [(c, fq12_w(a)) for c, a in e12]
    C["final_exponentiation"] = [(c, fq12_w(a)) for c, a in e12[:2]] + [("one", fq12_w(o.FQ12_ONE))] + \
                                [(c, fq12_w(a)) for c, a in e12 if c == "line"]
    a, b = rng.randrange(1, R), rng.randrange(1, R)
    gp, hq = o.G1.mul(o.G1_GEN, a), o.G2.mul(o.G2_GEN, b)
    pairs = [("generators", o.G1_GEN, o.G2_GEN), ("random", gp, hq), ("P=O", None, hq), ("Q=O", gp, None),
             ("-P", o.G1.neg(gp), hq), ("-Q", gp, o.G2.neg(hq))]
    C["pairing"] = [(c, G1.aff_w(x) + G2.aff_w(y)) for c, x, y in pairs]
    C["g2_frobenius_twist"] = [("generator", G2.aff_w(o.G2_GEN)), ("random", G2.aff_w(hq)), ("-Q", G2.aff_w(o.G2.neg(hq)))]

    lam = dl.LAMBDA
    ks = [("edges", k) for k in (0, 1, lam, R - 1, R - lam)]
    ks += [("designed_halves", dl.glv_compose(k1, k2)) for k1, k2 in dl.glv_designed_halves()]
    ks += [("extremes", k) for k in dl.glv_extremes()]
    ks += [("random", rng.randrange(R)) for _ in range(16)]
    C["glv_decompose"] = [(c, words(k)) for c, k in ks]

    for gname, g in (("g1", G1), ("g2", G2)):
        for s, recs in _ec_corpus(g, rng).items():
            C["%s_%s" % (gname, s)] = recs
    for name, recs in C.items():
        op = OPS[name]
        assert recs and all(len(r) == op.n_in for _, r in recs), name
    assert set(C) == set(OPS), set(OPS) ^ set(C)
    return C


def fq2_raw(a) -> List[int]:
    """An Fq2 given by its raw Montgomery coefficients (no conversion)."""
    return words(a[0]) + words(a[1])


def expected(name: str) -> list:
    op = OPS[name]
    return [op.ref(r) for _, r in corpus()[name]]


def mismatches(name: str, outs) -> List[str]:
    """Compare device / host output records with the exact answers: one line per failing record (class, input in hex)."""
    op = OPS[name]
    bad = []
    for (cls, rec), out, want in zip(corpus()[name], outs, expected(name)):
        got = op.view([int(w) for w in out])
        if got != want:
            bad.append("%s [%s] in=%s got=%s want=%s" % (name, cls, " ".join("%016x" % w for w in rec), got, want))
    return bad
