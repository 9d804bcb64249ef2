"""Pure-Python restatement of the circuit hash (csHash) of snarkjs `zkey new` (TEST INFRASTRUCTURE ONLY), the yardstick of
distributed_groth16_b200.groth16.cshash.  It has its own reading of the zkey, its own encodings and its own group law.

  csHash = Blake2b-512( U(alpha_1) U(beta_1) U(beta_2) U(gamma_2) U(delta_1) U(delta_2)
                        u32(#IC) U(IC) u32(n - 1) U(H) u32(#C) U(C) u32(n_vars) U(A) u32(n_vars) U(B1) u32(n_vars) U(B2) )

with U = ffjavascript toRprUncompressed (big-endian x || y, G2 as x.c1 x.c0 y.c1 y.c0, infinity 0x40 then zeros), u32 a
big-endian count and H_i = tau^(n+i) G1 - tau^i G1, i < n - 1.

The H points come either from a ceremony's tau powers (h_from_tau, by subtraction) or, for a key with no contributions,
from its own section 9 (h_from_lagrange).  Section 9 holds h_k = L^(2n)_(2k+1)(tau) G1, the odd Lagrange points of the
2n domain; tau^i (tau^n - 1) has degree < 2n, vanishes on the even points and is -2 w_2n^(i (2k+1)) at w_2n^(2k+1), so

  H_i = -2 w_2n^i sum_k w_n^(i k) h_k,

a forward DFT of the h_k over G1 followed by one scalar per point.  The DFT runs in two passes of independent column /
row transforms of size sqrt(n) (the four-step split) on a process pool, on Jacobian integer points."""
import hashlib
import os
import struct
from concurrent.futures import ProcessPoolExecutor

from oracle import bn254 as o

Q, R = o.P, o.R
_RINV_Q = pow(1 << 256, -1, Q)
_INF = (1, 1, 0)


# ---- reading and encoding ----------------------------------------------------------------------------------------------
def _fq(buf, off) -> int:
    return int.from_bytes(buf[off:off + 32], "little") * _RINV_Q % Q


def u_g1_bytes(buf, off) -> bytes:
    """U of the Montgomery little-endian G1 point at buf[off:off + 64]."""
    if not any(buf[off:off + 64]):
        return b"\x40" + bytes(63)
    return _fq(buf, off).to_bytes(32, "big") + _fq(buf, off + 32).to_bytes(32, "big")


def u_g2_bytes(buf, off) -> bytes:
    if not any(buf[off:off + 128]):
        return b"\x40" + bytes(127)
    return b"".join(_fq(buf, off + 32 * k).to_bytes(32, "big") for k in (1, 0, 3, 2))


def u_g1(pt) -> bytes:
    """U of an oracle G1 point (x, y) or None."""
    return b"\x40" + bytes(63) if pt is None else pt[0].to_bytes(32, "big") + pt[1].to_bytes(32, "big")


def zkey_sections(zkey: bytes) -> dict:
    assert zkey[:4] == b"zkey"
    _v, n = struct.unpack_from("<II", zkey, 4)
    off, out = 12, {}
    for _ in range(n):
        sid, ln = struct.unpack_from("<IQ", zkey, off)
        out[sid] = zkey[off + 12:off + 12 + ln]
        off += 12 + ln
    return out


def cs_hash(zkey: bytes, h_points) -> bytes:
    """The csHash of a zkey's sections 2, 3 and 5-8 with the given H points (oracle G1 points, n - 1 of them)."""
    s = zkey_sections(zkey)
    hdr = s[2]
    n_vars, n_public, n = struct.unpack_from("<III", hdr, 72)
    assert len(h_points) == n - 1
    h = hashlib.blake2b(digest_size=64)
    off = 84
    for g2 in (False, False, True, True, False, True):        # alpha_1 beta_1 beta_2 gamma_2 delta_1 delta_2
        h.update(u_g2_bytes(hdr, off) if g2 else u_g1_bytes(hdr, off))
        off += 128 if g2 else 64

    def section(sid, count, g2=False):
        w = 128 if g2 else 64
        assert len(s[sid]) == count * w
        h.update(struct.pack(">I", count))
        for i in range(count):
            h.update(u_g2_bytes(s[sid], i * w) if g2 else u_g1_bytes(s[sid], i * w))

    section(3, n_public + 1)
    h.update(struct.pack(">I", n - 1))
    for p in h_points:
        h.update(u_g1(p))
    section(8, n_vars - n_public - 1)
    section(5, n_vars)
    section(6, n_vars)
    section(7, n_vars, True)
    return h.digest()


# ---- H by subtraction --------------------------------------------------------------------------------------------------
def h_from_tau(tau_g1: bytes, n: int) -> list:
    """H_i = tau^(n+i) G1 - tau^i G1 (i < n - 1) from the bytes of ptau section 2."""
    pt = lambda i: None if not any(tau_g1[64 * i:64 * i + 64]) else (_fq(tau_g1, 64 * i), _fq(tau_g1, 64 * i + 32))
    return [o.G1.add(pt(n + i), o.G1.neg(pt(i))) for i in range(n - 1)]


# ---- H from section 9: a DFT over G1 on Jacobian integers --------------------------------------------------------------
def _dbl(p):
    X, Y, Z = p
    if Z == 0:
        return p
    A, B = X * X % Q, Y * Y % Q
    C = B * B % Q
    D = 2 * ((X + B) * (X + B) - A - C) % Q
    E = 3 * A
    F = E * E % Q
    X3 = (F - 2 * D) % Q
    return X3, (E * (D - X3) - 8 * C) % Q, 2 * Y * Z % Q


def _add(p, q):
    X1, Y1, Z1 = p
    X2, Y2, Z2 = q
    if Z1 == 0:
        return q
    if Z2 == 0:
        return p
    Z1Z1, Z2Z2 = Z1 * Z1 % Q, Z2 * Z2 % Q
    U1, U2 = X1 * Z2Z2 % Q, X2 * Z1Z1 % Q
    S1, S2 = Y1 * Z2 * Z2Z2 % Q, Y2 * Z1 * Z1Z1 % Q
    H, r = (U2 - U1) % Q, 2 * (S2 - S1) % Q
    if H == 0:
        return _dbl(p) if r == 0 else _INF
    I = 4 * H * H % Q
    J, V = H * I % Q, U1 * I % Q
    X3 = (r * r - J - 2 * V) % Q
    return X3, (r * (V - X3) - 2 * S1 * J) % Q, ((Z1 + Z2) * (Z1 + Z2) - Z1Z1 - Z2Z2) * H % Q


def _neg(p):
    return p[0], (-p[1]) % Q, p[2]


def _mul(p, k: int):
    """k p, k in [0, r), with 4-bit windows."""
    k %= R
    if k == 0 or p[2] == 0:
        return _INF
    if k == 1:
        return p
    tab = [_INF, p]
    for _ in range(14):
        tab.append(_add(tab[-1], p))
    acc = _INF
    for sh in range(252, -1, -4):
        for _ in range(4):
            acc = _dbl(acc)
        d = (k >> sh) & 15
        if d:
            acc = _add(acc, tab[d])
    return acc


def _dft(a: list, w: int) -> list:
    """A_i = sum_j w^(i j) a_j over Jacobian points, radix-2 in place after a bit reversal."""
    m = len(a)
    lg = m.bit_length() - 1
    a = [a[int(format(i, "0%db" % lg)[::-1], 2) if lg else 0] for i in range(m)]
    length = 2
    while length <= m:
        wl, half = pow(w, m // length, R), length // 2
        tw = [pow(wl, j, R) for j in range(half)]
        for start in range(0, m, length):
            for j in range(half):
                u, v = a[start + j], a[start + j + half]
                v = _mul(v, tw[j]) if j else v
                a[start + j], a[start + j + half] = _add(u, v), _add(u, _neg(v))
        length <<= 1
    return a


def _to_affine(p):
    X, Y, Z = p
    if Z == 0:
        return None
    zi = pow(Z, Q - 2, Q)
    zi2 = zi * zi % Q
    return X * zi2 % Q, Y * zi2 * zi % Q


def _column(args):
    """Pass 1 for column k1: the size-n2 DFT of x[k1 + n1 k2], then times w^(i2 k1)."""
    col, k1, w, n1 = args
    out = _dft(col, pow(w, n1, R))
    return [_mul(p, pow(w, i2 * k1, R)) if i2 * k1 else p for i2, p in enumerate(out)]


def _row(args):
    """Pass 2 for row i2: the size-n1 DFT over k1, output i = i2 + n2 i1, times -2 w_2n^i; affine."""
    row, i2, w, w2n, n2 = args
    out = _dft(row, pow(w, n2, R))
    return [_to_affine(_mul(p, (-2 * pow(w2n, i2 + n2 * i1, R)) % R)) for i1, p in enumerate(out)]


def h_from_lagrange(h_query, workers: int | None = None) -> list:
    """H_0 .. H_(n-2) (oracle G1 points) from the n points of zkey section 9 (oracle G1 points or None)."""
    n = len(h_query)
    lg = n.bit_length() - 1
    assert n == 1 << lg and lg >= 1
    n1 = 1 << (lg // 2)
    n2 = n // n1
    w2n = o.fr_root_of_unity(2 * n)
    w = w2n * w2n % R
    x = [_INF if p is None else (p[0], p[1], 1) for p in h_query]
    workers = workers or os.cpu_count() or 1
    with ProcessPoolExecutor(max_workers=workers) as ex:
        cols = list(ex.map(_column, [(x[k1::n1], k1, w, n1) for k1 in range(n1)], chunksize=1))
        rows = list(ex.map(_row, [([cols[k1][i2] for k1 in range(n1)], i2, w, w2n, n2) for i2 in range(n2)], chunksize=1))
    out = [None] * n
    for i2, r in enumerate(rows):
        for i1, p in enumerate(r):
            out[i2 + n2 * i1] = p
    return out[:n - 1]
