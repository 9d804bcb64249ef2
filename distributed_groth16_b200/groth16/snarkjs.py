"""snarkjs's Groth16 JSON files on the device: proof.json, public.json and verification_key.json (formats.py reads and
writes the text), and the witness check of snarkjs `wtns check`.

Coordinates cross between the JSON's decimals and the device's Montgomery points through ffjavascript's uncompressed
encoding (b200zk_points_encode_dev / b200zk_points_decode_dev, fmt 0: big-endian, G2 as c1 || c0, infinity 0x40), so no
field arithmetic runs on the host.  Decoding gives snarkjs's well-formedness checks: canonical coordinates, on the curve,
and for G2 in the order-r subgroup.  vk_alphabeta_12 comes from b200zk_vk_alphabeta_12, the satisfaction check from
b200zk_r1cs_check_dev."""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field

import numpy as np

from .. import formats
from ..ark_serialize import ArkVerifyingKey, deserialize_proof
from ..context import Net, _as_u64, _ptr, c_vp
from . import phase1

_INF = b"\x40"


def _be(v: int) -> bytes:
    return int(v).to_bytes(32, "big")


def _encode_ints(points, g2: bool) -> bytes:
    """Coordinates as ints (None = infinity) -> ffjavascript uncompressed encodings, back to back."""
    w = 128 if g2 else 64
    out = []
    for p in points:
        if p is None:
            out.append(_INF + bytes(w - 1))
        elif g2:
            out.append(_be(p[0][1]) + _be(p[0][0]) + _be(p[1][1]) + _be(p[1][0]))
        else:
            out.append(_be(p[0]) + _be(p[1]))
    return b"".join(out)


def _decode_ints(enc: bytes, g2: bool) -> list:
    """The inverse of _encode_ints on the device's encodings."""
    w = 128 if g2 else 64
    ints = lambda b: int.from_bytes(b, "big")
    out = []
    for i in range(0, len(enc), w):
        e = enc[i:i + w]
        if e[0] & 0x40:
            out.append(None)
        elif g2:
            out.append(((ints(e[32:64]), ints(e[0:32])), (ints(e[96:128]), ints(e[64:96]))))
        else:
            out.append((ints(e[0:32]), ints(e[32:64])))
    return out


def points_to_ints(net: Net, points, g2: bool = False) -> list:
    """Affine Montgomery points (host u64 (n, 8 | 16) or CUDA int64) -> canonical coordinates as ints, encoded on the device."""
    w = 16 if g2 else 8
    pts = points if hasattr(points, "data_ptr") else net.to_device(_as_u64(points, w).reshape(-1, w))
    if int(pts.shape[0]) == 0:
        return []
    return _decode_ints(phase1.points_encode(net, pts, g2=g2).cpu().numpy().tobytes(), g2)


def points_from_ints(net: Net, points, g2: bool = False) -> np.ndarray:
    """Coordinates as ints (each < q; None = infinity) -> host u64 (n, 8 | 16) affine Montgomery points, decoded on the
    device.  Raises phase1.InvalidEncodings (a FormatError) for a point off the curve or, on G2, outside the order-r
    subgroup."""
    w = 16 if g2 else 8
    if not points:
        return np.zeros((0, w), dtype=np.uint64)
    enc = np.frombuffer(_encode_ints(points, g2), dtype=np.uint8).copy()
    return phase1.points_decode(net, enc, g2=g2, compressed=False, check_subgroup=g2).cpu().numpy().view(np.uint64)


def _limbs_to_int(row) -> int:
    return sum(int(x) << (64 * i) for i, x in enumerate(np.asarray(row, dtype=np.uint64).reshape(-1)))


def proof_to_json(net: Net, proof_bytes: bytes) -> str:
    """The 128 compressed bytes of a proof (ark-serialize) -> snarkjs's proof.json."""
    a, b, c = deserialize_proof(net, bytes(proof_bytes), check_subgroup=False)
    (pa, pc), (pb,) = points_to_ints(net, np.stack([a, c])), points_to_ints(net, b.reshape(1, 16), g2=True)
    return formats.write_proof_json(formats.SnarkjsProof(pa, pb, pc))


def public_to_json(public_limbs) -> str:
    """Public inputs as canonical limbs (n, 4) -> snarkjs's public.json."""
    return formats.write_public_json([_limbs_to_int(r) for r in np.asarray(public_limbs, dtype=np.uint64).reshape(-1, 4)])


def alphabeta_12(net: Net, alpha_g1, beta_g2) -> list:
    """snarkjs's vk_alphabeta_12 for Montgomery alpha (8 limbs) and beta (16 limbs): 2 x 3 x 2 canonical Fq ints."""
    out = np.zeros(48, dtype=np.uint64)
    net.check(net._lib.b200zk_vk_alphabeta_12(net._h, _ptr(_as_u64(alpha_g1, 0).reshape(-1)), _ptr(_as_u64(beta_g2, 0).reshape(-1)),
                                              _ptr(out)))
    v = [_limbs_to_int(out[4 * i:4 * i + 4]) for i in range(12)]
    return [[[v[6 * h + 2 * k], v[6 * h + 2 * k + 1]] for k in range(3)] for h in range(2)]


def vk_from_zkey(net: Net, zkey: formats.ZKey) -> formats.SnarkjsVerificationKey:
    """The verification key snarkjs `zkey export verificationkey` exports from a zkey."""
    (alpha,) = points_to_ints(net, zkey.alpha_g1.reshape(1, 8))
    beta, gamma, delta = points_to_ints(net, np.stack([zkey.beta_g2, zkey.gamma_g2, zkey.delta_g2]), g2=True)
    return formats.SnarkjsVerificationKey(zkey.n_public, alpha, beta, gamma, delta, alphabeta_12(net, zkey.alpha_g1, zkey.beta_g2),
                                          points_to_ints(net, zkey.ic))


def read_vk_json(net: Net, text) -> ArkVerifyingKey:
    """verification_key.json -> ArkVerifyingKey for verify.verify_proof.  Raises FormatError for a malformed file or a point
    that does not decode.  vk_alphabeta_12 is read but not used, as in snarkjs's verifier."""
    return _ark_vk(net, formats.read_vk_json(text))


def _ark_vk(net: Net, vk: formats.SnarkjsVerificationKey) -> ArkVerifyingKey:
    g1 = points_from_ints(net, [vk.alpha_1] + list(vk.ic))
    g2 = points_from_ints(net, [vk.beta_2, vk.gamma_2, vk.delta_2], g2=True)
    return ArkVerifyingKey(g1[0], g2[0], g2[1], g2[2], g1[1:])


def verify_json(net: Net, vk_text, public_text, proof_text) -> bool:
    """snarkjs `groth16 verify`.  FormatError for text that is not a well-formed file of its kind (see formats.read_*_json) or
    a verification-key point that does not decode.  False where snarkjs's publicInputsAreValid / isWellConstructed reject
    (a public count other than nPublic, a signal >= r, a proof point off the curve or outside the G2 subgroup) and when
    the pairing check fails."""
    from .verify import verify_proof
    vk = formats.read_vk_json(vk_text)
    public = formats.read_public_json(public_text)
    proof = formats.read_proof_json(proof_text)
    avk = _ark_vk(net, vk)
    if len(public) != vk.n_public or any(v >= formats.FR_MODULUS for v in public):
        return False
    try:
        (a, c), (b,) = points_from_ints(net, [proof.pi_a, proof.pi_c]), points_from_ints(net, [proof.pi_b], g2=True)
    except phase1.InvalidEncodings:
        return False
    x = []
    if public:
        limbs = np.array([[(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] for v in public], dtype=np.uint64)
        x = net.fr_convert(net.to_device(limbs), to_mont=True).cpu().numpy().view(np.uint64)
    return verify_proof(net, avk, x, (a, b, c))


# ---- snarkjs `wtns check` ----------------------------------------------------------------------------------------------------

@dataclass
class WtnsCheckReport:
    """ok: every check holds.  n_failed / first_failed: the failing constraints and the lowest of them (n_constraints when
    none fails or when the witness was rejected before the constraints were evaluated).  lines: one per failure."""
    ok: bool
    n_failed: int
    first_failed: int
    lines: list = field(default_factory=list)


def r1cs_check(net: Net, csr, w, n_constraints: int):
    """b200zk_r1cs_check_dev: csr = three (row_ptr, col, val) triples of CUDA tensors (val Montgomery), w a CUDA (n, 4)
    Montgomery tensor -> (n_failed, first_failed)."""
    args = []
    for ptr, col, val in csr:
        args += [c_vp(t.data_ptr()) if t is not None and t.numel() else None for t in (ptr, col, val)]
    n_failed, first = ctypes.c_uint64(0), ctypes.c_uint64(0)
    net.check(net._lib.b200zk_r1cs_check_dev(net._h, 0, *args, int(n_constraints), c_vp(w.data_ptr()) if w is not None else None,
                                             ctypes.byref(n_failed), ctypes.byref(first)))
    return int(n_failed.value), int(first.value)


_R_LIMBS = np.array([(formats.FR_MODULUS >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


def _not_below_r(w: np.ndarray) -> np.ndarray:
    """Per row of canonical limbs (n, 4): value >= r."""
    ge, eq = np.zeros(w.shape[0], dtype=bool), np.ones(w.shape[0], dtype=bool)
    for i in (3, 2, 1, 0):
        ge |= eq & (w[:, i] > _R_LIMBS[i])
        eq &= w[:, i] == _R_LIMBS[i]
    return ge | eq


def check_witness(net: Net, r1: formats.R1CS, w: np.ndarray) -> WtnsCheckReport:
    """The checks of snarkjs `wtns check` on a parsed circuit and canonical witness limbs (n, 4)."""
    nc = r1.n_constraints
    fail = lambda line: WtnsCheckReport(False, 0, nc, [line])
    if w.shape[0] != r1.n_wires:
        return fail("the witness has %d entries, the circuit has %d wires" % (w.shape[0], r1.n_wires))
    if w.shape[0] and _limbs_to_int(w[0]) != 1:
        return fail("w[0] = %d, the constant wire must be 1" % _limbs_to_int(w[0]))
    big = np.flatnonzero(_not_below_r(w))
    if big.size:
        i = int(big[0])
        return fail("%d witness entries are not below r, the first is w[%d] = %d" % (big.size, i, _limbs_to_int(w[i])))
    csr = [formats.coo_to_csr(r1.rows[k], r1.cols[k], r1.vals[k], nc) for k in range(3)]
    to_mont = lambda v: net.fr_convert(net.to_device(v), to_mont=True) if v.shape[0] else None
    dev = [(net.to_device(p.view(np.int32)), net.to_device(c.view(np.int32)) if c.size else None, to_mont(v)) for p, c, v in csr]
    n_failed, first = r1cs_check(net, dev, to_mont(w), nc)
    if not n_failed:
        return WtnsCheckReport(True, 0, nc, [])
    wi = lambda j: _limbs_to_int(w[j])
    dots = []
    for ptr, col, val in csr:
        lo, hi = int(ptr[first]), int(ptr[first + 1])
        dots.append(sum(_limbs_to_int(val[k]) * wi(int(col[k])) for k in range(lo, hi)) % formats.FR_MODULUS)
    return WtnsCheckReport(False, n_failed, first, [
        "constraint %d does not hold: <A,w> = %d, <B,w> = %d, <C,w> = %d (%d of %d constraints fail)"
        % (first, dots[0], dots[1], dots[2], n_failed, nc)])
