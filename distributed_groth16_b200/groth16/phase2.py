"""Phase 2 of a Groth16 ceremony on a .zkey: snarkjs `zkey contribute`, `zkey beacon` and `zkey verify` on the GPU.

`zkey new` (circom.zkey_new) makes a key with gamma = delta = 1.  Anyone who knows delta can move the public-input terms
of a proof into its private part, so the reference's scripts/phase2_proving_key.sh never proves with such a key: it runs
`zkey contribute`, `zkey verify`, `zkey beacon` and `zkey verify` first.  A contribution with secret x

  * multiplies delta_1, delta_2 by x and every point of the L (section 8) and H (section 9) queries by x^-1 -- the data-
    parallel step, b200zk_points_scale_dev on the device;
  * appends a record to section 10 (formats.Contribution): deltaAfter = the new delta_1, a proof of knowledge of x
    (g1_s, g1_sx = x g1_s, g2_spx = x hashToG2(transcript)) and the transcript that binds it to the earlier records.

Verification rebuilds the initial key from the r1cs and the Powers-of-Tau file, checks every record with same-ratio
pairings (b200zk_groth16_verify with one pairing pair per side) and the L / H sections with random linear combinations
(the G1 MSM); H is checked in the tau basis, so that a key imported from a bellman MPC-params file (groth16/bellman.py),
which has infinity in the one tau component the prover never uses, verifies too (_check_h).

Hashing and transcript (restated from snarkjs zkey_utils / misc and ffjavascript; this module is the one place that holds
them):
  * U(P) = ffjavascript toRprUncompressed: canonical big-endian x || y; G2 as x.c1 || x.c0 || y.c1 || y.c0; infinity is
    0x40 followed by zeros.  hashPubKey(c) = U(deltaAfter) || U(g1_s) || U(g1_sx) || U(g2_spx) || transcript.
  * transcript_j = Blake2b-512(csHash || hashPubKey(c_1) .. hashPubKey(c_{j-1}) || U(g1_s) || U(g1_sx)); the printed
    contribution hash is Blake2b-512(hashPubKey(c_j)).
  * hashToG2(t): ffjavascript's ChaCha seeded with the 8 big-endian u32 words of t[:32], then G2.fromRng.
  * F.fromRng: n64 = 4 u64 words (each hi word first, nextU64 = hi 2^32 + lo), word i at bit 64 i, masked to the
    modulus' bit length, values >= the modulus rejected; the result is read as a Montgomery value (element = v R^-1).
    Fq2.fromRng draws c0 then c1.
  * G.fromRng: repeat { x = F.fromRng; greatest = nextU32 & 1 } until x^3 + b is a square; y = sqrt, negated unless
    "y is the larger of (y, -y)" equals greatest (the ark-serialize flag of the codec: Fq2 compares c1 first); then
    times the cofactor (1 on G1, the twist cofactor on G2).
  * rngFromBeaconParams(h, e): SHA-256 iterated 2^e times on h, the 8 big-endian words of the result seed the ChaCha;
    then x = Fr.fromRng and g1_s = G1.fromRng.
Unpinned: none of this has been run against snarkjs itself (no snarkjs and no snarkjs-contributed zkey were at hand); it
agrees with the repository's own Python restatement (tests/phase2_oracle.py) only.  The ChaCha core is pinned to RFC 7539
ChaCha20 (key = the seed words, counter 0, nonce 0)."""
from __future__ import annotations

import ctypes
import hashlib
import os
import struct
from dataclasses import dataclass, field

import numpy as np

from .. import _native, formats
from .._native import c_vp
from ..context import _as_u64, _ptr

Q = formats.FQ_MODULUS
R = formats.FR_MODULUS
G2_COFACTOR = 21888242871839275222246405745257275088844257914179612981679871602714643921549
_RINV_Q = pow(1 << 256, -1, Q)
_RINV_R = pow(1 << 256, -1, R)
_MASK254 = (1 << 254) - 1                      # both moduli are 254-bit
_HDR_DELTA = 4 + 32 + 4 + 32 + 12 + 64 + 64 + 128 + 128      # byte offset of delta_1 in the header section (2)
_CANDIDATES = 16                               # fromRng candidates decompressed per device call


# ---- ffjavascript's ChaCha and fromRng ---------------------------------------------------------------------------------
def _rotl(v, c):
    return ((v << c) & 0xFFFFFFFF) | (v >> (32 - c))


def _quarter(s, a, b, c, d):
    s[a] = (s[a] + s[b]) & 0xFFFFFFFF; s[d] = _rotl(s[d] ^ s[a], 16)
    s[c] = (s[c] + s[d]) & 0xFFFFFFFF; s[b] = _rotl(s[b] ^ s[c], 12)
    s[a] = (s[a] + s[b]) & 0xFFFFFFFF; s[d] = _rotl(s[d] ^ s[a], 8)
    s[c] = (s[c] + s[d]) & 0xFFFFFFFF; s[b] = _rotl(s[b] ^ s[c], 7)


class ChaCha:
    """ffjavascript's ChaCha RNG: ChaCha20 blocks (10 double rounds) of the state constants || 8 seed words || a 32-bit
    block counter from 0 || three zero words, read one u32 at a time."""

    def __init__(self, seed):
        seed = [int(w) & 0xFFFFFFFF for w in seed]
        if len(seed) != 8:
            raise ValueError("ChaCha seed must be 8 u32 words")
        self._state = [0x61707865, 0x3320646E, 0x79622D32, 0x6B206574] + seed + [0, 0, 0, 0]
        self._buf, self._idx = [], 16

    @classmethod
    def from_hash(cls, h: bytes) -> "ChaCha":
        """Seeded with the 8 big-endian u32 words of h[:32] (snarkjs hashToG2, rngFromBeaconParams)."""
        return cls(struct.unpack(">8I", bytes(h[:32])))

    def _update(self):
        x = list(self._state)
        for _ in range(10):
            _quarter(x, 0, 4, 8, 12); _quarter(x, 1, 5, 9, 13); _quarter(x, 2, 6, 10, 14); _quarter(x, 3, 7, 11, 15)
            _quarter(x, 0, 5, 10, 15); _quarter(x, 1, 6, 11, 12); _quarter(x, 2, 7, 8, 13); _quarter(x, 3, 4, 9, 14)
        self._buf = [(a + b) & 0xFFFFFFFF for a, b in zip(x, self._state)]
        self._idx = 0
        self._state[12] = (self._state[12] + 1) & 0xFFFFFFFF
        if self._state[12] == 0:
            self._state[13] = (self._state[13] + 1) & 0xFFFFFFFF

    def next_u32(self) -> int:
        if self._idx == 16:
            self._update()
        v = self._buf[self._idx]
        self._idx += 1
        return v

    def next_u64(self) -> int:
        hi = self.next_u32()
        return (hi << 32) | self.next_u32()

    def next_bool(self) -> bool:
        return (self.next_u32() & 1) == 1

    def snapshot(self):
        """The position in the stream, for restore(): the block counter, the current block and the index into it."""
        return list(self._state), self._buf, self._idx

    def restore(self, snap) -> None:
        state, buf, idx = snap
        self._state, self._buf, self._idx = list(state), buf, idx


def field_from_rng(rng: ChaCha, modulus: int) -> int:
    """F.fromRng: the Montgomery REPRESENTATION v of the drawn element (the element itself is v R^-1 mod modulus)."""
    while True:
        v = 0
        for i in range(4):
            v |= rng.next_u64() << (64 * i)
        v &= _MASK254
        if v < modulus:
            return v


def rng_from_beacon(beacon_hash: bytes, num_iterations_exp: int) -> ChaCha:
    """snarkjs rngFromBeaconParams: SHA-256 iterated 2^e times on the host (out of reach for large e)."""
    h = bytes(beacon_hash)
    for _ in range(1 << num_iterations_exp):
        h = hashlib.sha256(h).digest()
    return ChaCha.from_hash(h)


# ---- canonical encodings and the transcript ----------------------------------------------------------------------------
def _fq(limbs) -> int:
    """Montgomery limbs (4 u64) -> canonical Fq integer.  Host arithmetic on a handful of record points only."""
    v = 0
    for i, w in enumerate(np.asarray(limbs, dtype=np.uint64).reshape(-1)[:4]):
        v |= int(w) << (64 * i)
    return v * _RINV_Q % Q


def u_g1(p) -> bytes:
    """ffjavascript toRprUncompressed of a G1 point (8 Montgomery limbs)."""
    p = np.asarray(p, dtype=np.uint64).reshape(-1)
    if not p.any():
        return b"\x40" + bytes(63)
    return _fq(p[:4]).to_bytes(32, "big") + _fq(p[4:8]).to_bytes(32, "big")


def u_g2(p) -> bytes:
    """ffjavascript toRprUncompressed of a G2 point (16 Montgomery limbs x.c0 x.c1 y.c0 y.c1): x.c1 x.c0 y.c1 y.c0."""
    p = np.asarray(p, dtype=np.uint64).reshape(-1)
    if not p.any():
        return b"\x40" + bytes(127)
    return b"".join(_fq(p[4 * k:4 * k + 4]).to_bytes(32, "big") for k in (1, 0, 3, 2))


def hash_pub_key(c: formats.Contribution) -> bytes:
    return u_g1(c.delta_after) + u_g1(c.g1_s) + u_g1(c.g1_sx) + u_g2(c.g2_spx) + bytes(c.transcript)


def transcript(cs_hash: bytes, previous, g1_s, g1_sx) -> bytes:
    h = hashlib.blake2b(digest_size=64)
    h.update(bytes(cs_hash))
    for c in previous:
        h.update(hash_pub_key(c))
    h.update(u_g1(g1_s))
    h.update(u_g1(g1_sx))
    return h.digest()


def contribution_hash(c: formats.Contribution) -> bytes:
    return hashlib.blake2b(hash_pub_key(c), digest_size=64).digest()


# ---- device steps ------------------------------------------------------------------------------------------------------
def points_scale(net, points, k: int, g2: bool = False, out=None):
    """out[i] = k points[i] on the device (b200zk_points_scale_dev); points: CUDA int64 (n, 8 | 16).  out may be points."""
    import torch
    if not 0 <= k < (1 << 256):
        raise ValueError("points_scale: k must be a 256-bit non-negative integer")
    points = points.contiguous()
    if out is None:
        out = torch.empty_like(points)
    kl = np.array([(k >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)
    net.check(net._lib.b200zk_points_scale_dev(net._h, 0, int(g2), c_vp(points.data_ptr()), int(points.shape[0]),
                                               c_vp(kl.ctypes.data), c_vp(out.data_ptr())))
    return out


def _scale_one(net, p, k: int, g2: bool = False) -> np.ndarray:
    w = 16 if g2 else 8
    t = points_scale(net, net.to_device(np.ascontiguousarray(p, dtype=np.uint64).reshape(1, w)), k, g2)
    return t.cpu().numpy().view(np.uint64)[0].copy()


def _same_ratio(net, p1, p2, q1, q2) -> bool:
    """sameRatio(P1, P2; Q1, Q2): e(P1, Q2) == e(P2, Q1), as b200zk_groth16_verify with no public inputs, IC_0 = C =
    infinity: it checks e(A, B) == e(alpha, beta) with A = P1, B = Q2, alpha = P2, beta = Q1."""
    g1 = lambda a: _as_u64(np.asarray(a, dtype=np.uint64).reshape(-1), 8).reshape(-1)
    g2 = lambda a: _as_u64(np.asarray(a, dtype=np.uint64).reshape(-1), 16).reshape(-1)
    a, alpha, b, beta = g1(p1), g1(p2), g2(q2), g2(q1)
    inf = np.zeros(8, dtype=np.uint64)
    ok = ctypes.c_int(0)
    net.check(net._lib.b200zk_groth16_verify(net._h, _ptr(alpha), _ptr(beta), _ptr(beta), _ptr(beta), _ptr(inf), 0, None,
                                             _ptr(a), _ptr(b), _ptr(inf), ctypes.byref(ok)))
    return bool(ok.value)


def _from_rng(net, rng: ChaCha, g2: bool) -> np.ndarray:
    """G.fromRng (see the module docstring).  Candidates are drawn from the RNG in order and decompressed on the device
    in batches (b200zk_points_decompress_dev, check_subgroup = 0: an invalid slot means x^3 + b is not a square); the
    first valid one is the result.  The RNG is left right after the accepted candidate's last word, as a one-at-a-time
    fromRng leaves it (a phase-1 key draws three G1.fromRng from one RNG): the position after each candidate is saved
    and the winner's restored."""
    import torch
    while True:
        enc = bytearray()
        after = []
        for _ in range(_CANDIDATES):
            if g2:
                c0 = field_from_rng(rng, Q) * _RINV_Q % Q
                c1 = field_from_rng(rng, Q) * _RINV_Q % Q
                b = bytearray(c0.to_bytes(32, "little") + c1.to_bytes(32, "little"))
            else:
                b = bytearray((field_from_rng(rng, Q) * _RINV_Q % Q).to_bytes(32, "little"))
            if rng.next_bool():
                b[-1] |= 0x80
            enc += b
            after.append(rng.snapshot())
        data = torch.from_numpy(np.frombuffer(bytes(enc), dtype=np.uint8).copy()).to(net._dev())
        out = torch.empty((_CANDIDATES, 16 if g2 else 8), dtype=torch.int64, device=data.device)
        bad = ctypes.c_size_t(0)
        rc = net._lib.b200zk_points_decompress_dev(net._h, 0, int(g2), c_vp(data.data_ptr()), _CANDIDATES, 0,
                                                   c_vp(out.data_ptr()), ctypes.byref(bad))
        if rc not in (_native.OK, _native.ERR_ARG) or (rc == _native.ERR_ARG and bad.value == 0):
            net.check(rc)
        pts = out.cpu().numpy().view(np.uint64)
        for i in range(_CANDIDATES):
            if pts[i].any():
                p = pts[i].copy()
                rng.restore(after[i])
                return _scale_one(net, p, G2_COFACTOR, g2=True) if g2 else p


def hash_to_g2(net, t: bytes) -> np.ndarray:
    """snarkjs hashToG2: G2.fromRng of the ChaCha seeded with t[:32] (16 Montgomery limbs)."""
    return _from_rng(net, ChaCha.from_hash(t), g2=True)


def beacon_secrets(net, beacon_hash: bytes, num_iterations_exp: int):
    """(x, g1_s) of a beacon: x = Fr.fromRng (canonical int), g1_s = G1.fromRng (8 Montgomery limbs)."""
    rng = rng_from_beacon(beacon_hash, num_iterations_exp)
    x = field_from_rng(rng, R) * _RINV_R % R
    return x, _from_rng(net, rng, g2=False)


# ---- zkey surgery --------------------------------------------------------------------------------------------------------
def _section_table(zkey_bytes: bytes):
    """[(sid, offset, length)] in file order; FormatError for a table that runs past the file."""
    buf = zkey_bytes
    if buf[:4] != b"zkey" or len(buf) < 12:
        raise formats.FormatError("bad magic %r (expected b'zkey')" % buf[:4])
    _version, nsec = struct.unpack_from("<II", buf, 4)
    off, out = 12, []
    for _ in range(nsec):
        if off + 12 > len(buf):
            raise formats.FormatError("zkey section table runs past the end of the file")
        sid, ln = struct.unpack_from("<IQ", buf, off)
        off += 12
        if off + ln > len(buf):
            raise formats.FormatError("zkey section %d runs past the end of the file" % sid)
        out.append((sid, off, ln))
        off += ln
    return out


def _section(zkey_bytes: bytes, sid: int) -> bytes:
    for s, off, ln in _section_table(zkey_bytes):
        if s == sid:
            return zkey_bytes[off:off + ln]
    raise formats.FormatError("zkey section %d missing" % sid)


def _replace_sections(zkey_bytes: bytes, new: dict) -> bytes:
    """The same file with the bodies of the sections in `new` replaced; every other byte and the section order kept."""
    table = _section_table(zkey_bytes)
    parts = [zkey_bytes[:12]]
    for sid, off, ln in table:
        body = new.get(sid, zkey_bytes[off:off + ln])
        parts.append(struct.pack("<IQ", sid, len(body)) + body)
    return b"".join(parts)


def _header_delta(hdr: bytes):
    if len(hdr) < _HDR_DELTA + 192:
        raise formats.FormatError("zkey header section too short (%d bytes)" % len(hdr))
    d1 = np.frombuffer(hdr, dtype="<u8", count=8, offset=_HDR_DELTA).copy()
    d2 = np.frombuffer(hdr, dtype="<u8", count=16, offset=_HDR_DELTA + 64).copy()
    return d1, d2


def _scale_section(net, sec: bytes, k: int, timings=None) -> bytes:
    """A G1 section times k: upload, b200zk_points_scale_dev in place, download."""
    import time
    if not sec:
        return sec
    t0 = time.perf_counter()
    pts = net.to_device(np.frombuffer(sec, dtype="<u8").reshape(-1, 8).copy())
    net.sync(0)
    t1 = time.perf_counter()
    points_scale(net, pts, k, out=pts)
    net.sync(0)
    t2 = time.perf_counter()
    out = pts.cpu().numpy().tobytes()
    t3 = time.perf_counter()
    if timings is not None:
        timings["transfer_s"] = timings.get("transfer_s", 0.0) + (t1 - t0) + (t3 - t2)
        timings["scale_s"] = timings.get("scale_s", 0.0) + (t2 - t1)
    return out


def _apply(net, zkey_bytes: bytes, x: int, g1_s, record: dict, timings=None):
    """Shared by contribute and beacon: the new zkey bytes and the new record."""
    import time
    x %= R
    if x == 0:
        raise ValueError("the contribution secret must be non-zero mod r")
    t0 = time.perf_counter()
    mpc = formats.read_mpc_params(zkey_bytes)
    hdr = _section(zkey_bytes, 2)
    d1, d2 = _header_delta(hdr)
    t1 = time.perf_counter()
    g1_s = np.ascontiguousarray(g1_s, dtype=np.uint64).reshape(-1)
    g1_sx = _scale_one(net, g1_s, x)
    t = transcript(mpc.cs_hash, mpc.contributions, g1_s, g1_sx)
    g2_spx = _scale_one(net, hash_to_g2(net, t), x, g2=True)
    d1n, d2n = _scale_one(net, d1, x), _scale_one(net, d2, x, g2=True)
    t2 = time.perf_counter()
    xinv = pow(x, -1, R)
    l_sec = _scale_section(net, _section(zkey_bytes, 8), xinv, timings)
    h_sec = _scale_section(net, _section(zkey_bytes, 9), xinv, timings)
    t3 = time.perf_counter()
    c = formats.Contribution(delta_after=d1n, g1_s=g1_s, g1_sx=g1_sx, g2_spx=g2_spx, transcript=t, **record)
    mpc.contributions.append(c)
    new_hdr = hdr[:_HDR_DELTA] + d1n.astype("<u8").tobytes() + d2n.astype("<u8").tobytes() + hdr[_HDR_DELTA + 192:]
    out = _replace_sections(zkey_bytes, {2: new_hdr, 8: l_sec, 9: h_sec, 10: formats.mpc_params_bytes(mpc)})
    t4 = time.perf_counter()
    if timings is not None:
        timings["parse_s"] = t1 - t0
        timings["record_s"] = t2 - t1                  # proof of knowledge, transcript, hash-to-G2, delta
        timings["sections_s"] = t3 - t2                # L and H: transfer + kernel (split above)
        timings["serialise_s"] = t4 - t3
    return out, contribution_hash(c)


def contribute(net, zkey_bytes: bytes, x: int, g1_s, name: str | None = None, timings: dict | None = None):
    """One phase-2 contribution with a known secret x (non-zero mod r) and proof-of-knowledge base g1_s (8 Montgomery
    limbs): delta_1, delta_2 times x, L and H times x^-1 on the device, a type-0 record appended to section 10.  Sections
    1 and 3-7 stay byte-identical.  Returns (zkey bytes, contribution hash)."""
    if name is not None and len(name.encode("utf-8")) > 64:
        raise ValueError("contribution name longer than 64 bytes")
    return _apply(net, zkey_bytes, x, g1_s, dict(type=0, name=name), timings)


def beacon(net, zkey_bytes: bytes, beacon_hash: bytes, num_iterations_exp: int, name: str | None = None,
           timings: dict | None = None):
    """A beacon contribution: x and g1_s derived from (beacon_hash, 2^num_iterations_exp SHA-256 rounds) as snarkjs
    `zkey beacon` does; the record is type 1 with those parameters.  Returns (zkey bytes, contribution hash)."""
    if name is not None and len(name.encode("utf-8")) > 64:
        raise ValueError("contribution name longer than 64 bytes")
    x, g1_s = beacon_secrets(net, beacon_hash, num_iterations_exp)
    return _apply(net, zkey_bytes, x, g1_s, dict(type=1, name=name, num_iterations_exp=int(num_iterations_exp),
                                                 beacon_hash=bytes(beacon_hash)), timings)


# ---- verification --------------------------------------------------------------------------------------------------------
@dataclass
class Phase2Report:
    ok: bool
    failures: list = field(default_factory=list)          # one line per failed check
    contributions: list = field(default_factory=list)     # (name, type, contribution hash) per record, oldest first
    cs_hash: bytes = b""                                   # as found in the file
    cs_hash_expected: bytes = b""                          # recomputed from the circuit and ceremony (check_cs_hash only)


def _g1_gen():
    mont = lambda v: [((v << 256) % Q >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)]
    return np.array(mont(1) + mont(2), dtype=np.uint64)


def _rlc(net, pts_bytes: bytes, rho):
    """sum_i rho_i P_i (affine, 8 limbs) over a G1 section on the device (the existing G1 MSM)."""
    pts = net.to_device(np.frombuffer(pts_bytes, dtype="<u8").reshape(-1, 8).copy())
    xyzz = net.msm_dev(pts, rho)
    out, inf = net.sum_points_dev(xyzz, 1)
    return np.zeros(8, dtype=np.uint64) if inf else out


def _random_scalars(net, n: int):
    """n scalars of 128 random bits (os.urandom) as Montgomery limbs on the device."""
    raw = np.zeros((n, 4), dtype=np.uint64)
    raw[:, :2] = np.frombuffer(os.urandom(16 * n), dtype="<u8").reshape(n, 2)
    return net.fr_convert(net.to_device(raw), to_mont=True)


def verify(net, r1cs_bytes: bytes, ptau_path: str, zkey_bytes: bytes, check_cs_hash: bool = False) -> Phase2Report:
    """snarkjs `zkey verify <r1cs> <ptau> <zkey>` on the GPU: the key is the `zkey new` key of this circuit and ceremony
    followed by a valid chain of phase-2 contributions.  The report holds the csHash found in the file.  check_cs_hash
    also recomputes it from the rebuilt initial key and the ceremony (cshash.cs_hash) into cs_hash_expected and fails on
    a mismatch; without it the csHash is carried, not checked."""
    from .circom import zkey_new
    from .setup import _fixed_base, _mont_limbs
    rep = Phase2Report(ok=False)
    fail = rep.failures.append
    try:
        mpc = formats.read_mpc_params(zkey_bytes)
        hdr = _section(zkey_bytes, 2)
        d1, d2 = _header_delta(hdr)
        cur = {sid: _section(zkey_bytes, sid) for sid in (1, 3, 4, 5, 6, 7, 8, 9)}
    except formats.FormatError as e:
        fail("not a zkey with phase-2 parameters: %s" % e)
        return rep
    rep.cs_hash = mpc.cs_hash
    init = zkey_new(net, r1cs_bytes, ptau_path, cs_hash=check_cs_hash)
    if check_cs_hash:
        rep.cs_hash_expected = _section(init, 10)[:64]
        if bytes(mpc.cs_hash) != rep.cs_hash_expected:
            fail("circuit hash (csHash) %s... differs from %s..., the one of this circuit and ceremony"
                 % (bytes(mpc.cs_hash)[:8].hex(), rep.cs_hash_expected[:8].hex()))
    ihdr = _section(init, 2)
    if len(ihdr) != len(hdr) or ihdr[:_HDR_DELTA] != hdr[:_HDR_DELTA] or ihdr[_HDR_DELTA + 192:] != hdr[_HDR_DELTA + 192:]:
        fail("header (apart from delta) differs from the initial key of this circuit and ceremony")
    for sid in (1, 3, 4, 5, 6, 7):
        if _section(init, sid) != cur[sid]:
            fail("section %d differs from the initial key of this circuit and ceremony" % sid)
    import torch
    one = torch.from_numpy(_mont_limbs(1).view(np.int64)).to(net._dev()).reshape(1, 4)
    g1 = _g1_gen()
    g2 = _fixed_base(net, one, g2=True).cpu().numpy().view(np.uint64)[0].copy()
    prev, delta = [], g1
    for j, c in enumerate(mpc.contributions):
        label = "contribution %d (%s)" % (j + 1, c.name or "unnamed")
        rep.contributions.append((c.name, c.type, contribution_hash(c)))
        if transcript(mpc.cs_hash, prev, c.g1_s, c.g1_sx) != bytes(c.transcript):
            fail("%s: inconsistent transcript" % label)
        g2_sp = hash_to_g2(net, c.transcript)
        if not _same_ratio(net, c.g1_s, c.g1_sx, g2_sp, c.g2_spx):
            fail("%s: the proof of knowledge (g1_s, g1_sx; g2_sp, g2_spx) does not hold" % label)
        if not _same_ratio(net, delta, c.delta_after, g2_sp, c.g2_spx):
            fail("%s: deltaAfter is not the previous delta times the contribution's secret" % label)
        if c.type == 1:
            e, bh = c.num_iterations_exp, c.beacon_hash
            if e is None or bh is None or not 0 <= e <= 63:
                fail("%s: beacon record without usable parameters" % label)
            else:
                x, s = beacon_secrets(net, bh, e)
                want = (s, _scale_one(net, s, x), _scale_one(net, g2_sp, x, g2=True), _scale_one(net, delta, x))
                got = (c.g1_s, c.g1_sx, c.g2_spx, c.delta_after)
                if not all((np.asarray(a, dtype=np.uint64) == np.asarray(b, dtype=np.uint64)).all() for a, b in zip(want, got)):
                    fail("%s: the beacon parameters do not reproduce the record" % label)
        elif c.type != 0:
            fail("%s: unknown record type %d" % (label, c.type))
        prev.append(c)
        delta = np.asarray(c.delta_after, dtype=np.uint64)
    if not (delta == d1).all():
        fail("delta_1 of the header is not the last contribution's deltaAfter")
    if not _same_ratio(net, g1, d1, g2, d2):
        fail("delta_1 and delta_2 of the header do not match")
    for sid, what in ((8, "L"), (9, "H")):
        a, b = _section(init, sid), cur[sid]
        if len(a) != len(b):
            fail("the %s section has %d points, the initial key %d" % (what, len(b) // 64, len(a) // 64))
            continue
        if not a:
            continue
        if sid == 9:
            _check_h(net, a, b, g2, d2, fail)
            continue
        rho = _random_scalars(net, len(a) // 64)
        # e(sum rho P, delta_2) == e(sum rho P_init, G2): every point is the initial one times delta^-1
        if not _same_ratio(net, _rlc(net, b, rho), _rlc(net, a, rho), g2, d2):
            fail("the %s section is not the initial one times delta^-1" % what)
    rep.ok = not rep.failures
    return rep


def _check_h(net, init_h: bytes, cur_h: bytes, g2, d2, fail) -> None:
    """The H section (h_k = L^2n_(2k+1)(tau) delta^-1 G1, k < n) checked in the tau basis, H_i = tau^i (tau^n - 1) delta^-1
    G1 = -2 w_2n^i sum_k w_n^(i k) h_k.  The prover only uses H_0 .. H_(n-2) (h(X) has degree <= n - 2), and a key that
    went through a bellman round (groth16/bellman.py) has H_(n-1) = infinity: the MPC-params file does not carry it.  So
    sum_(i < n-1) rho_i H_i = MSM(h, s) with s = NTT(rho_i (-2) w_2n^i), rho_(n-1) = 0, must be the initial one times
    delta^-1, and H_(n-1) = MSM(h, t), t = NTT of the same transform of the last unit vector, must be infinity or the
    initial one times delta^-1."""
    import torch
    from .setup import _powers
    n = len(init_h) // 64
    w2n = pow(5, (R - 1) // (2 * n), R)
    rho = _random_scalars(net, n)
    rho[n - 1] = 0
    c = _powers(net, w2n, R - 2, n)                                       # -2 w_2n^i
    net.check(net._lib.b200zk_fr_mul_sub_dev(net._h, 0, c_vp(rho.data_ptr()), c_vp(c.data_ptr()),
                                             c_vp(torch.zeros_like(c).data_ptr()), c_vp(c.data_ptr()), n))
    s = net.ntt_dev(c)
    if not _same_ratio(net, _rlc(net, cur_h, s), _rlc(net, init_h, s), g2, d2):
        fail("the H section is not the initial one times delta^-1 in its first n - 1 tau components")
    t = _powers(net, pow(w2n, 2 * (n - 1), R), (R - 2) * pow(w2n, n - 1, R) % R, n)   # NTT(-2 w_2n^(n-1) e_(n-1))
    x_cur, x_init = _rlc(net, cur_h, t), _rlc(net, init_h, t)
    if x_cur.any() and not _same_ratio(net, x_cur, x_init, g2, d2):
        fail("the last tau component of the H section is neither infinity nor the initial one times delta^-1")
