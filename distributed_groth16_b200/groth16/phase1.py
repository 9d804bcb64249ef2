"""Phase 1 of a Groth16 ceremony on the GPU: snarkjs `powersoftau new`, `contribute`, `beacon` and `verify`.

A phase-1 file (formats.PTau(prepared=False)) holds tau^i G1 (section 2, 2^(p+1) - 1 points), tau^i G2 (3), alpha tau^i G1
(4), beta tau^i G1 (5), beta G2 (6) and the contribution records (7).  `new` writes the generators in every slot.  A
contribution with secrets (tau, alpha, beta) multiplies point i of sections 2 / 3 by tau^i, of 4 by alpha tau^i and of 5
by beta tau^i, and section 6 by beta: every point by a different scalar.  That is b200zk_points_mul_powers_dev, the whole
cost of the step (about 16.8 M G1 and 4.2 M G2 scalar multiplications at power 22).  The record it appends proves
knowledge of the three secrets and chains the contribution to the previous one through two Blake2b-512 hashes:

  * key: tau, alpha, beta = Fr.fromRng x 3 (in that order), then for each of tau, alpha, beta in turn g1_s = G1.fromRng,
    g1_sx = x g1_s, g2_sp = hashToG2(Blake2b-512(u8 personalisation 0 / 1 / 2 || lastChallenge || U(g1_s) ||
    U(g1_sx))), g2_spx = x g2_sp (phase2: ChaCha, fromRng, hashToG2; U = toRprUncompressed);
  * response hash: Blake2b-512 of lastChallenge, the C encodings (toRprCompressed) of the new sections 2..6, then the
    public key as U(tau.g1_s) U(tau.g1_sx) U(alpha.g1_s) U(alpha.g1_sx) U(beta.g1_s) U(beta.g1_sx) U(tau.g2_spx)
    U(alpha.g2_spx) U(beta.g2_spx).  The record stores the hasher's state before the key (partialHash, csrc/blake2b.cuh);
  * nextChallenge = Blake2b-512(responseHash || U of the new sections 2..6), which the next contribution starts from.
    Before the first contribution, lastChallenge = first_challenge_hash(power).

The encodings of every point are made on the device (b200zk_points_encode_dev); the hashing runs on the host.

A coordinated ceremony moves two bare files instead of the .ptau (n = 2^power; snarkjs `powersoftau export challenge`,
`challenge contribute` and `import response`):

  * challenge, 384 n + 128 bytes: lastResponseHash (64 bytes; Blake2b-512("") before any contribution), then U of
    sections 2 (2n - 1 G1), 3 (n G2), 4 (n G1), 5 (n G1) and 6 (1 G2).  Its Blake2b-512 is the file's current
    challenge: the last record's nextChallenge, or first_challenge_hash(power) before any contribution;
  * response, 192 n + 864 bytes: the challenge hash (64 bytes), C of the five new sections in the same order, then
    pub_key_bytes(key) (768 bytes).  Its Blake2b-512 is the responseHash; the hasher's state before the key is the
    record's partialHash.

Reading them back decodes every point on the device (b200zk_points_decode_dev): one square root per compressed point.

Unpinned: there was no snarkjs and no published ceremony file to check against.  The section-7 layout and the 216-byte
partialHash layout (formats.parse_ptau_contributions, blake2b.cuh), the compressed encoding's flag rule, the order of the
key draws, the personalisation bytes and the stream hashed by first_challenge_hash are restated from memory of snarkjs /
ffjavascript; they agree with the repository's own Python restatement (tests/phase1_oracle.py) only.  First checks on a
real file: `verify` on powersOfTau28_hez_final_{10..14}.ptau (a failed proof of knowledge points at the draw order or the
personalisation, a failed nextChallenge at the encodings or partialHash), and first_challenge_hash(p) against what
snarkjs prints for `powersoftau new bn128 p`."""
from __future__ import annotations

import ctypes
import hashlib
import os
import time
import warnings
from dataclasses import dataclass, field

import numpy as np

from .. import _native, formats
from .._native import c_vp
from . import phase2

R = formats.FR_MODULUS
Q = formats.FQ_MODULUS
_RINV_R = pow(1 << 256, -1, R)
_KEYS = ("tau", "alpha", "beta")
# section -> (G2?, first scalar ("one", "alpha" or "beta"), points at power p)
_SECTIONS = {2: (False, "one", lambda p: (2 << p) - 1), 3: (True, "one", lambda p: 1 << p),
             4: (False, "alpha", lambda p: 1 << p), 5: (False, "beta", lambda p: 1 << p), 6: (True, "beta", lambda p: 1)}
DEFAULT_CHUNK = 1 << 22


# ---- Blake2b-512 with an exportable state (the library's host entries) --------------------------------------------------
class Blake2b512:
    """Blake2b-512 whose 216-byte state can be exported (state()) and resumed (Blake2b512(state)): b200zk_blake2b512_*.
    Needs the library, not a GPU."""

    def __init__(self, state: bytes | None = None):
        self._lib = _native.lib()
        self._s = ctypes.create_string_buffer(216)
        if state is None:
            self._check(self._lib.b200zk_blake2b512_init(self._s))
        else:
            if len(state) != 216:
                raise ValueError("a Blake2b state is 216 bytes, got %d" % len(state))
            ctypes.memmove(self._s, bytes(state), 216)

    @staticmethod
    def _check(rc):
        if rc != _native.OK:
            raise ValueError("Blake2b: invalid state or argument (b200zk error %d)" % rc)

    def update(self, data) -> None:
        a = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data).reshape(-1).view(np.uint8)
        if a.size:
            self._check(self._lib.b200zk_blake2b512_update(self._s, c_vp(a.ctypes.data), a.size))

    def state(self) -> bytes:
        return self._s.raw

    def digest(self) -> bytes:
        out = ctypes.create_string_buffer(64)
        self._check(self._lib.b200zk_blake2b512_final(self._s, out))
        return out.raw


# ---- generators and encodings ----------------------------------------------------------------------------------------
def _mont(v: int) -> list:
    x = v * (1 << 256) % Q
    return [(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)]


G1_GEN = np.array(_mont(1) + _mont(2), dtype=np.uint64)
G2_GEN = np.array(_mont(10857046999023057135944570762232829481370756359578518086990519993285655852781) +
                  _mont(11559732032986387107991004021392285783925812861821192530917403151452391805634) +
                  _mont(8495653923123431417604973247489272438418190587263600148770280649306958101930) +
                  _mont(4082367875863433681332203403145435568316851327593401208105741076214120093531), dtype=np.uint64)


def first_challenge_hash(power: int) -> bytes:
    """snarkjs calculateFirstChallengeHash: Blake2b-512 of Blake2b-512("") || U(G1) x (2^(p+1) - 1) || U(G2) x 2^p ||
    U(G1) x 2^p twice || U(G2) once -- the challenge of a file fresh from `new`."""
    h = hashlib.blake2b(digest_size=64)
    h.update(hashlib.blake2b(b"", digest_size=64).digest())
    u1, u2 = phase2.u_g1(G1_GEN), phase2.u_g2(G2_GEN)

    def repeat(u, n):
        block = u * min(n, 1 << 14)
        per = len(block) // len(u)
        while n >= per:
            h.update(block)
            n -= per
        h.update(u * n)

    repeat(u1, (2 << power) - 1)
    repeat(u2, 1 << power)
    repeat(u1, 1 << power)
    repeat(u1, 1 << power)
    h.update(u2)
    return h.digest()


def points_mul_powers(net, points, first: int, ratio: int, g2: bool = False, out=None):
    """out[i] = (first ratio^i) points[i] on the device (b200zk_points_mul_powers_dev); points: CUDA int64 (n, 8 | 16).
    out may be points."""
    import torch
    if not (0 <= first < (1 << 256) and 0 <= ratio < (1 << 256)):
        raise ValueError("points_mul_powers: first and ratio must be 256-bit non-negative integers")
    points = points.contiguous()
    if out is None:
        out = torch.empty_like(points)
    limbs = lambda v: np.array([(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)
    f, r = limbs(first), limbs(ratio)
    net.check(net._lib.b200zk_points_mul_powers_dev(net._h, 0, int(g2), c_vp(points.data_ptr()), int(points.shape[0]),
                                                    c_vp(f.ctypes.data), c_vp(r.ctypes.data), c_vp(out.data_ptr())))
    return out


def points_sub(net, a, b, g2: bool = False, out=None):
    """out[i] = a[i] - b[i] on the device (b200zk_points_sub_dev); a, b: CUDA int64 (n, 8 | 16).  out may be a or b."""
    import torch
    a, b = a.contiguous(), b.contiguous()
    if a.shape != b.shape:
        raise ValueError("points_sub: a and b have shapes %s and %s" % (tuple(a.shape), tuple(b.shape)))
    if out is None:
        out = torch.empty_like(a)
    net.check(net._lib.b200zk_points_sub_dev(net._h, 0, int(g2), c_vp(a.data_ptr()), c_vp(b.data_ptr()), int(a.shape[0]),
                                             c_vp(out.data_ptr())))
    return out


def points_encode(net, points, g2: bool = False, compressed: bool = False):
    """ffjavascript toRprUncompressed (compressed=False) / toRprCompressed encodings of CUDA int64 (n, 8 | 16) points on
    the device (b200zk_points_encode_dev) -> CUDA uint8 tensor (n, bytes per point)."""
    import torch
    points = points.contiguous()
    n = int(points.shape[0])
    w = (64 if g2 else 32) * (1 if compressed else 2)
    out = torch.empty((n, w), dtype=torch.uint8, device=points.device)
    net.check(net._lib.b200zk_points_encode_dev(net._h, 0, int(g2), c_vp(points.data_ptr()), n, int(compressed),
                                                c_vp(out.data_ptr())))
    return out


class InvalidEncodings(formats.FormatError):
    """points_decode met encodings that are not points: `count` of them, the first at index `first`."""

    def __init__(self, msg: str, count: int, first: int):
        super().__init__(msg)
        self.count, self.first = count, first


def points_decode(net, data, g2: bool = False, compressed: bool = False, check_subgroup: bool = False):
    """The inverse of points_encode on the device (b200zk_points_decode_dev): ffjavascript encodings (a CUDA uint8 tensor,
    or host bytes / uint8 array) -> CUDA int64 (n, 8 | 16) affine Montgomery points.  check_subgroup also requires
    [r] P == O on G2.  Raises InvalidEncodings (count, first index) when an encoding is not a valid point."""
    import torch
    w = (64 if g2 else 32) * (1 if compressed else 2)
    if not isinstance(data, torch.Tensor):
        host = np.ascontiguousarray(data).reshape(-1).view(np.uint8) if isinstance(data, np.ndarray) else \
            np.frombuffer(data, dtype=np.uint8)
        data = net.to_device(host if host.flags.writeable else host.copy())
    data = data.contiguous()
    if data.numel() % w:
        raise ValueError("points_decode: %d bytes are not a whole number of %d-byte encodings" % (data.numel(), w))
    n = data.numel() // w
    out = torch.empty((n, 16 if g2 else 8), dtype=torch.int64, device=data.device)
    bad, first = ctypes.c_size_t(0), ctypes.c_size_t(0)
    rc = net._lib.b200zk_points_decode_dev(net._h, 0, int(g2), c_vp(data.data_ptr()), n, int(compressed), int(check_subgroup),
                                           c_vp(out.data_ptr()), ctypes.byref(bad), ctypes.byref(first))
    if rc != _native.OK and bad.value:
        raise InvalidEncodings("%d of %d %s %s encodings are not valid points%s, the first at index %d"
                               % (bad.value, n, "G2" if g2 else "G1", "compressed" if compressed else "uncompressed",
                                  " of the order-r subgroup" if check_subgroup and g2 else "", first.value),
                               bad.value, first.value)
    net.check(rc)
    return out


def c_g1(p) -> bytes:
    """ffjavascript toRprCompressed of a G1 point on the host (8 Montgomery limbs): big-endian x, 0x80 in byte 0 when y
    is the larger of (y, -y)."""
    p = np.asarray(p, dtype=np.uint64).reshape(-1)
    if not p.any():
        return b"\x40" + bytes(31)
    x, y = phase2._fq(p[:4]), phase2._fq(p[4:8])
    b = bytearray(x.to_bytes(32, "big"))
    if y > Q - y:
        b[0] |= 0x80
    return bytes(b)


def c_g2(p) -> bytes:
    """The same for G2 (16 limbs): x.c1 || x.c0, the flag decided by y.c1 unless it is zero, then by y.c0."""
    p = np.asarray(p, dtype=np.uint64).reshape(-1)
    if not p.any():
        return b"\x40" + bytes(63)
    x0, x1, y0, y1 = (phase2._fq(p[4 * k:4 * k + 4]) for k in range(4))
    b = bytearray(x1.to_bytes(32, "big") + x0.to_bytes(32, "big"))
    y = y1 if y1 else y0
    if y > Q - y:
        b[0] |= 0x80
    return bytes(b)


def pub_key_bytes(key: dict) -> bytes:
    """snarkjs toPtauPubKeyRpr (not Montgomery): U of the six G1 points, then of the three G2 points."""
    return (b"".join(phase2.u_g1(key[k][f]) for k in _KEYS for f in ("g1_s", "g1_sx")) +
            b"".join(phase2.u_g2(key[k]["g2_spx"]) for k in _KEYS))


# ---- the key -------------------------------------------------------------------------------------------------------------
def g2_sp(net, personalisation: int, challenge: bytes, g1_s, g1_sx) -> np.ndarray:
    """snarkjs getG2sp: hashToG2(Blake2b-512(u8 personalisation || challenge || U(g1_s) || U(g1_sx)))."""
    h = hashlib.blake2b(bytes([personalisation]) + bytes(challenge) + phase2.u_g1(g1_s) + phase2.u_g1(g1_sx),
                        digest_size=64).digest()
    return phase2.hash_to_g2(net, h)


def create_key(net, rng: phase2.ChaCha, challenge: bytes) -> dict:
    """snarkjs createPTauKey: {"tau" | "alpha" | "beta": {"prv", "g1_s", "g1_sx", "g2_sp", "g2_spx"}} with prv canonical."""
    key = {k: {"prv": phase2.field_from_rng(rng, R) * _RINV_R % R} for k in _KEYS}
    for pers, k in enumerate(_KEYS):
        x = key[k]["prv"]
        g1_s = phase2._from_rng(net, rng, g2=False)
        g1_sx = phase2._scale_one(net, g1_s, x)
        sp = g2_sp(net, pers, challenge, g1_s, g1_sx)
        key[k].update(g1_s=g1_s, g1_sx=g1_sx, g2_sp=sp, g2_spx=phase2._scale_one(net, sp, x, g2=True))
    return key


# ---- new -----------------------------------------------------------------------------------------------------------------
def new(path: str, power: int) -> None:
    """snarkjs `powersoftau new bn128 <power>`: the generators in every slot of sections 2-6 and no contributions.  File
    writing only (no GPU)."""
    with formats.PTauWriter(path, power) as w:
        for sid, (g2, _, count) in _SECTIONS.items():
            gen = (G2_GEN if g2 else G1_GEN).astype("<u8").tobytes()
            n = count(power)
            block = gen * min(n, 1 << 16)
            per = len(block) // len(gen)
            while n >= per:
                w.write(sid, block)
                n -= per
            if n:
                w.write(sid, gen * n)
        w.write_contributions(formats.ptau_contributions_bytes([]))
        w.close()


# ---- contribute / beacon -------------------------------------------------------------------------------------------------
def _last_challenge(pt: formats.PTau, records: list) -> bytes:
    return bytes(records[-1].next_challenge) if records else first_challenge_hash(pt.ceremony_power)


def _read_records(pt: formats.PTau) -> list:
    return formats.parse_ptau_contributions(b"".join(pt.section_chunks(7)))


def _hash_written(net, fd: int, offsets: dict, power: int, hasher, chunk: int, t: dict, grab=None, out=None) -> None:
    """Feed U of sections 2..6 as written at `offsets` in the open file fd to hasher (encodings on the device), and
    write them to the open file `out` too when given.  grab[(sid, i)] is filled with point i of section sid when asked
    for."""
    for sid, (g2, _, count) in _SECTIONS.items():
        w, n = 16 if g2 else 8, count(power)
        for lo in range(0, n, chunk):
            cnt = min(chunk, n - lo)
            t0 = time.perf_counter()
            raw = os.pread(fd, cnt * w * 8, offsets[sid] + lo * w * 8)
            if len(raw) != cnt * w * 8:
                raise formats.FormatError("ptau section %d is shorter than power %d requires" % (sid, power))
            host = np.frombuffer(raw, dtype="<u8").reshape(cnt, w)
            t1 = time.perf_counter()
            d = net.to_device(host)
            enc = points_encode(net, d, g2, compressed=False).cpu().numpy()
            t2 = time.perf_counter()
            hasher.update(enc)
            t3 = time.perf_counter()
            if grab is not None:
                for (s, i) in grab:
                    if s == sid and lo <= i < lo + cnt:
                        grab[(s, i)] = host[i - lo].copy()
            if out is not None:
                out.write(enc)
            t4 = time.perf_counter()
            t["file_s"] += (t1 - t0) + (t4 - t3)
            t["encode_s"] += t2 - t1
            t["hash_s"] += t3 - t2


def _timings() -> dict:
    return {"kernel_s": 0.0, "decode_s": 0.0, "encode_s": 0.0, "hash_s": 0.0, "transfer_s": 0.0, "file_s": 0.0, "key_s": 0.0}


def _open_ceremony(src: str, dst: str, command: str) -> formats.PTau:
    """The input of contribute / beacon / import response: not the output file, not reduced; prepared with a warning."""
    if os.path.exists(dst) and os.path.exists(src) and os.path.samefile(src, dst):
        raise ValueError("powersoftau %s: the output %r is the input file" % (command, dst))
    pt = formats.PTau(src, prepared=False)
    try:
        if pt.power != pt.ceremony_power:
            raise ValueError("ptau %r is reduced (power %d of a ceremony of power %d): %s the full ceremony file"
                             % (src, pt.power, pt.ceremony_power, "contribute to" if command == "contribute" else
                                "use"))
        if any(pt.has_section(s) for s in (12, 13, 14, 15)):
            warnings.warn("ptau %r is prepared for phase 2: its Lagrange sections are dropped, the output has sections 1-7 "
                          "only (prepare it again afterwards)" % src)
    except BaseException:
        pt.close()
        raise
    return pt


def _public_key(key: dict) -> dict:
    return {k: {f: key[k][f] for f in ("g1_s", "g1_sx", "g2_spx")} for k in _KEYS}


def _mul_chunk(net, d, g2: bool, first: int, tau: int, response, t: dict) -> np.ndarray:
    """One chunk of a contribution: d <- (first tau^i) d[i] in place on the device, its compressed encodings hashed into
    the response hasher.  -> the encodings on the host."""
    t1 = time.perf_counter()
    points_mul_powers(net, d, first, tau, g2, out=d)
    net.sync(0)
    t2 = time.perf_counter()
    enc = points_encode(net, d, g2, compressed=True)
    net.sync(0)
    t3 = time.perf_counter()
    enc = enc.cpu().numpy()
    t4 = time.perf_counter()
    response.update(enc)
    t5 = time.perf_counter()
    t["kernel_s"] += t2 - t1
    t["encode_s"] += t3 - t2
    t["transfer_s"] += t4 - t3
    t["hash_s"] += t5 - t4
    return enc


def _finish(net, w: formats.PTauWriter, dst: str, records: list, pub: dict, partial: bytes, response_hash: bytes,
            record: dict, chunk: int, t: dict) -> bytes:
    """Close a ceremony file whose sections 2-6 are written: nextChallenge = Blake2b-512(responseHash || U of the written
    sections) in a second pass over the file, then the new record (the points it names read back from the file) appended
    to section 7.  -> nextChallenge."""
    w.flush()
    nxt = hashlib.blake2b(digest_size=64)
    nxt.update(response_hash)
    grab = {(2, 1): None, (3, 1): None, (4, 0): None, (5, 0): None, (6, 0): None}
    fd = os.open(dst, os.O_RDONLY)
    try:
        _hash_written(net, fd, w.section_offsets, w.power, nxt, chunk, t, grab)
    finally:
        os.close(fd)
    next_challenge = nxt.digest()
    rec = formats.PTauContribution(tau_g1=grab[(2, 1)], tau_g2=grab[(3, 1)], alpha_g1=grab[(4, 0)],
                                   beta_g1=grab[(5, 0)], beta_g2=grab[(6, 0)], key=pub, partial_hash=partial,
                                   next_challenge=next_challenge, **record)
    t0 = time.perf_counter()
    w.write_contributions(formats.ptau_contributions_bytes(records + [rec]))
    w.close()
    t["file_s"] += time.perf_counter() - t0
    return next_challenge


def _contribute(net, src: str, dst: str, rng: phase2.ChaCha, record: dict, chunk: int, timings: dict | None):
    if chunk < 1:
        raise ValueError("chunk must be at least 1 point")
    t = _timings()
    with _open_ceremony(src, dst, "contribute") as pt:
        power = pt.power
        records = _read_records(pt)
        last = _last_challenge(pt, records)
        t0 = time.perf_counter()
        key = create_key(net, rng, last)
        t["key_s"] += time.perf_counter() - t0
        tau = key["tau"]["prv"]
        first_of = {"one": 1, "alpha": key["alpha"]["prv"], "beta": key["beta"]["prv"]}
        response = Blake2b512()
        response.update(last)
        w = formats.PTauWriter(dst, power)
        try:
            for sid, (g2, first_name, count) in _SECTIONS.items():
                width, n = 16 if g2 else 8, count(power)
                first = first_of[first_name]
                for lo in range(0, n, chunk):
                    cnt = min(chunk, n - lo)
                    t0 = time.perf_counter()
                    d = net.to_device(pt.points(sid, lo, cnt, width))
                    net.sync(0)
                    t["transfer_s"] += time.perf_counter() - t0
                    _mul_chunk(net, d, g2, first * pow(tau, lo, R) % R, tau, response, t)
                    t0 = time.perf_counter()
                    host = d.cpu().numpy()
                    t1 = time.perf_counter()
                    w.write(sid, host)
                    t["transfer_s"] += t1 - t0
                    t["file_s"] += time.perf_counter() - t1
            partial = response.state()
            pub = _public_key(key)
            response.update(pub_key_bytes(pub))
            response_hash = response.digest()
            next_challenge = _finish(net, w, dst, records, pub, partial, response_hash, record, chunk, t)
        except BaseException:
            w.__exit__(None, None, None)
            os.unlink(dst)
            raise
    for k in _KEYS:
        key[k]["prv"] = 0                   # the secrets go no further than this frame
    if timings is not None:
        timings.update(t)
    return response_hash, next_challenge


def contribute(net, src: str, dst: str, rng: phase2.ChaCha, name: str | None = None, chunk: int = DEFAULT_CHUNK,
               timings: dict | None = None):
    """snarkjs `powersoftau contribute <src> <dst>` with the key drawn from `rng` (create_key): sections 2-6 of src times
    the powers of the new secrets on the device, streamed to dst with a type-0 record appended to section 7.  src must
    not be reduced (power == ceremonyPower); a prepared src is accepted with a warning and dst has sections 1-7 only.
    `chunk` points go to the device at a time.  Returns (responseHash, nextChallenge)."""
    if name is not None and len(name.encode("utf-8")) > 64:
        raise ValueError("contribution name longer than 64 bytes")
    return _contribute(net, src, dst, rng, dict(type=0, name=name), chunk, timings)


def beacon(net, src: str, dst: str, beacon_hash: bytes, num_iterations_exp: int, name: str | None = None,
           chunk: int = DEFAULT_CHUNK, timings: dict | None = None):
    """snarkjs `powersoftau beacon`: a contribution whose rng is phase2.rng_from_beacon(beacon_hash, num_iterations_exp),
    recorded as type 1 with those parameters.  Returns (responseHash, nextChallenge)."""
    if name is not None and len(name.encode("utf-8")) > 64:
        raise ValueError("contribution name longer than 64 bytes")
    rng = phase2.rng_from_beacon(bytes(beacon_hash), int(num_iterations_exp))
    return _contribute(net, src, dst, rng, dict(type=1, name=name, num_iterations_exp=int(num_iterations_exp),
                                                beacon_hash=bytes(beacon_hash)), chunk, timings)


# ---- challenge / response ------------------------------------------------------------------------------------------------
def _last_response_hash(records: list) -> bytes:
    """The responseHash of the last record, from its partialHash and key (as verify recomputes it); Blake2b-512("")
    before any contribution."""
    if not records:
        return hashlib.blake2b(b"", digest_size=64).digest()
    h = Blake2b512(bytes(records[-1].partial_hash))
    h.update(pub_key_bytes(records[-1].key))
    return h.digest()


def _section_layout(power: int, compressed: bool) -> list:
    """[(sid, g2, points, byte offset in the challenge / response file, bytes per point)] for sections 2-6."""
    out, off = [], 64
    for sid, (g2, _, count) in _SECTIONS.items():
        per = (64 if g2 else 32) * (1 if compressed else 2)
        out.append((sid, g2, count(power), off, per))
        off += count(power) * per
    return out


def _pread_exact(fd: int, n: int, off: int) -> bytearray:
    buf = bytearray(n)
    got = os.preadv(fd, [buf], off)
    if got != n:
        raise formats.FormatError("file ends at byte %d, %d bytes were expected" % (off + got, off + n))
    return buf


def export_challenge(net, ptau: str, challenge: str, chunk: int = DEFAULT_CHUNK, timings: dict | None = None) -> bytes:
    """snarkjs `powersoftau export challenge <ptau> <challenge>`: the last responseHash (recomputed from the last record's
    partialHash and key) followed by U of sections 2-6, encoded on the device and hashed on the way out.  Refuses, and
    deletes the output, when the hash is not the file's current challenge (the last nextChallenge, or the first challenge
    hash of a fresh file).  Returns the challenge hash."""
    if chunk < 1:
        raise ValueError("chunk must be at least 1 point")
    t = _timings()
    with formats.PTau(ptau, prepared=False) as pt:
        records = _read_records(pt)
        want = _last_challenge(pt, records)
        h = hashlib.blake2b(digest_size=64)
        prefix = _last_response_hash(records)
        h.update(prefix)
        try:
            with open(challenge, "wb") as out:
                out.write(prefix)
                fd = os.open(ptau, os.O_RDONLY)
                try:
                    _hash_written(net, fd, {sid: pt.section_span(sid)[0] for sid in _SECTIONS}, pt.power, h, chunk, t,
                                  out=out)
                finally:
                    os.close(fd)
            got = h.digest()
            if got != want:
                raise ValueError("ptau %r: its challenge hash %s is not the file's current challenge %s (the file's points or "
                                 "its last record were altered)" % (ptau, got.hex(), want.hex()))
        except BaseException:
            if os.path.exists(challenge):
                os.unlink(challenge)
            raise
    if timings is not None:
        timings.update(t)
    return got


def challenge_contribute(net, challenge: str, response: str, rng: phase2.ChaCha, chunk: int = DEFAULT_CHUNK,
                         timings: dict | None = None):
    """snarkjs `powersoftau challenge contribute <challenge> <response>` with the key drawn from `rng`: the key is drawn
    against Blake2b-512 of the challenge (a first pass over the file); then every point is decoded on the device, multiplied
    by its power of the new secrets (as contribute does) and written compressed to the response, which ends with the
    public key.  Returns (challengeHash, responseHash)."""
    if chunk < 1:
        raise ValueError("chunk must be at least 1 point")
    if os.path.exists(response) and os.path.samefile(challenge, response):
        raise ValueError("challenge contribute: the response %r is the challenge file" % response)
    t = _timings()
    fd = os.open(challenge, os.O_RDONLY)
    try:
        size = os.fstat(fd).st_size
        power = formats.ptau_challenge_power(size)
        t0 = time.perf_counter()
        h = hashlib.blake2b(digest_size=64)
        for lo in range(0, size, 1 << 26):
            h.update(_pread_exact(fd, min(1 << 26, size - lo), lo))
        challenge_hash = h.digest()
        t["hash_s"] += time.perf_counter() - t0
        t0 = time.perf_counter()
        key = create_key(net, rng, challenge_hash)
        t["key_s"] += time.perf_counter() - t0
        tau = key["tau"]["prv"]
        first_of = {"one": 1, "alpha": key["alpha"]["prv"], "beta": key["beta"]["prv"]}
        resp = hashlib.blake2b(digest_size=64)
        resp.update(challenge_hash)
        try:
            with open(response, "wb") as out:
                out.write(challenge_hash)
                for sid, g2, n, off, per in _section_layout(power, compressed=False):
                    first = first_of[_SECTIONS[sid][1]]
                    for lo in range(0, n, chunk):
                        cnt = min(chunk, n - lo)
                        t0 = time.perf_counter()
                        raw = _pread_exact(fd, cnt * per, off + lo * per)
                        t1 = time.perf_counter()
                        enc = net.to_device(np.frombuffer(raw, dtype=np.uint8))
                        net.sync(0)
                        t2 = time.perf_counter()
                        try:
                            d = points_decode(net, enc, g2, compressed=False)
                        except InvalidEncodings as e:
                            raise formats.FormatError("challenge %r, section %d: %d points are not valid uncompressed "
                                                      "encodings, the first is point %d" % (challenge, sid, e.count, lo + e.first))
                        t3 = time.perf_counter()
                        c = _mul_chunk(net, d, g2, first * pow(tau, lo, R) % R, tau, resp, t)
                        t4 = time.perf_counter()
                        out.write(c)
                        t["file_s"] += (t1 - t0) + (time.perf_counter() - t4)
                        t["transfer_s"] += t2 - t1
                        t["decode_s"] += t3 - t2
                pub = pub_key_bytes(_public_key(key))
                out.write(pub)
                resp.update(pub)
        except BaseException:
            if os.path.exists(response):
                os.unlink(response)
            raise
    finally:
        os.close(fd)
    for k in _KEYS:
        key[k]["prv"] = 0                   # the secrets go no further than this frame
    if timings is not None:
        timings.update(t)
    return challenge_hash, resp.digest()


def _read_pub_key(net, raw: bytes) -> dict:
    """The 768-byte public key of a response (pub_key_bytes' layout) -> {"tau" | "alpha" | "beta": {"g1_s", "g1_sx",
    "g2_spx"}} as Montgomery limbs, decoded on the device (G2 with the subgroup check)."""
    try:
        g1 = points_decode(net, raw[:384], g2=False).cpu().numpy().view(np.uint64)
        g2 = points_decode(net, raw[384:], g2=True, check_subgroup=True).cpu().numpy().view(np.uint64)
    except InvalidEncodings as e:
        raise formats.FormatError("the response's public key holds %d invalid points (%s)" % (e.count, e))
    return {k: {"g1_s": g1[2 * j].copy(), "g1_sx": g1[2 * j + 1].copy(), "g2_spx": g2[j].copy()} for j, k in enumerate(_KEYS)}


def import_response(net, ptau: str, response: str, dst: str, name: str | None = None, chunk: int = DEFAULT_CHUNK,
                    timings: dict | None = None):
    """snarkjs `powersoftau import response <ptau> <response> <dst>`: the response's points decoded on the device (the G2
    sections 3 and 6 and the key's G2 points with the subgroup check: the file comes from outside) and written to dst with
    a type-0 record whose partialHash is the response hasher's state before the key.  The response must answer the
    file's current challenge.  Refuses a reduced ptau and dst == ptau, warns on a prepared one, as contribute does; like
    snarkjs it does not verify the contribution (verify does).  Returns (responseHash, nextChallenge)."""
    if name is not None and len(name.encode("utf-8")) > 64:
        raise ValueError("contribution name longer than 64 bytes")
    if chunk < 1:
        raise ValueError("chunk must be at least 1 point")
    t = _timings()
    with _open_ceremony(ptau, dst, "import response") as pt:
        power = pt.power
        records = _read_records(pt)
        last = _last_challenge(pt, records)
        fd = os.open(response, os.O_RDONLY)
        try:
            size = os.fstat(fd).st_size
            if size != formats.ptau_response_bytes(power):
                raise formats.FormatError("response %r is %d bytes, a power-%d response is %d" % (
                    response, size, power, formats.ptau_response_bytes(power)))
            prefix = bytes(_pread_exact(fd, 64, 0))
            if prefix != last:
                raise ValueError("response %r answers challenge %s, the file's current challenge is %s" % (
                    response, prefix.hex(), last.hex()))
            resp = Blake2b512()
            resp.update(prefix)
            w = formats.PTauWriter(dst, power)
            try:
                for sid, g2, n, off, per in _section_layout(power, compressed=True):
                    for lo in range(0, n, chunk):
                        cnt = min(chunk, n - lo)
                        t0 = time.perf_counter()
                        raw = _pread_exact(fd, cnt * per, off + lo * per)
                        t1 = time.perf_counter()
                        resp.update(raw)
                        t2 = time.perf_counter()
                        enc = net.to_device(np.frombuffer(raw, dtype=np.uint8))
                        net.sync(0)
                        t3 = time.perf_counter()
                        try:
                            d = points_decode(net, enc, g2, compressed=True, check_subgroup=g2)
                        except InvalidEncodings as e:
                            raise formats.FormatError("response %r, section %d: %d points are not valid compressed encodings%s, "
                                                      "the first is point %d" % (response, sid, e.count,
                                                                                 " of the order-r subgroup" if g2 else "",
                                                                                 lo + e.first))
                        t4 = time.perf_counter()
                        host = d.cpu().numpy()
                        t5 = time.perf_counter()
                        w.write(sid, host)
                        t6 = time.perf_counter()
                        t["file_s"] += (t1 - t0) + (t6 - t5)
                        t["hash_s"] += t2 - t1
                        t["transfer_s"] += (t3 - t2) + (t5 - t4)
                        t["decode_s"] += t4 - t3
                partial = resp.state()
                key_raw = bytes(_pread_exact(fd, 768, size - 768))
                pub = _read_pub_key(net, key_raw)
                resp.update(key_raw)
                response_hash = resp.digest()
                next_challenge = _finish(net, w, dst, records, pub, partial, response_hash, dict(type=0, name=name), chunk, t)
            except BaseException:
                w.__exit__(None, None, None)
                os.unlink(dst)
                raise
        finally:
            os.close(fd)
    if timings is not None:
        timings.update(t)
    return response_hash, next_challenge


# ---- verify --------------------------------------------------------------------------------------------------------------
@dataclass
class Phase1Report:
    ok: bool
    failures: list = field(default_factory=list)          # one line per failed check, naming the contribution or section
    contributions: list = field(default_factory=list)     # (name, type, nextChallenge) per record, oldest first


def _eq(a, b) -> bool:
    return bool((np.asarray(a, dtype=np.uint64).reshape(-1) == np.asarray(b, dtype=np.uint64).reshape(-1)).all())


def _shifted_sums(net, pt: formats.PTau, sid: int, g2: bool, n: int, chunk: int):
    """(sum_i rho_i P_i, sum_i rho_i P_{i+1}) over i < n - 1 for fresh 128-bit rho, by the existing MSM in chunks."""
    import torch
    w = 16 if g2 else 8
    parts = ([], [])
    for lo in range(0, n - 1, chunk):
        cnt = min(chunk, n - 1 - lo)
        rho = phase2._random_scalars(net, cnt)
        pts = net.to_device(pt.points(sid, lo, cnt + 1, w))
        for k in (0, 1):
            parts[k].append(net.msm_dev(pts[k:k + cnt].contiguous(), rho, g2=g2))
    out = []
    for p in parts:
        xyzz = torch.stack(p).contiguous()
        s, inf = net.sum_points_dev(xyzz, len(p), g2=g2)
        out.append(np.zeros(w, dtype=np.uint64) if inf else s)
    return out


def verify(net, path: str, chunk: int = DEFAULT_CHUNK) -> Phase1Report:
    """snarkjs `powersoftau verify <ptau>` on the GPU: every record's proofs of knowledge and its link to the previous
    one (sameRatio pairings), beacon records reproduced from their parameters, the file's points against the last record
    and against each other (random linear combinations on the MSM), the last nextChallenge recomputed from its
    partialHash and the file, and the Lagrange sections 12-15 when present (ptau.check_lagrange).  A file without
    contributions fails."""
    rep = Phase1Report(ok=False)
    fail = rep.failures.append
    try:
        pt = formats.PTau(path, prepared=False)
    except formats.FormatError as e:
        fail("not a phase-1 ptau: %s" % e)
        return rep
    with pt:
        try:
            records = _read_records(pt)
        except formats.FormatError as e:
            fail("section 7: %s" % e)
            return rep
        if not records:
            fail("no contributions: the file is fresh from `new`")
            return rep
        power = pt.power
        same = lambda a, b, c, d: phase2._same_ratio(net, a, b, c, d)
        prev = dict(tau_g1=G1_GEN, tau_g2=G2_GEN, alpha_g1=G1_GEN, beta_g1=G1_GEN, beta_g2=G2_GEN,
                    next_challenge=first_challenge_hash(pt.ceremony_power))
        for j, c in enumerate(records):
            label = "contribution %d (%s)" % (j + 1, c.name or "unnamed")
            rep.contributions.append((c.name, c.type, bytes(c.next_challenge)))
            sp = {k: g2_sp(net, pers, prev["next_challenge"], c.key[k]["g1_s"], c.key[k]["g1_sx"])
                  for pers, k in enumerate(_KEYS)}
            for k in _KEYS:
                if not same(c.key[k]["g1_s"], c.key[k]["g1_sx"], sp[k], c.key[k]["g2_spx"]):
                    fail("%s: the %s proof of knowledge (g1_s, g1_sx; g2_sp, g2_spx) does not hold" % (label, k))
            if not same(prev["tau_g1"], c.tau_g1, sp["tau"], c.key["tau"]["g2_spx"]):
                fail("%s: tauG1 is not the previous tauG1 times its tau" % label)
            if not same(c.key["tau"]["g1_s"], c.key["tau"]["g1_sx"], prev["tau_g2"], c.tau_g2):
                fail("%s: tauG2 is not the previous tauG2 times its tau" % label)
            if not same(prev["alpha_g1"], c.alpha_g1, sp["alpha"], c.key["alpha"]["g2_spx"]):
                fail("%s: alphaG1 is not the previous alphaG1 times its alpha" % label)
            if not same(prev["beta_g1"], c.beta_g1, sp["beta"], c.key["beta"]["g2_spx"]):
                fail("%s: betaG1 is not the previous betaG1 times its beta" % label)
            if not same(c.key["beta"]["g1_s"], c.key["beta"]["g1_sx"], prev["beta_g2"], c.beta_g2):
                fail("%s: betaG2 is not the previous betaG2 times its beta" % label)
            if c.type == 1:
                e, bh = c.num_iterations_exp, c.beacon_hash
                if e is None or bh is None or not 0 <= e <= 63:
                    fail("%s: beacon record without usable parameters" % label)
                else:
                    want = create_key(net, phase2.rng_from_beacon(bytes(bh), e), prev["next_challenge"])
                    if not all(_eq(want[k][f], c.key[k][f]) for k in _KEYS for f in ("g1_s", "g1_sx", "g2_spx")):
                        fail("%s: the beacon parameters do not reproduce its key" % label)
            elif c.type != 0:
                fail("%s: unknown record type %d" % (label, c.type))
            prev = dict(tau_g1=c.tau_g1, tau_g2=c.tau_g2, alpha_g1=c.alpha_g1, beta_g1=c.beta_g1, beta_g2=c.beta_g2,
                        next_challenge=bytes(c.next_challenge))
        last, llabel = records[-1], "contribution %d (%s)" % (len(records), records[-1].name or "unnamed")
        tg1, tg2 = pt.points(2, 0, 2, 8), pt.points(3, 0, 2, 16)
        if not _eq(tg1[0], G1_GEN):
            fail("section 2: tauG1[0] is not the G1 generator")
        if not _eq(tg2[0], G2_GEN):
            fail("section 3: tauG2[0] is not the G2 generator")
        for sid, idx, attr in ((2, 1, "tau_g1"), (3, 1, "tau_g2"), (4, 0, "alpha_g1"), (5, 0, "beta_g1"), (6, 0, "beta_g2")):
            w = 16 if _SECTIONS[sid][0] else 8
            if not _eq(pt.points(sid, idx, 1, w)[0], getattr(last, attr)):
                fail("section %d: point %d is not the %s of %s" % (sid, idx, attr, llabel))
        # consecutive points in the ratio tau: e(sum rho P_i, tau G2) == e(sum rho P_{i+1}, G2)
        for sid in (2, 4, 5):
            n = _SECTIONS[sid][2](power)
            if n > 1:
                a, b = _shifted_sums(net, pt, sid, False, n, chunk)
                if not same(a, b, G2_GEN, tg2[1]):
                    fail("section %d: the points are not successive powers of tau" % sid)
        n3 = _SECTIONS[3][2](power)
        a, b = _shifted_sums(net, pt, 3, True, n3, chunk)
        if not same(G1_GEN, tg1[1], a, b):
            fail("section 3: the points are not successive powers of tau")
        # nextChallenge of the last record from its partialHash and the file
        t = {"file_s": 0.0, "encode_s": 0.0, "hash_s": 0.0}
        try:
            resp = Blake2b512(bytes(last.partial_hash))
            resp.update(pub_key_bytes(last.key))
            nxt = hashlib.blake2b(digest_size=64)
            nxt.update(resp.digest())
            fd = os.open(path, os.O_RDONLY)
            try:
                _hash_written(net, fd, {sid: pt.section_span(sid)[0] for sid in _SECTIONS}, power, nxt, chunk, t)
            finally:
                os.close(fd)
            ok = nxt.digest() == bytes(last.next_challenge)
        except ValueError:
            ok = False
        if not ok:
            fail("%s: nextChallenge does not follow from its partialHash and the file's points" % llabel)
        has_lagrange = all(pt.has_section(s) for s in (12, 13, 14, 15))
    if has_lagrange:
        from .ptau import check_lagrange
        lr = check_lagrange(net, path)
        rep.failures += lr.failures
    rep.ok = not rep.failures
    return rep
