"""Pure-Python restatement of snarkjs `zkey contribute` and `zkey beacon` for tiny keys (TEST INFRASTRUCTURE ONLY), on the
oracle's group law and square roots.  It is the yardstick of distributed_groth16_b200.groth16.phase2: the byte-level
conventions (ChaCha draws, U(P), the transcript) are taken from the product's host helpers, which
tests/test_phase2_formats.py pins on their own; every group operation, square root, cofactor multiplication and the
zkey surgery are restated here."""
import hashlib
import struct

from oracle import bn254 as o, layout
from distributed_groth16_b200.groth16 import phase2 as p2

_RINV_Q = pow(o.MONT_R, -1, o.P)
_RINV_R = pow(o.MONT_R, -1, o.R)
_HDR_DELTA = 4 + 32 + 4 + 32 + 12 + 64 + 64 + 128 + 128


def u_g1(pt) -> bytes:
    return b"\x40" + bytes(63) if pt is None else pt[0].to_bytes(32, "big") + pt[1].to_bytes(32, "big")


def u_g2(pt) -> bytes:
    if pt is None:
        return b"\x40" + bytes(127)
    (x0, x1), (y0, y1) = pt
    return b"".join(v.to_bytes(32, "big") for v in (x1, x0, y1, y0))


def g2_times(pt, k):
    """k pt on the twist without reducing k mod r (cofactor clearing)."""
    return o.G2.from_jac(o.G2.jac_mul(o.G2.to_jac(pt), k))


def from_rng(rng, g2: bool):
    while True:
        if g2:
            x = tuple(p2.field_from_rng(rng, o.P) * _RINV_Q % o.P for _ in range(2))
            enc = bytearray(x[0].to_bytes(32, "little") + x[1].to_bytes(32, "little"))
        else:
            enc = bytearray((p2.field_from_rng(rng, o.P) * _RINV_Q % o.P).to_bytes(32, "little"))
        if rng.next_bool():
            enc[-1] |= 0x80
        try:
            pt = (o.g2_decompress if g2 else o.g1_decompress)(bytes(enc))
        except ValueError:
            continue
        return g2_times(pt, p2.G2_COFACTOR) if g2 else pt


def hash_to_g2(t: bytes):
    return from_rng(p2.ChaCha.from_hash(t), g2=True)


def _records(sec10: bytes):
    """section 10 -> (csHash, [record dicts with oracle points and the raw parameter bytes])."""
    cs, n = sec10[:64], struct.unpack_from("<I", sec10, 64)[0]
    off, recs = 68, []
    for _ in range(n):
        rd1 = lambda k: o._rd_g1(sec10, off + 64 * k)
        r = dict(delta_after=rd1(0), g1_s=rd1(1), g1_sx=rd1(2), g2_spx=o._rd_g2(sec10, off + 192))
        r["transcript"] = sec10[off + 320:off + 384]
        r["type"], plen = struct.unpack_from("<II", sec10, off + 384)
        r["params"] = sec10[off + 392:off + 392 + plen]
        off += 392 + plen
        recs.append(r)
    return cs, recs


def _pub_key(r) -> bytes:
    return u_g1(r["delta_after"]) + u_g1(r["g1_s"]) + u_g1(r["g1_sx"]) + u_g2(r["g2_spx"]) + r["transcript"]


def _rec_bytes(r) -> bytes:
    g1 = lambda p: layout.g1_to_arr([p]).tobytes()
    return (g1(r["delta_after"]) + g1(r["g1_s"]) + g1(r["g1_sx"]) + layout.g2_to_arr([r["g2_spx"]]).tobytes() +
            r["transcript"] + struct.pack("<II", r["type"], len(r["params"])) + r["params"])


def _apply(zkey: bytes, x: int, g1_s, rtype: int, params: bytes):
    secs = o._sections(zkey, b"zkey")
    body = lambda sid: zkey[secs[sid][0][0]:secs[sid][0][0] + secs[sid][0][1]]
    hdr = body(2)
    d1, d2 = o._rd_g1(hdr, _HDR_DELTA), o._rd_g2(hdr, _HDR_DELTA + 64)
    cs, recs = _records(body(10))
    g1_sx = o.G1.mul(g1_s, x)
    h = hashlib.blake2b(digest_size=64)
    h.update(cs)
    for r in recs:
        h.update(_pub_key(r))
    h.update(u_g1(g1_s) + u_g1(g1_sx))
    t = h.digest()
    d1n, d2n = o.G1.mul(d1, x), o.G2.mul(d2, x)
    rec = dict(delta_after=d1n, g1_s=g1_s, g1_sx=g1_sx, g2_spx=o.G2.mul(hash_to_g2(t), x), transcript=t, type=rtype,
               params=params)
    xinv = pow(x, -1, o.R)
    scale = lambda sid: layout.g1_to_arr([o.G1.mul(o._rd_g1(zkey, secs[sid][0][0] + 64 * i), xinv)
                                          for i in range(secs[sid][0][1] // 64)]).tobytes()
    new = {2: hdr[:_HDR_DELTA] + layout.g1_to_arr([d1n]).tobytes() + layout.g2_to_arr([d2n]).tobytes() + hdr[_HDR_DELTA + 192:],
           8: scale(8), 9: scale(9),
           10: cs + struct.pack("<I", len(recs) + 1) + b"".join(_rec_bytes(r) for r in recs + [rec])}
    _version, nsec = struct.unpack_from("<II", zkey, 4)
    out, off = [zkey[:12]], 12
    for _ in range(nsec):
        sid, ln = struct.unpack_from("<IQ", zkey, off)
        b = new.get(sid, zkey[off + 12:off + 12 + ln])
        out.append(struct.pack("<IQ", sid, len(b)) + b)
        off += 12 + ln
    return b"".join(out), hashlib.blake2b(_pub_key(rec), digest_size=64).digest()


def _name_param(name):
    if not name:
        return b""
    n = name.encode("utf-8")
    return bytes([1, len(n)]) + n


def contribute(zkey: bytes, x: int, g1_s, name=None):
    """g1_s: an oracle point.  -> (zkey bytes, contribution hash)."""
    return _apply(zkey, x % o.R, g1_s, 0, _name_param(name))


def beacon(zkey: bytes, beacon_hash: bytes, e: int, name=None):
    h = bytes(beacon_hash)
    for _ in range(1 << e):
        h = hashlib.sha256(h).digest()
    rng = p2.ChaCha.from_hash(h)
    x = p2.field_from_rng(rng, o.R) * _RINV_R % o.R
    g1_s = from_rng(rng, g2=False)
    params = _name_param(name) + bytes([2, e, 3, len(h := bytes(beacon_hash))]) + h
    return _apply(zkey, x, g1_s, 1, params)
