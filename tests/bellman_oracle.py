"""Pure-Python restatement of snarkjs `zkey export bellman`, `zkey bellman contribute` and `zkey import bellman` for tiny
keys (TEST INFRASTRUCTURE ONLY), the yardstick of distributed_groth16_b200.groth16.bellman.  Encodings and the zkey
reading come from cshash_oracle, the record, transcript and hash-to-G2 from phase2_oracle; the file walk, the group
arithmetic and both basis changes are restated here, the basis changes as direct sums (no FFT):

  export:  H_i = sum_k (-2 w_2n^i w_n^(i k)) h_k,                       i < n - 1
  import:  h_k = sum_(i < n-1) (-1/2 n^-1 w_2n^-i w_n^(-i k)) H_i,     k < n   (H_(n-1) taken as infinity)."""
import hashlib
import struct

import cshash_oracle as co
import phase2_oracle as p2o
from oracle import bn254 as o, layout

R = o.R
_HDR = (False, False, True, True, False, True)           # alpha_1 beta_1 beta_2 gamma_2 delta_1 delta_2
_HDR_DELTA = p2o._HDR_DELTA


def _dec_g1(b):
    return None if b[0] == 0x40 else (int.from_bytes(b[:32], "big"), int.from_bytes(b[32:64], "big"))


def _dec_g2(b):
    if b[0] == 0x40:
        return None
    x1, x0, y1, y0 = (int.from_bytes(b[32 * k:32 * k + 32], "big") for k in range(4))
    return (x0, x1), (y0, y1)


def _sum(points, scalars):
    acc = None
    for p, k in zip(points, scalars):
        acc = o.G1.add(acc, o.G1.mul(p, k % R)) if p is not None else acc
    return acc


def _walk(buf: bytes):
    """-> (offsets of the six header points, {part: (count, offset)}, csHash offset, records offset, record count)."""
    off, hdr = 0, []
    for g2 in _HDR:
        hdr.append(off)
        off += 128 if g2 else 64
    vec = {}
    for part, w in (("ic", 64), ("h", 64), ("l", 64), ("a", 64), ("b1", 64), ("b2", 128)):
        cnt = struct.unpack_from(">I", buf, off)[0]
        vec[part] = (cnt, off + 4)
        off += 4 + cnt * w
    k = struct.unpack_from(">I", buf, off + 64)[0]
    assert len(buf) == off + 68 + 384 * k
    return hdr, vec, off, off + 68, k


def export(zkey: bytes) -> bytes:
    s = co.zkey_sections(zkey)
    hdr = s[2]
    n_vars, n_public, n = struct.unpack_from("<III", hdr, 72)
    out, off = [], 84
    for g2 in _HDR:
        out.append(co.u_g2_bytes(hdr, off) if g2 else co.u_g1_bytes(hdr, off))
        off += 128 if g2 else 64

    def vec(sid, count, g2=False):
        w = 128 if g2 else 64
        assert len(s[sid]) == count * w
        out.append(struct.pack(">I", count))
        out.extend(co.u_g2_bytes(s[sid], i * w) if g2 else co.u_g1_bytes(s[sid], i * w) for i in range(count))

    vec(3, n_public + 1)
    h = [o._rd_g1(s[9], 64 * k) for k in range(n)]
    w2n = o.fr_root_of_unity(2 * n)
    w = w2n * w2n % R
    out.append(struct.pack(">I", n - 1))
    out.extend(co.u_g1(_sum(h, [-2 * pow(w2n, i, R) * pow(w, i * k, R) for k in range(n)])) for i in range(n - 1))
    vec(8, n_vars - n_public - 1)
    vec(5, n_vars)
    vec(6, n_vars)
    vec(7, n_vars, True)
    cs, recs = p2o._records(s[10])
    out += [cs, struct.pack(">I", len(recs))] + [p2o._pub_key(r) for r in recs]
    return b"".join(out)


def contribute(challenge: bytes, x: int, g1_s):
    """g1_s: an oracle point.  -> (response bytes, contribution hash)."""
    x %= R
    hdr, vec, cs_off, rec_off, k = _walk(challenge)
    out = bytearray(challenge)
    xinv = pow(x, -1, R)
    for part in ("h", "l"):
        cnt, off = vec[part]
        for i in range(cnt):
            a = off + 64 * i
            out[a:a + 64] = co.u_g1(o.G1.mul(_dec_g1(challenge[a:a + 64]), xinv))
    d1 = o.G1.mul(_dec_g1(challenge[hdr[4]:hdr[4] + 64]), x)
    d2 = o.G2.mul(_dec_g2(challenge[hdr[5]:hdr[5] + 128]), x)
    out[hdr[4]:hdr[4] + 64] = co.u_g1(d1)
    out[hdr[5]:hdr[5] + 128] = p2o.u_g2(d2)
    g1_sx = o.G1.mul(g1_s, x)
    t = hashlib.blake2b(challenge[cs_off:cs_off + 64] + challenge[rec_off:] + co.u_g1(g1_s) + co.u_g1(g1_sx),
                        digest_size=64).digest()
    rec = co.u_g1(d1) + co.u_g1(g1_s) + co.u_g1(g1_sx) + p2o.u_g2(o.G2.mul(p2o.hash_to_g2(t), x)) + t
    out[cs_off + 64:cs_off + 68] = struct.pack(">I", k + 1)
    return bytes(out) + rec, hashlib.blake2b(rec, digest_size=64).digest()


def import_response(zkey: bytes, response: bytes, name=None) -> bytes:
    s = co.zkey_sections(zkey)
    hdr, vec, cs_off, rec_off, k = _walk(response)
    n = struct.unpack_from("<III", s[2], 72)[2]
    cs, recs = p2o._records(s[10])
    assert response[cs_off:cs_off + 64] == cs and k > len(recs)
    g1 = lambda part, i: _dec_g1(response[vec[part][1] + 64 * i:vec[part][1] + 64 * i + 64])
    H = [g1("h", i) for i in range(vec["h"][0])]
    w2n = o.fr_root_of_unity(2 * n)
    w = w2n * w2n % R
    c = -pow(2 * n, -1, R)
    h = [_sum(H, [c * pow(w2n, -i, R) * pow(w, -i * j, R) for i in range(len(H))]) for j in range(n)]
    d1 = _dec_g1(response[hdr[4]:hdr[4] + 64])
    d2 = _dec_g2(response[hdr[5]:hdr[5] + 128])
    added = []
    for j in range(len(recs), k):
        b = response[rec_off + 384 * j:rec_off + 384 * j + 384]
        added.append(dict(delta_after=_dec_g1(b[:64]), g1_s=_dec_g1(b[64:128]), g1_sx=_dec_g1(b[128:192]),
                          g2_spx=_dec_g2(b[192:320]), transcript=b[320:], type=0, params=p2o._name_param(name)))
    old10 = s[10][68:]                                       # the key's own records, kept byte for byte
    new = {2: s[2][:_HDR_DELTA] + layout.g1_to_arr([d1]).tobytes() + layout.g2_to_arr([d2]).tobytes() + s[2][_HDR_DELTA + 192:],
           8: layout.g1_to_arr([g1("l", i) for i in range(vec["l"][0])]).tobytes() if vec["l"][0] else b"",
           9: layout.g1_to_arr(h).tobytes(),
           10: cs + struct.pack("<I", k) + old10 + b"".join(p2o._rec_bytes(r) for r in added)}
    _version, nsec = struct.unpack_from("<II", zkey, 4)
    out, off = [zkey[:12]], 12
    for _ in range(nsec):
        sid, ln = struct.unpack_from("<IQ", zkey, off)
        b = new.get(sid, zkey[off + 12:off + 12 + ln])
        out.append(struct.pack("<IQ", sid, len(b)) + b)
        off += 12 + ln
    return b"".join(out)
