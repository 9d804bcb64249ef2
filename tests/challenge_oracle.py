"""Pure-Python restatement of snarkjs `powersoftau export challenge`, `challenge contribute` and `import response` for tiny
ceremonies (powers 1-2; TEST INFRASTRUCTURE ONLY), on tests/phase1_oracle.py: its group law, Blake2b with an exported
state, encodings, key draw and file layout.  The decoders of ffjavascript's encodings are restated here."""
import hashlib
import struct

from oracle import bn254 as o
import phase1_oracle as po

_G2S = po._G2S
_NAMES = ("tau", "alpha", "beta")


# ---- sizes ---------------------------------------------------------------------------------------------------------------
def challenge_size(power: int) -> int:
    n = 1 << power
    return 64 + (2 * n - 1) * 64 + n * 128 + 2 * n * 64 + 128


def response_size(power: int) -> int:
    n = 1 << power
    return 64 + (2 * n - 1) * 32 + n * 64 + 2 * n * 32 + 64 + 768


# ---- decoders ------------------------------------------------------------------------------------------------------------
def _larger(y: int) -> bool:
    return y > o.P - y


def _fq_sqrt(a: int):
    s = pow(a, (o.P + 1) // 4, o.P)
    return s if s * s % o.P == a % o.P else None


def _be(b: bytes) -> int:
    v = int.from_bytes(b, "big")
    if v >= o.P:
        raise ValueError("coordinate >= q")
    return v


def _inf(b: bytes) -> bool:
    if b[0] & 0x40:
        if b[0] != 0x40 or any(b[1:]):
            raise ValueError("bad infinity")
        return True
    return False


def dec_u_g1(b: bytes):
    if _inf(b):
        return None
    if b[0] & 0x80:
        raise ValueError("flag on an uncompressed point")
    x, y = _be(b[:32]), _be(b[32:])
    if (y * y - x ** 3 - o.B_G1) % o.P:
        raise ValueError("not on the curve")
    return (x, y)


def _subgroup(pt):
    if o.G2.from_jac(o.G2.jac_mul(o.G2.to_jac(pt), o.R)) is not None:
        raise ValueError("outside the order-r subgroup")
    return pt


def dec_u_g2(b: bytes, check_subgroup: bool = False):
    if _inf(b):
        return None
    if b[0] & 0x80:
        raise ValueError("flag on an uncompressed point")
    x = (_be(b[32:64]), _be(b[:32]))
    y = (_be(b[96:128]), _be(b[64:96]))
    if o.fq2_sqr(y) != o.fq2_add(o.fq2_mul(o.fq2_sqr(x), x), o.B_G2):
        raise ValueError("not on the twist")
    return _subgroup((x, y)) if check_subgroup else (x, y)


def dec_c_g1(b: bytes):
    if _inf(b):
        return None
    x = _be(bytes([b[0] & 0x3F]) + b[1:32])
    y = _fq_sqrt((x ** 3 + o.B_G1) % o.P)
    if y is None:
        raise ValueError("no point with this x")
    if _larger(y) != bool(b[0] & 0x80):
        y = (o.P - y) % o.P
    return (x, y)


def dec_c_g2(b: bytes, check_subgroup: bool = False):
    if _inf(b):
        return None
    x = (_be(b[32:64]), _be(bytes([b[0] & 0x3F]) + b[1:32]))
    y = o.fq2_sqrt(o.fq2_add(o.fq2_mul(o.fq2_sqr(x), x), o.B_G2))
    if y is None:
        raise ValueError("no point with this x")
    if _larger(y[1] if y[1] else y[0]) != bool(b[0] & 0x80):
        y = ((o.P - y[0]) % o.P, (o.P - y[1]) % o.P)
    return _subgroup((x, y)) if check_subgroup else (x, y)


def rogue_g2():
    """A point of the twist outside the order-r subgroup (smallest x0 with x = x0 + u on the twist and [r] P != O)."""
    x0 = 1
    while True:
        x = (x0, 1)
        y = o.fq2_sqrt(o.fq2_add(o.fq2_mul(o.fq2_sqr(x), x), o.B_G2))
        if y is not None and o.G2.from_jac(o.G2.jac_mul(o.G2.to_jac((x, y)), o.R)) is not None:
            return (x, y)
        x0 += 1


def non_curve_x(g2: bool) -> int:
    """The smallest x0 such that no point has x = x0 (G1) or x = x0 + 0 u (G2)."""
    x0 = 1
    while True:
        if g2:
            if o.fq2_sqrt(o.fq2_add(o.fq2_mul(o.fq2_sqr((x0, 0)), (x0, 0)), o.B_G2)) is None:
                return x0
        elif _fq_sqrt((x0 ** 3 + o.B_G1) % o.P) is None:
            return x0
        x0 += 1


# ---- the three steps -----------------------------------------------------------------------------------------------------
def _pub(k) -> bytes:
    return (b"".join(po.u_g1(k[nm][f]) for nm in _NAMES for f in ("g1_s", "g1_sx")) +
            b"".join(po.u_g2(k[nm]["g2_spx"]) for nm in _NAMES))


def export_challenge(ptau: bytes) -> bytes:
    """-> the challenge file: lastResponseHash (from the last record's partialHash and key) || U of sections 2-6."""
    power, pts, sec7 = po._read(ptau)
    recs = po._records(sec7)
    if recs:
        rec = recs[-1][0]
        h = po.Blake2b.from_state(rec[1216:1432])
        g1 = [po.u_g1(o._rd_g1(rec, 448 + 64 * i)) for i in range(6)]
        g2 = [po.u_g2(o._rd_g2(rec, 832 + 128 * i)) for i in range(3)]
        h.update(b"".join(g1) + b"".join(g2))
        prefix = h.digest()
    else:
        prefix = hashlib.blake2b(b"", digest_size=64).digest()
    return prefix + b"".join((po.u_g2 if sid in _G2S else po.u_g1)(p) for sid in (2, 3, 4, 5, 6) for p in pts[sid])


def _split(buf: bytes, power: int, per_g1: int, per_g2: int) -> dict:
    off, out = 64, {}
    for sid, n in po._counts(power).items():
        w = per_g2 if sid in _G2S else per_g1
        out[sid] = [buf[off + w * i:off + w * (i + 1)] for i in range(n)]
        off += w * n
    return out


def challenge_contribute(challenge: bytes, rng):
    """-> (response file, challengeHash, responseHash)"""
    power = {challenge_size(p): p for p in range(1, 28)}[len(challenge)]
    challenge_hash = hashlib.blake2b(challenge, digest_size=64).digest()
    k = po.key(rng, challenge_hash)
    tau, alpha, beta = (k[nm]["prv"] for nm in _NAMES)
    first = {2: 1, 3: 1, 4: alpha, 5: beta, 6: beta}
    enc = _split(challenge, power, 64, 128)
    body = b""
    for sid in (2, 3, 4, 5, 6):
        grp, dec, c = (o.G2, dec_u_g2, po.c_g2) if sid in _G2S else (o.G1, dec_u_g1, po.c_g1)
        body += b"".join(c(grp.mul(dec(e), first[sid] * pow(tau, i, o.R))) for i, e in enumerate(enc[sid]))
    resp = challenge_hash + body + _pub(k)
    return resp, challenge_hash, hashlib.blake2b(resp, digest_size=64).digest()


def import_response(ptau: bytes, response: bytes, name=None):
    """-> (ptau file, responseHash, nextChallenge)"""
    power, _, sec7 = po._read(ptau)
    recs = po._records(sec7)
    last = recs[-1][1] if recs else po.first_challenge_hash(power)
    assert response[:64] == last, "the response answers another challenge"
    assert len(response) == response_size(power)
    enc = _split(response, power, 32, 64)
    new_pts = {sid: [dec_c_g2(e, check_subgroup=True) if sid in _G2S else dec_c_g1(e) for e in enc[sid]]
               for sid in (2, 3, 4, 5, 6)}
    h = po.Blake2b()
    h.update(response[:-768])
    partial = h.state()
    key = response[-768:]
    h.update(key)
    response_hash = h.digest()
    nxt = hashlib.blake2b(digest_size=64)
    nxt.update(response_hash)
    for sid in (2, 3, 4, 5, 6):
        nxt.update(b"".join((po.u_g2 if sid in _G2S else po.u_g1)(p) for p in new_pts[sid]))
    next_challenge = nxt.digest()
    g1k = [dec_u_g1(key[64 * i:64 * i + 64]) for i in range(6)]
    g2k = [dec_u_g2(key[384 + 128 * i:384 + 128 * i + 128]) for i in range(3)]
    params = po.p2o._name_param(name)
    rec = (po.g1b([new_pts[2][1]]) + po.g2b([new_pts[3][1]]) + po.g1b([new_pts[4][0], new_pts[5][0]]) +
           po.g2b([new_pts[6][0]]) + po.g1b(g1k) + po.g2b(g2k) + partial + next_challenge +
           struct.pack("<II", 0, len(params)) + params)
    sec7 = struct.pack("<I", len(recs) + 1) + b"".join(r for r, _ in recs) + rec
    secs = {sid: (po.g2b if sid in _G2S else po.g1b)(new_pts[sid]) for sid in (2, 3, 4, 5, 6)}
    return po._file(power, secs, sec7), response_hash, next_challenge
