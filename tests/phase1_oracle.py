"""Pure-Python restatement of snarkjs `powersoftau new`, `contribute` and `beacon` for tiny ceremonies (powers 1-2; TEST
INFRASTRUCTURE ONLY), on the oracle's group law, with its own Blake2b whose state can be exported.  It is the yardstick of
distributed_groth16_b200.groth16.phase1: the ChaCha draws and the fromRng conventions come from the product's host helpers
(pinned on their own by the phase-2 tests), U(P) and fromRng / hashToG2 from tests/phase2_oracle.py; every group
operation, the compressed encoding, the hashes, the record layout and the file layout are restated here."""
import hashlib
import struct

from oracle import bn254 as o, layout
from distributed_groth16_b200.groth16 import phase2 as p2
import phase2_oracle as p2o

_RINV_R = pow(o.MONT_R, -1, o.R)
_M64 = (1 << 64) - 1


# ---- Blake2b (RFC 7693) with the 216-byte exported state -------------------------------------------------------------
class Blake2b:
    IV = [0x6A09E667F3BCC908, 0xBB67AE8584CAA73B, 0x3C6EF372FE94F82B, 0xA54FF53A5F1D36F1,
          0x510E527FADE682D1, 0x9B05688C2B3E6C1F, 0x1F83D9ABFB41BD6B, 0x5BE0CD19137E2179]
    SIGMA = [[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15], [14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3],
             [11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4], [7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8],
             [9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13], [2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9],
             [12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11], [13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10],
             [6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5], [10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0]]

    def __init__(self):
        self.h = list(self.IV)
        self.h[0] ^= 0x01010000 ^ 64
        self.t = 0
        self.b = bytearray(128)
        self.c = 0

    def _compress(self, last):
        v = self.h + self.IV
        v[12] ^= self.t & _M64
        v[13] ^= self.t >> 64
        if last:
            v[14] ^= _M64
        m = struct.unpack("<16Q", bytes(self.b))
        rot = lambda x, n: ((x >> n) | (x << (64 - n))) & _M64

        def g(a, b, c, d, x, y):
            v[a] = (v[a] + v[b] + x) & _M64; v[d] = rot(v[d] ^ v[a], 32)
            v[c] = (v[c] + v[d]) & _M64; v[b] = rot(v[b] ^ v[c], 24)
            v[a] = (v[a] + v[b] + y) & _M64; v[d] = rot(v[d] ^ v[a], 16)
            v[c] = (v[c] + v[d]) & _M64; v[b] = rot(v[b] ^ v[c], 63)

        for r in range(12):
            s = self.SIGMA[r % 10]
            g(0, 4, 8, 12, m[s[0]], m[s[1]]); g(1, 5, 9, 13, m[s[2]], m[s[3]])
            g(2, 6, 10, 14, m[s[4]], m[s[5]]); g(3, 7, 11, 15, m[s[6]], m[s[7]])
            g(0, 5, 10, 15, m[s[8]], m[s[9]]); g(1, 6, 11, 12, m[s[10]], m[s[11]])
            g(2, 7, 8, 13, m[s[12]], m[s[13]]); g(3, 4, 9, 14, m[s[14]], m[s[15]])
        self.h = [self.h[i] ^ v[i] ^ v[i + 8] for i in range(8)]

    def update(self, data):
        for byte in bytes(data):
            if self.c == 128:                       # compress a full buffer only when more input arrives
                self.t += 128
                self._compress(False)
                self.c = 0
            self.b[self.c] = byte
            self.c += 1

    def state(self) -> bytes:
        return (bytes(self.b) + struct.pack("<8Q", *self.h) + struct.pack("<QQ", self.t & _M64, self.t >> 64) +
                struct.pack("<II", self.c, 64))

    @classmethod
    def from_state(cls, s: bytes):
        h = cls()
        h.b = bytearray(s[:128])
        h.h = list(struct.unpack_from("<8Q", s, 128))
        lo, hi = struct.unpack_from("<QQ", s, 192)
        h.t = lo | hi << 64
        h.c = struct.unpack_from("<I", s, 208)[0]
        return h

    def digest(self) -> bytes:
        t = Blake2b.from_state(self.state())
        t.t += t.c
        t.b[t.c:] = bytes(128 - t.c)
        t._compress(True)
        return struct.pack("<8Q", *t.h)


# ---- encodings -----------------------------------------------------------------------------------------------------------
u_g1, u_g2 = p2o.u_g1, p2o.u_g2


def c_g1(pt) -> bytes:
    if pt is None:
        return b"\x40" + bytes(31)
    b = bytearray(pt[0].to_bytes(32, "big"))
    if pt[1] > o.P - pt[1]:
        b[0] |= 0x80
    return bytes(b)


def c_g2(pt) -> bytes:
    if pt is None:
        return b"\x40" + bytes(63)
    (x0, x1), (y0, y1) = pt
    b = bytearray(x1.to_bytes(32, "big") + x0.to_bytes(32, "big"))
    y = y1 if y1 else y0
    if y > o.P - y:
        b[0] |= 0x80
    return bytes(b)


g1b = lambda pts: layout.g1_to_arr(pts).tobytes()
g2b = lambda pts: layout.g2_to_arr(pts).tobytes()


# ---- file ----------------------------------------------------------------------------------------------------------------
def _counts(power):
    return {2: (2 << power) - 1, 3: 1 << power, 4: 1 << power, 5: 1 << power, 6: 1}


_G2S = {3, 6}


def _file(power: int, secs: dict, sec7: bytes) -> bytes:
    s1 = struct.pack("<I", 32) + o.P.to_bytes(32, "little") + struct.pack("<II", power, power)
    body = [(1, s1)] + [(sid, secs[sid]) for sid in (2, 3, 4, 5, 6)] + [(7, sec7)]
    return b"ptau" + struct.pack("<II", 1, 7) + b"".join(struct.pack("<IQ", sid, len(b)) + b for sid, b in body)


def new(power: int) -> bytes:
    secs = {sid: (g2b if sid in _G2S else g1b)([o.G2_GEN if sid in _G2S else o.G1_GEN] * n)
            for sid, n in _counts(power).items()}
    return _file(power, secs, struct.pack("<I", 0))


def first_challenge_hash(power: int) -> bytes:
    h = hashlib.blake2b(digest_size=64)
    h.update(hashlib.blake2b(b"", digest_size=64).digest())
    g1, g2 = u_g1(o.G1_GEN), u_g2(o.G2_GEN)
    h.update(g1 * ((2 << power) - 1) + g2 * (1 << power) + g1 * (1 << power) * 2 + g2)
    return h.digest()


def _read(ptau: bytes):
    secs = o._sections(ptau, b"ptau")
    body = lambda sid: ptau[secs[sid][0][0]:secs[sid][0][0] + secs[sid][0][1]]
    power = struct.unpack_from("<I", body(1), 36)[0]
    pts = {}
    for sid, n in _counts(power).items():
        b = body(sid)
        pts[sid] = [(o._rd_g2(b, 128 * i) if sid in _G2S else o._rd_g1(b, 64 * i)) for i in range(n)]
    return power, pts, body(7)


def _records(sec7: bytes):
    """-> [(record bytes, nextChallenge)]"""
    n = struct.unpack_from("<I", sec7, 0)[0]
    off, out = 4, []
    for _ in range(n):
        plen = struct.unpack_from("<I", sec7, off + 1500)[0]
        out.append((sec7[off:off + 1504 + plen], sec7[off + 1216 + 216:off + 1216 + 280]))
        off += 1504 + plen
    return out


def key(rng, challenge: bytes) -> dict:
    k = {nm: {"prv": p2.field_from_rng(rng, o.R) * _RINV_R % o.R} for nm in ("tau", "alpha", "beta")}
    for pers, nm in enumerate(("tau", "alpha", "beta")):
        x = k[nm]["prv"]
        s = p2o.from_rng(rng, g2=False)
        sx = o.G1.mul(s, x)
        t = hashlib.blake2b(bytes([pers]) + challenge + u_g1(s) + u_g1(sx), digest_size=64).digest()
        sp = p2o.hash_to_g2(t)
        k[nm].update(g1_s=s, g1_sx=sx, g2_sp=sp, g2_spx=o.G2.mul(sp, x))
    return k


def _apply(ptau: bytes, rng, rtype: int, params: bytes):
    power, pts, sec7 = _read(ptau)
    recs = _records(sec7)
    last = recs[-1][1] if recs else first_challenge_hash(power)
    k = key(rng, last)
    tau, alpha, beta = (k[nm]["prv"] for nm in ("tau", "alpha", "beta"))
    first = {2: 1, 3: 1, 4: alpha, 5: beta, 6: beta}
    new_pts = {sid: [(o.G2 if sid in _G2S else o.G1).mul(p, first[sid] * pow(tau, i, o.R)) for i, p in enumerate(ps)]
               for sid, ps in pts.items()}
    resp = Blake2b()
    resp.update(last)
    for sid in (2, 3, 4, 5, 6):
        resp.update(b"".join((c_g2 if sid in _G2S else c_g1)(p) for p in new_pts[sid]))
    partial = resp.state()
    names = ("tau", "alpha", "beta")
    pub = b"".join(u_g1(k[nm][f]) for nm in names for f in ("g1_s", "g1_sx")) + b"".join(u_g2(k[nm]["g2_spx"]) for nm in names)
    resp.update(pub)
    response_hash = resp.digest()
    nxt = hashlib.blake2b(digest_size=64)
    nxt.update(response_hash)
    for sid in (2, 3, 4, 5, 6):
        nxt.update(b"".join((u_g2 if sid in _G2S else u_g1)(p) for p in new_pts[sid]))
    next_challenge = nxt.digest()
    rec = (g1b([new_pts[2][1]]) + g2b([new_pts[3][1]]) + g1b([new_pts[4][0], new_pts[5][0]]) + g2b([new_pts[6][0]]) +
           g1b([k[nm][f] for nm in names for f in ("g1_s", "g1_sx")]) + g2b([k[nm]["g2_spx"] for nm in names]) +
           partial + next_challenge + struct.pack("<II", rtype, len(params)) + params)
    sec7 = struct.pack("<I", len(recs) + 1) + b"".join(r for r, _ in recs) + rec
    secs = {sid: (g2b if sid in _G2S else g1b)(new_pts[sid]) for sid in (2, 3, 4, 5, 6)}
    return _file(power, secs, sec7), response_hash, next_challenge


def contribute(ptau: bytes, rng, name=None):
    """-> (ptau bytes, responseHash, nextChallenge)"""
    return _apply(ptau, rng, 0, p2o._name_param(name))


def beacon(ptau: bytes, beacon_hash: bytes, e: int, name=None):
    rng = p2.rng_from_beacon(beacon_hash, e)
    params = p2o._name_param(name) + bytes([2, e, 3, len(beacon_hash)]) + bytes(beacon_hash)
    return _apply(ptau, rng, 1, params)
