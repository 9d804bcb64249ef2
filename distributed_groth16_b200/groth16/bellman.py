"""Phase 2 by challenge and response: snarkjs `zkey export bellman`, `zkey bellman contribute` and `zkey import bellman`
on the GPU.

A coordinated phase-2 ceremony passes bellman's MPC-params file around instead of the zkey (formats.parse_bellman has the
layout): the key's points in ffjavascript's uncompressed encoding, the csHash and one 384-byte public key per record.  It
differs from the zkey in one part, the H query.  zkey section 9 holds h_k = L^2n_(2k+1)(tau) delta^-1 G1, k < n (the odd
Lagrange points of the 2n domain); the file holds the tau basis

  H_i = tau^i (tau^n - 1) delta^-1 G1 = -2 w_2n^i sum_k w_n^(i k) h_k,   i < cshash.h_point_count(n),

a forward NTT over points (b200zk_points_ntt_dev) and one scalar per point (b200zk_points_mul_powers_dev, ffjavascript's
batchApplyKey(-2, w_2n)).  Import runs the inverse: H_(n-1), which the file does not carry, is taken as infinity, every
point is multiplied by -1/2 w_2n^-i and the point iNTT gives section 9 back.  An imported H therefore differs from the
original along the one tau component the prover never uses (h(X) has degree <= n - 2): proofs are unchanged, and
phase2.verify checks that component separately.

A contribution with secret x multiplies delta_1, delta_2 by x and the H and L points by x^-1 on the device, and appends
the record phase2 would append (the same transcript and hash-to-G2).  Bytes in, bytes out, as the rest of phase 2.

Pinned against snarkjs bytes: the export layout, the H basis change and the H count at domain 2^14, through the circuit
hash (Blake2b-512 of the part before the csHash is the csHash of a key with no contributions).  Pinned only against
this repository's restatement (tests/bellman_oracle.py): the record layout, the import rule for H_(n-1) and the
contributor step."""
from __future__ import annotations

import struct
import time
from contextlib import contextmanager

import numpy as np

from .. import formats
from . import cshash, phase1, phase2, ptau

R = formats.FR_MODULUS
MAX_LOG_DOMAIN = 27                               # w_2n must exist in Fr (two-adicity 28), as zkey_new's limit
_HDR_POINTS = 84                                  # offset of alpha_1 in the header section (2)
_G1, _G2 = 64, 128                                # bytes of one uncompressed encoding


def _root(n: int) -> int:
    """w_n, the root of unity of the device NTTs (Fr::GENERATOR = 5)."""
    return pow(5, (R - 1) // n, R)


def _timings() -> dict:
    return {k: 0.0 for k in ("ntt_s", "mul_powers_s", "decode_s", "scale_s", "encode_s", "transfer_s", "host_s")}


@contextmanager
def _stage(net, t: dict, key: str):
    """Seconds spent in the block, between two device synchronisations, added to t[key]."""
    net.sync(0)
    t0 = time.perf_counter()
    yield
    net.sync(0)
    t[key] += time.perf_counter() - t0


def _key_dims(zkey_bytes: bytes):
    hdr = phase2._section(zkey_bytes, 2)
    if len(hdr) < _HDR_POINTS + 576:
        raise formats.FormatError("zkey header section too short (%d bytes)" % len(hdr))
    n_vars, n_public, n = struct.unpack_from("<III", hdr, 72)
    if n == 0 or n & (n - 1):
        raise formats.FormatError("zkey header: domain size %d is not a power of two" % n)
    if n > 1 << MAX_LOG_DOMAIN:
        raise ValueError("a domain of 2^%d has no 2n-th root of unity in Fr: bellman params need a domain of at most 2^%d"
                         % (n.bit_length() - 1, MAX_LOG_DOMAIN))
    return hdr, n_vars, n_public, n


def _header_points(hdr: bytes) -> dict:
    """The six header points (alpha_1 .. delta_2) as Montgomery limbs, by formats.BELLMAN_HEADER name."""
    out, off = {}, _HDR_POINTS
    for part, w in formats.BELLMAN_HEADER:
        out[part] = np.frombuffer(hdr, dtype="<u8", count=w // 8, offset=off).copy()
        off += w
    return out


def _u(p, w: int) -> bytes:
    return phase2.u_g2(p) if w == _G2 else phase2.u_g1(p)


def _upload(net, raw: bytes, width: int, t: dict):
    with _stage(net, t, "transfer_s"):
        return net.to_device(np.frombuffer(raw, dtype="<u8").reshape(-1, width).copy())


def _encode(net, d, g2: bool, t: dict) -> bytes:
    if d.shape[0] == 0:
        return b""
    with _stage(net, t, "encode_s"):
        enc = phase1.points_encode(net, d, g2)
    with _stage(net, t, "transfer_s"):
        return enc.cpu().numpy().tobytes()


def _decode(net, raw: bytes, g2: bool, what: str, t: dict, check_subgroup: bool = False):
    """ffjavascript uncompressed encodings -> CUDA points; FormatError naming the part and the first bad index."""
    with _stage(net, t, "transfer_s"):
        enc = net.to_device(np.frombuffer(raw, dtype=np.uint8).copy())
    with _stage(net, t, "decode_s"):
        try:
            return phase1.points_decode(net, enc, g2, check_subgroup=check_subgroup)
        except phase1.InvalidEncodings as e:
            raise formats.FormatError("%s point %d is not a valid uncompressed %s point%s (%d invalid)"
                                      % (what, e.first, "G2" if g2 else "G1",
                                         " of the order-r subgroup" if check_subgroup else "", e.count)) from None


def _h_to_tau(net, sec9: bytes, n: int, t: dict):
    """Section 9 (n Lagrange-form points) -> the first h_point_count(n) points of the tau basis, on the device."""
    if len(sec9) != n * _G1:
        raise formats.FormatError("zkey section 9 holds %d bytes, a domain of %d needs %d" % (len(sec9), n, n * _G1))
    d = _upload(net, sec9, 8, t)
    with _stage(net, t, "ntt_s"):
        ptau.points_ntt(net, d, out=d)
    with _stage(net, t, "mul_powers_s"):
        phase1.points_mul_powers(net, d, R - 2, _root(2 * n), out=d)
    return d[:cshash.h_point_count(n)]


def _h_from_tau(net, h, n: int, t: dict):
    """The inverse of _h_to_tau: the tau-basis points h (CUDA) with infinity past their end -> section 9 (CUDA)."""
    import torch
    d = torch.zeros((n, 8), dtype=torch.int64, device=h.device)
    d[:h.shape[0]] = h
    with _stage(net, t, "mul_powers_s"):
        phase1.points_mul_powers(net, d, R - pow(2, -1, R), pow(_root(2 * n), -1, R), out=d)
    with _stage(net, t, "ntt_s"):
        ptau.points_intt(net, d, out=d)
    return d


def _export_parts(net, zkey_bytes: bytes, t: dict, with_h: bool = True):
    """The encoded parts of the key's bellman params by name (formats.BELLMAN_HEADER and BELLMAN_VECTORS; "h" only with
    with_h), their counts, and the key's section 10 (formats.MPCParams)."""
    hdr, n_vars, n_public, n = _key_dims(zkey_bytes)
    with _stage(net, t, "host_s"):
        mpc = formats.read_mpc_params(zkey_bytes)
        parts = {part: _u(p, w) for (part, w), p in zip(formats.BELLMAN_HEADER, _header_points(hdr).values())}
    counts = {"ic": n_public + 1, "h": cshash.h_point_count(n), "l": n_vars - n_public - 1, "a": n_vars, "b1": n_vars,
              "b2": n_vars}
    for part, sid, w in (("ic", 3, _G1), ("l", 8, _G1), ("a", 5, _G1), ("b1", 6, _G1), ("b2", 7, _G2)):
        sec = phase2._section(zkey_bytes, sid)
        if len(sec) != counts[part] * w:
            raise formats.FormatError("zkey section %d holds %d bytes, the header's counts give %d"
                                      % (sid, len(sec), counts[part] * w))
        parts[part] = _encode(net, _upload(net, sec, w // 8, t), w == _G2, t)
    if with_h:
        parts["h"] = _encode(net, _h_to_tau(net, phase2._section(zkey_bytes, 9), n, t), False, t)
    return parts, counts, mpc


def export(net, zkey_bytes: bytes, timings: dict | None = None) -> bytes:
    """snarkjs `zkey export bellman <zkey> <params>`: the MPC-params bytes of the key (every section encoded on the device,
    H moved to the tau basis there).  Every record of section 10 goes out as its public key; bellman has no types or
    names."""
    t = _timings()
    parts, counts, mpc = _export_parts(net, zkey_bytes, t)
    with _stage(net, t, "host_s"):
        out = [parts[p] for p, _ in formats.BELLMAN_HEADER]
        for p, _ in formats.BELLMAN_VECTORS:
            out += [struct.pack(">I", counts[p]), parts[p]]
        out += [bytes(mpc.cs_hash), struct.pack(">I", len(mpc.contributions))]
        out += [phase2.hash_pub_key(c) for c in mpc.contributions]
        out = b"".join(out)
    if timings is not None:
        timings.update(t)
    return out


def contribute(net, challenge: bytes, x: int, g1_s, timings: dict | None = None):
    """snarkjs `zkey bellman contribute bn128 <challenge> <response>` with a known secret x (non-zero mod r) and
    proof-of-knowledge base g1_s (8 Montgomery limbs): H and L decoded on the device with the curve check and multiplied by
    x^-1, delta_1 and delta_2 by x, the record of phase2.contribute appended; every other byte is copied.  Returns
    (response bytes, contribution hash)."""
    x %= R
    if x == 0:
        raise ValueError("the contribution secret must be non-zero mod r")
    t = _timings()
    with _stage(net, t, "host_s"):
        b = formats.parse_bellman(challenge)
        out = bytearray(challenge)
    xinv = pow(x, -1, R)
    for part in ("h", "l"):
        off, ln = b.spans[part]
        if not ln:
            continue
        d = _decode(net, challenge[off:off + ln], False, "challenge: " + part.upper(), t)
        with _stage(net, t, "scale_s"):
            phase2.points_scale(net, d, xinv, out=d)
        out[off:off + ln] = _encode(net, d, False, t)
    deltas = {}
    for part, g2 in (("delta_g1", False), ("delta_g2", True)):
        off, ln = b.spans[part]
        p = _decode(net, challenge[off:off + ln], g2, "challenge: " + part, t, check_subgroup=g2)
        with _stage(net, t, "scale_s"):
            deltas[part] = phase2._scale_one(net, p.cpu().numpy().view(np.uint64)[0], x, g2)
        out[off:off + ln] = _u(deltas[part], ln)
    with _stage(net, t, "host_s"):                     # the record: proof of knowledge, transcript, hash-to-G2
        g1_s = np.ascontiguousarray(g1_s, dtype=np.uint64).reshape(-1)
        g1_sx = phase2._scale_one(net, g1_s, x)
        tr = phase2.transcript(b.cs_hash, b.contributions, g1_s, g1_sx)
        g2_spx = phase2._scale_one(net, phase2.hash_to_g2(net, tr), x, g2=True)
        c = formats.Contribution(delta_after=deltas["delta_g1"], g1_s=g1_s, g1_sx=g1_sx, g2_spx=g2_spx, transcript=tr)
        out[b.params_end + 64:b.params_end + 68] = struct.pack(">I", len(b.contributions) + 1)
        out += phase2.hash_pub_key(c)
    if timings is not None:
        timings.update(t)
    return bytes(out), phase2.contribution_hash(c)


def _first_difference(a: bytes, b: bytes, w: int) -> int:
    return next(i for i in range(0, len(a), w) if a[i:i + w] != b[i:i + w]) // w


def import_response(net, zkey_bytes: bytes, response: bytes, name: str | None = None,
                    timings: dict | None = None) -> bytes:
    """snarkjs `zkey import bellman <zkey> <response> <dst>`: the key with the response's delta, L and H (section 9
    rebuilt from the tau basis) and its new records appended as type-0 records named `name`; the key's own records are
    kept as they are.  The response must answer this key: its csHash, its earlier records, every point but delta, L and
    H, and every count equal the key's export.  Points are decoded on the device (delta_2 and the new records' G2 points
    with the subgroup check).  Like snarkjs it runs no pairing check; phase2.verify checks the contribution.  Raises
    FormatError for a malformed response and ValueError for one that does not answer this key, naming the part and
    the index."""
    if name is not None and len(name.encode("utf-8")) > 64:
        raise ValueError("contribution name longer than 64 bytes")
    t = _timings()
    with _stage(net, t, "host_s"):
        b = formats.parse_bellman(response)
    parts, counts, mpc = _export_parts(net, zkey_bytes, t, with_h=False)
    for part, _ in formats.BELLMAN_VECTORS:
        if b.counts[part] != counts[part]:
            raise ValueError("response: %s holds %d points, the key's %d" % (part.upper(), b.counts[part], counts[part]))
    if bytes(b.cs_hash) != bytes(mpc.cs_hash):
        raise ValueError("response: its csHash %s... is not the key's %s...: it answers another key"
                         % (bytes(b.cs_hash)[:8].hex(), bytes(mpc.cs_hash)[:8].hex()))
    old, k = len(mpc.contributions), len(b.contributions)
    if k <= old:
        raise ValueError("response: %d records, the key already has %d: it holds no new contribution" % (k, old))
    for i, c in enumerate(mpc.contributions):
        off = b.records_offset + formats.BELLMAN_RECORD * i
        if response[off:off + formats.BELLMAN_RECORD] != phase2.hash_pub_key(c):
            raise ValueError("response: record %d differs from the key's record %d" % (i, i))
    for part, w in formats.BELLMAN_HEADER + formats.BELLMAN_VECTORS:
        if part in ("delta_g1", "delta_g2", "h", "l"):
            continue
        off, ln = b.spans[part]
        if response[off:off + ln] != parts[part]:
            raise ValueError("response: %s point %d differs from the key's"
                             % (part, _first_difference(response[off:off + ln], parts[part], w)))
    span = lambda part: response[b.spans[part][0]:b.spans[part][0] + b.spans[part][1]]
    host = lambda d: d.cpu().numpy().view(np.uint64)
    d1 = host(_decode(net, span("delta_g1"), False, "response: delta_g1", t))[0].copy()
    d2 = host(_decode(net, span("delta_g2"), True, "response: delta_g2", t, check_subgroup=True))[0].copy()
    new = response[b.records_offset + formats.BELLMAN_RECORD * old:]
    recs = [new[j:j + formats.BELLMAN_RECORD] for j in range(0, len(new), formats.BELLMAN_RECORD)]
    g1 = host(_decode(net, b"".join(r[:192] for r in recs), False, "response: new record G1", t)).reshape(-1, 3, 8)
    g2 = host(_decode(net, b"".join(r[192:320] for r in recs), True, "response: new record g2_spx", t, check_subgroup=True))
    added = [formats.Contribution(delta_after=g1[j, 0].copy(), g1_s=g1[j, 1].copy(), g1_sx=g1[j, 2].copy(),
                                  g2_spx=g2[j].copy(), transcript=recs[j][320:], type=0, name=name)
             for j in range(len(recs))]
    if not (added[-1].delta_after == d1).all():
        raise ValueError("response: delta_g1 is not the last record's deltaAfter")
    l_pts = _decode(net, span("l"), False, "response: L", t) if b.counts["l"] else None
    h_pts = _decode(net, span("h"), False, "response: H", t)
    n = _key_dims(zkey_bytes)[3]
    h_sec = _h_from_tau(net, h_pts, n, t)
    with _stage(net, t, "transfer_s"):
        sec9 = h_sec.cpu().numpy().tobytes()
        sec8 = l_pts.cpu().numpy().tobytes() if l_pts is not None else b""
    with _stage(net, t, "host_s"):
        hdr = phase2._section(zkey_bytes, 2)
        d = phase2._HDR_DELTA
        new_hdr = hdr[:d] + d1.astype("<u8").tobytes() + d2.astype("<u8").tobytes() + hdr[d + 192:]
        sec10 = formats.mpc_params_bytes(formats.MPCParams(cs_hash=mpc.cs_hash, contributions=mpc.contributions + added))
        out = phase2._replace_sections(zkey_bytes, {2: new_hdr, 8: sec8, 9: sec9, 10: sec10})
    if timings is not None:
        timings.update(t)
    return out
