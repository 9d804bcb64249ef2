"""The circuit hash (csHash) of snarkjs `zkey new` on the GPU: the first 64 bytes of zkey section 10, which every phase-2
transcript starts from and which snarkjs `zkey verify` recomputes.

csHash = Blake2b-512 of, in this order (U = ffjavascript toRprUncompressed, u32 = a big-endian 32-bit count):

  U(alpha_1) U(beta_1) U(beta_2)                         the first points of ptau sections 4, 5, 6
  U(gamma_2) U(delta_1) U(delta_2)                       the generators of a fresh key (G2, G1, G2)
  u32(n_public + 1)  U(IC_i)                             zkey section 3
  u32(h_point_count(n))  U(H_i)                          H_i = tau^(n+i) G1 - tau^i G1 from ptau section 2, n = domain
  u32(n_vars - n_public - 1)  U(C_i)                     zkey section 8
  u32(n_vars)  U(A_i), then the same for B1 and B2       zkey sections 5, 6, 7, points at infinity included

The H points are not the Lagrange form that zkey section 9 stores.  They stream from section 2 in chunks: two slices of
tau powers to the device, b200zk_points_sub_dev, b200zk_points_encode_dev, the encodings to the host, Blake2b.  Every
other section is encoded on the device from the key points `setup.ptau_key_points` returns.

Checked against snarkjs at domain 2^14: the reference's complex-circuit zkey (written by snarkjs `zkey new`) carries the
hash this module computes from its own points (tests/test_zkey_cshash_formats.py, tests/test_gpu_zkey_cshash.py).
Open for domains of 2^15 and above: see h_point_count."""
from __future__ import annotations

import hashlib
import struct
import time

from .. import formats
from . import phase1, phase2

DEFAULT_CHUNK = phase1.DEFAULT_CHUNK


def h_point_count(domain_size: int) -> int:
    """How many H points the circuit hash covers: n - 1, the count its length prefix states.  snarkjs hashes them in
    chunks of 2^14, and its chunk loop may hash min(n - 1, 2^14) points per chunk, which is n points, not n - 1, once
    n >= 2^15.  The reference zkey (n = 2^14) cannot tell the two apart; a snarkjs key of a larger domain can."""
    return int(domain_size) - 1


def _timings() -> dict:
    return {"sub_s": 0.0, "encode_s": 0.0, "copy_s": 0.0, "hash_s": 0.0, "file_s": 0.0}


def _hash_encoded(net, h, d, g2: bool, t: dict) -> None:
    """U of the CUDA points d, encoded on the device and fed to h."""
    t0 = time.perf_counter()
    enc = phase1.points_encode(net, d, g2, compressed=False)
    net.sync(0)
    t1 = time.perf_counter()
    enc = enc.cpu().numpy()
    t2 = time.perf_counter()
    h.update(enc)
    t3 = time.perf_counter()
    t["encode_s"] += t1 - t0
    t["copy_s"] += t2 - t1
    t["hash_s"] += t3 - t2


def _hash_section(net, h, pts, g2: bool, chunk: int, t: dict) -> None:
    n = int(pts.shape[0])
    h.update(struct.pack(">I", n))
    for lo in range(0, n, chunk):
        _hash_encoded(net, h, pts[lo:lo + chunk], g2, t)


def _hash_h_points(net, h, pt, n: int, chunk: int, t: dict) -> None:
    count = h_point_count(n)
    if not pt.has_section(2):
        raise formats.FormatError("ptau section 2 (tau^i G1) missing: the circuit hash needs it")
    have = pt.section_span(2)[1] // 64
    if have < n + count:
        raise formats.FormatError("ptau section 2 holds %d points, the circuit hash of a domain of 2^%d needs %d"
                                  % (have, n.bit_length() - 1, n + count))
    h.update(struct.pack(">I", count))
    for lo in range(0, count, chunk):
        cnt = min(chunk, count - lo)
        t0 = time.perf_counter()
        hi, lo_pts = pt.points(2, n + lo, cnt, 8), pt.points(2, lo, cnt, 8)
        t1 = time.perf_counter()
        a, b = net.to_device(hi), net.to_device(lo_pts)
        net.sync(0)
        t2 = time.perf_counter()
        phase1.points_sub(net, a, b, out=a)
        net.sync(0)
        t3 = time.perf_counter()
        t["file_s"] += t1 - t0
        t["copy_s"] += t2 - t1
        t["sub_s"] += t3 - t2
        _hash_encoded(net, h, a, False, t)


def cs_hash(net, q: dict, pt, chunk: int = DEFAULT_CHUNK, timings: dict | None = None) -> bytes:
    """The 64-byte csHash of the key points q (setup.ptau_key_points of a circuit and the prepared ceremony pt, a
    formats.PTau) as snarkjs `zkey new` computes it; pt also gives the tau powers of section 2.  chunk: points per device
    call (host memory holds one chunk of encodings).  timings, when given, is filled with seconds spent in the sub kernel,
    the encode kernel, host <-> device copies, host Blake2b and file reads."""
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError("cs_hash: chunk must be positive, got %d" % chunk)
    t = _timings()
    h = hashlib.blake2b(digest_size=64)
    t0 = time.perf_counter()
    h.update(phase2.u_g1(q["alpha_g1"]) + phase2.u_g1(q["beta_g1"]) + phase2.u_g2(q["beta_g2"]) +
             phase2.u_g2(q["gamma_g2"]) + phase2.u_g1(q["delta_g1"]) + phase2.u_g2(q["delta_g2"]))
    t["hash_s"] += time.perf_counter() - t0
    _hash_section(net, h, q["ic"], False, chunk, t)
    _hash_h_points(net, h, pt, int(q["domain_size"]), chunk, t)
    _hash_section(net, h, q["l_query"], False, chunk, t)
    _hash_section(net, h, q["a_query"], False, chunk, t)
    _hash_section(net, h, q["b_g1_query"], False, chunk, t)
    _hash_section(net, h, q["b_g2_query"], True, chunk, t)
    t0 = time.perf_counter()
    out = h.digest()
    t["hash_s"] += time.perf_counter() - t0
    if timings is not None:
        timings.update(t)
    return out
