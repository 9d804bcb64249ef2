"""The ffjavascript decoder of csrc/codec.cuh (ffjs_get / ffjs_decode, the device code of b200zk_points_decode_dev)
compiled for the host vs the Python restatements: round trips of both encodings of random points, their negatives and
infinity, and every kind of refusal."""
import os
import struct
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cases(cref):
    """[(g2, compressed, check_subgroup, valid, encoding, point or None)]"""
    from oracle import bn254 as o, layout
    import challenge_oracle as co
    import phase1_oracle as po
    enc = {(False, False): po.u_g1, (False, True): po.c_g1, (True, False): po.u_g2, (True, True): po.c_g2}
    pts1 = layout.arr_to_g1(cref.g1_generate(0xFF15, 24))
    pts2 = layout.arr_to_g2(cref.g2_generate(0xFF15, 8))
    cases = []
    for g2, pts in ((False, pts1), (True, pts2)):
        grp = o.G2 if g2 else o.G1
        for c in (False, True):
            for pt in pts + [grp.neg(p) for p in pts] + [None]:
                cases.append((g2, c, int(g2), 1, enc[(g2, c)](pt), pt))
    q = o.P.to_bytes(32, "big")
    p1, p2 = pts1[0], pts2[0]
    bad = []
    # x >= q (each Fq2 half on its own), y >= q
    bad += [(False, True, q), (False, False, q + po.u_g1(p1)[32:])]
    for c in (False, True):
        e = enc[(True, c)](p2)
        bad += [(True, c, q + e[32:]), (True, c, e[:32] + q + e[64:])]
    bad.append((False, False, po.u_g1(p1)[:32] + (p1[1] + o.P).to_bytes(32, "big")))
    e = po.u_g2(p2)
    bad += [(True, False, e[:64] + (p2[1][1] + o.P).to_bytes(32, "big") + e[96:]),
            (True, False, e[:96] + (p2[1][0] + o.P).to_bytes(32, "big"))]
    # a compressed x with no curve point; an uncompressed (x, y) off the curve
    bad += [(False, True, co.non_curve_x(False).to_bytes(32, "big")),
            (True, True, bytes(32) + co.non_curve_x(True).to_bytes(32, "big"))]
    bad += [(False, False, po.u_g1((p1[0], (p1[1] + 1) % o.P))),
            (True, False, po.u_g2((p2[0], (p2[1][0], (p2[1][1] + 1) % o.P))))]
    # infinity with any other bit set: the sign flag, a bit in byte 1, a bit in the last byte; 0x80 on an uncompressed point
    for g2 in (False, True):
        for c in (False, True):
            n = (64 if g2 else 32) * (1 if c else 2)
            bad += [(g2, c, b"\xC0" + bytes(n - 1)), (g2, c, b"\x40\x01" + bytes(n - 2)), (g2, c, b"\x40" + bytes(n - 2) + b"\x01"),
                    (g2, c, b"\x41" + bytes(n - 1))]
        u = enc[(g2, False)](p2 if g2 else p1)
        bad.append((g2, False, bytes([u[0] | 0x80]) + u[1:]))
    cases += [(g2, c, 0, 0, e, None) for g2, c, e in bad]
    # a twist point outside the subgroup: accepted without the check, refused with it
    rogue = co.rogue_g2()
    for c in (False, True):
        cases += [(True, c, 0, 1, enc[(True, c)](rogue), rogue), (True, c, 1, 0, enc[(True, c)](rogue), None)]
    return cases


def test_ffjs_decode_header_matches_the_oracle(tmp_path, cref):
    from oracle import layout
    import challenge_oracle as co
    cases = _cases(cref)
    # the Python restatement agrees with every vector first
    dec = {(False, False): co.dec_u_g1, (False, True): co.dec_c_g1, (True, False): co.dec_u_g2, (True, True): co.dec_c_g2}
    for g2, c, sub, valid, enc, pt in cases:
        try:
            got = dec[(g2, c)](enc, bool(sub)) if g2 else dec[(g2, c)](enc)
            ok = True
        except ValueError:
            ok = False
        assert ok == bool(valid) and (not ok or got == pt), (g2, c, sub, enc.hex())
    blob = struct.pack("<Q", len(cases))
    for g2, c, sub, valid, enc, pt in cases:
        arr = (layout.g2_to_arr if g2 else layout.g1_to_arr)([pt]).astype("<u8").reshape(-1)
        blob += struct.pack("<IIII", g2, c, sub, valid) + enc.ljust(128, b"\0") + \
            np.concatenate([arr, np.zeros(16 - arr.size, dtype="<u8")]).tobytes()
    vec = tmp_path / "ffjs_vectors.bin"
    vec.write_bytes(blob)
    exe = tmp_path / "ffjs_decode_host_test"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-o", str(exe),
                           os.path.join(ROOT, "tests", "host", "ffjs_decode_host_test.cpp")])
    out = subprocess.run([str(exe), str(vec)], capture_output=True, text=True)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout + out.stderr
    assert sum(1 for cs in cases if not cs[3]) >= 30
