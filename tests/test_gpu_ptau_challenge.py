"""A phase-1 ceremony by challenge and response on the GPU (snarkjs `powersoftau export challenge`, `challenge contribute`
and `import response`): the ffjavascript decoder (b200zk_points_decode_dev) exact against the encoder and the host
restatements, the three steps byte for byte against tests/challenge_oracle.py, export -> challenge contribute -> import
byte for byte against a direct contribution, and the refusals."""
import ctypes
import os
import struct
import sys
import warnings

import numpy as np
import pytest

from distributed_groth16_b200 import _native
from distributed_groth16_b200._native import c_vp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
_QL = [np.uint64((Q >> (64 * j)) & 0xFFFFFFFFFFFFFFFF) for j in range(4)]
SEEDS = ([0xC1, 2, 3, 4, 5, 6, 7, 8], [0xD2, 9, 10, 11, 12, 13, 14, 15])


def _negate_rows(a, rows, w):
    """-P for the given rows of a host (n, w) u64 array of affine Montgomery points: y -> q - y limb-wise."""
    for c in range(w // 2, w, 4):
        y = a[rows, c:c + 4]
        out = np.empty_like(y)
        borrow = np.zeros(len(rows), dtype=np.uint64)
        for j in range(4):
            t = y[:, j] + borrow
            nb = ((t < y[:, j]) | (t > _QL[j])).astype(np.uint64)
            out[:, j] = _QL[j] - t
            borrow = nb
        a[rows, c:c + 4] = out


def _points(net, g2, n, seed):
    """n generated points, every fifth negated, a few at infinity (host u64 array)."""
    pts = (net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)).cpu().numpy().view(np.uint64).copy()
    _negate_rows(pts, np.arange(0, n, 5), 16 if g2 else 8)
    pts[np.unique(np.random.default_rng(seed).integers(0, n, size=min(n, 7)))] = 0
    pts[0] = 0
    return pts


def _decode_raw(net, enc, g2, fmt, check, n=None):
    """-> (rc, n_invalid, first_invalid, points) from the C entry."""
    import torch
    n = enc.shape[0] if n is None else n
    out = torch.full((n, 16 if g2 else 8), 7, dtype=torch.int64, device=enc.device)
    bad, first = ctypes.c_size_t(99), ctypes.c_size_t(99)
    rc = net._lib.b200zk_points_decode_dev(net._h, 0, int(g2), c_vp(enc.data_ptr()), n, fmt, check, c_vp(out.data_ptr()),
                                           ctypes.byref(bad), ctypes.byref(first))
    return rc, bad.value, first.value, out


# ---- the decoder -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("g2,n", [(False, 1), (False, 1000), (False, 1 << 23), (True, 1), (True, 1000), (True, 1 << 22)])
def test_decode_inverts_encode(net, g2, n):
    import torch
    from distributed_groth16_b200.groth16 import phase1
    pts = net.to_device(_points(net, g2, n, 0xDEC0 + n + g2))
    for compressed in (False, True):
        enc = phase1.points_encode(net, pts, g2, compressed)
        back = phase1.points_decode(net, enc, g2, compressed, check_subgroup=g2)
        assert torch.equal(back, pts), (n, compressed)
    del pts, enc, back
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("g2", [False, True])
def test_decode_host_restatements(net, g2):
    """Bytes made on the host (phase2.u_g1 / u_g2, phase1.c_g1 / c_g2) decode to the same points, 2^12 of them."""
    import torch
    from distributed_groth16_b200.groth16 import phase1, phase2
    n = 1 << 12
    pts = _points(net, g2, n, 0xB0B + g2)
    for compressed, f in ((False, phase2.u_g2 if g2 else phase2.u_g1), (True, phase1.c_g2 if g2 else phase1.c_g1)):
        blob = b"".join(f(p) for p in pts)
        got = phase1.points_decode(net, blob, g2, compressed).cpu().numpy().view(np.uint64)
        assert (got == pts).all(), compressed


@pytest.mark.gpu
@pytest.mark.parametrize("g2,compressed", [(False, False), (False, True), (True, False), (True, True)])
def test_decode_planted_invalid(net, g2, compressed):
    """Invalid encodings at known indices: exact n_invalid / first_invalid, ERR_ARG, infinity in those slots and the right
    points everywhere else."""
    import torch
    import challenge_oracle as co
    from distributed_groth16_b200.groth16 import phase1
    n = 3000
    pts = net.to_device(_points(net, g2, n, 0x1A7 + 2 * g2 + compressed))
    enc = phase1.points_encode(net, pts, g2, compressed).cpu().numpy()
    w = enc.shape[1]
    q = Q.to_bytes(32, "big")
    bad = {2999: q + bytes(w - 32), 1234: b"\xC0" + bytes(w - 1), 17: None, 640: None}
    # a non-curve x (compressed) / a point off the curve (uncompressed) and the 0x80 flag on an uncompressed point
    x0 = co.non_curve_x(g2).to_bytes(32, "big")
    bad[17] = ((bytes(32) + x0) if g2 else x0) if compressed else bytes(enc[18][:w - 1]) + bytes([enc[18][w - 1] ^ 1])
    bad[640] = bytes([enc[641][0] | 0x80]) + bytes(enc[641][1:]) if not compressed else bytes([0x41]) + bytes(w - 1)
    for i, b in bad.items():
        enc[i] = np.frombuffer(b, dtype=np.uint8)
    d = net.to_device(enc)
    rc, nbad, first, out = _decode_raw(net, d, g2, int(compressed), 0)
    assert rc == _native.ERR_ARG and (nbad, first) == (4, 17)
    msg = net._lib.b200zk_last_error(net._h)
    assert b"4 of 3000" in msg and b"index 17" in msg, msg
    keep = torch.ones(n, dtype=torch.bool, device=out.device)
    keep[list(bad)] = False
    assert torch.equal(out[keep], pts[keep])
    assert not out[~keep].any()
    with pytest.raises(phase1.InvalidEncodings) as e:
        phase1.points_decode(net, d, g2, compressed)
    assert (e.value.count, e.value.first) == (4, 17)
    # all valid: the counters say so
    rc, nbad, first, _ = _decode_raw(net, net.to_device(enc[1:2]), g2, int(compressed), 0)
    assert (rc, nbad, first) == (_native.OK, 0, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("compressed", [False, True])
def test_decode_subgroup_flag(net, compressed):
    import challenge_oracle as co
    import phase1_oracle as po
    from oracle import layout
    rogue = co.rogue_g2()
    good = layout.arr_to_g2(net.generate_g2(5, 3).cpu().numpy().view(np.uint64))
    f = po.c_g2 if compressed else po.u_g2
    blob = f(good[0]) + f(rogue) + f(good[1]) + f(rogue) + f(None)
    d = net.to_device(np.frombuffer(bytearray(blob), dtype=np.uint8))
    rc, nbad, first, out = _decode_raw(net, d, True, int(compressed), 0, n=5)
    assert (rc, nbad) == (_native.OK, 0)
    assert (out[1].cpu().numpy().view(np.uint64) == layout.g2_to_arr([rogue])[0]).all()
    rc, nbad, first, out = _decode_raw(net, d, True, int(compressed), 1, n=5)
    assert (rc, nbad, first) == (_native.ERR_ARG, 2, 1)
    assert not out[1].any() and not out[3].any() and not out[4].any()
    assert (out[2].cpu().numpy().view(np.uint64) == layout.g2_to_arr([good[1]])[0]).all()


@pytest.mark.gpu
def test_decode_arguments(net):
    import torch
    lib = net._lib
    d = torch.zeros(64 * 4, dtype=torch.uint8, device="cuda")
    out = torch.zeros((4, 8), dtype=torch.int64, device="cuda")
    bad, first = ctypes.c_size_t(5), ctypes.c_size_t(5)
    call = lambda b, n, fmt, o: lib.b200zk_points_decode_dev(net._h, 0, 0, b, n, fmt, 0, o, ctypes.byref(bad), ctypes.byref(first))
    assert call(None, 4, 0, c_vp(out.data_ptr())) == _native.ERR_ARG
    assert call(c_vp(d.data_ptr()), 4, 0, None) == _native.ERR_ARG
    assert call(c_vp(d.data_ptr()), 4, 2, c_vp(out.data_ptr())) == _native.ERR_ARG
    assert call(c_vp(d.data_ptr() + 1), 1, 0, c_vp(out.data_ptr())) == _native.ERR_ARG
    before = net.launch_count()
    assert call(None, 0, 0, None) == _native.OK and (bad.value, first.value) == (0, 0)
    assert net.launch_count() == before
    assert lib.b200zk_points_decode_dev(net._h, 0, 0, None, 0, 1, 0, None, None, None) == _native.OK


# ---- the three steps against the Python restatement -----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("power", [1, 2])
def test_challenge_response_equal_the_oracle(net, tmp_path, power):
    import challenge_oracle as co
    import phase1_oracle as po
    from distributed_groth16_b200.groth16 import phase1, phase2
    p0, ch, rs, p1 = (str(tmp_path / f) for f in ("p0.ptau", "c.bin", "r.bin", "p1.ptau"))
    phase1.new(p0, power)
    b0 = po.new(power)
    h = phase1.export_challenge(net, p0, ch, chunk=1)
    assert open(ch, "rb").read() == co.export_challenge(b0) and h == po.first_challenge_hash(power)
    got = phase1.challenge_contribute(net, ch, rs, phase2.ChaCha(SEEDS[0]), chunk=1)
    want_resp, wch, wrh = co.challenge_contribute(co.export_challenge(b0), phase2.ChaCha(SEEDS[0]))
    assert got == (wch, wrh)
    assert open(rs, "rb").read() == want_resp
    got = phase1.import_response(net, p0, rs, p1, name="remote", chunk=1)
    want, irh, inc = co.import_response(b0, want_resp, name="remote")
    assert got == (irh, inc)
    assert open(p1, "rb").read() == want
    ch2 = str(tmp_path / "c2.bin")
    phase1.export_challenge(net, p1, ch2, chunk=1)
    assert open(ch2, "rb").read() == co.export_challenge(want)


# ---- the central check: a round by challenge and response equals a direct contribution ------------------------------------
def _current_challenge(path):
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase1
    with formats.PTau(path, prepared=False) as pt:
        return phase1._last_challenge(pt, phase1._read_records(pt))


def _round(net, d, src, tag, seed, name, chunk):
    from distributed_groth16_b200.groth16 import circom, phase1, phase2
    ch, rs, imp, direct = (str(d / ("%s.%s" % (tag, e))) for e in ("challenge", "response", "imported.ptau", "direct.ptau"))
    assert circom.ptau_export_challenge(net, src, ch) == _current_challenge(src)
    chh, rh = phase1.challenge_contribute(net, ch, rs, phase2.ChaCha(seed), chunk=chunk)
    irh, inc = phase1.import_response(net, src, rs, imp, name=name, chunk=chunk)
    drh, dnc = phase1.contribute(net, src, direct, phase2.ChaCha(seed), name=name, chunk=chunk)
    assert (rh, irh, inc) == (drh, drh, dnc)
    assert open(imp, "rb").read() == open(direct, "rb").read()
    return dict(challenge=ch, response=rs, imported=imp)


@pytest.fixture(scope="module")
def rounds(net, tmp_path_factory):
    from distributed_groth16_b200.groth16 import phase1
    d = tmp_path_factory.mktemp("challenge")
    p0 = str(d / "p0.ptau")
    phase1.new(p0, 15)
    r1 = _round(net, d, p0, "r1", SEEDS[0], "first remote", 1 << 22)
    r2 = _round(net, d, r1["imported"], "r2", SEEDS[1], "second remote", 5000)
    return dict(dir=d, p0=p0, r1=r1, r2=r2)


@pytest.mark.gpu
def test_round_trip_equals_contribute_and_verifies(net, rounds):
    from distributed_groth16_b200.groth16 import circom
    for k, r in enumerate((rounds["r1"], rounds["r2"])):
        rep = circom.ptau_verify(net, r["imported"])
        assert rep.ok, (k, rep.failures)
        assert [c[0] for c in rep.contributions] == ["first remote", "second remote"][:k + 1]


@pytest.mark.gpu
def test_round_trip_at_power_20(net, tmp_path):
    from distributed_groth16_b200.groth16 import phase1
    p0 = str(tmp_path / "p0.ptau")
    phase1.new(p0, 20)
    _round(net, tmp_path, p0, "r20", SEEDS[1], None, 1 << 18)


# ---- refusals -------------------------------------------------------------------------------------------------------------
def _copy_with(path, dst, patch):
    b = bytearray(open(path, "rb").read())
    patch(b)
    open(dst, "wb").write(bytes(b))
    return dst


@pytest.mark.gpu
def test_refuses_foreign_and_wrong_sized_files(net, rounds, tmp_path):
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase1, phase2
    r1, r2 = rounds["r1"], rounds["r2"]
    out = str(tmp_path / "out.ptau")
    with pytest.raises(ValueError) as e:                           # the round-2 response does not answer p0's challenge
        phase1.import_response(net, rounds["p0"], r2["response"], out)
    assert open(r2["response"], "rb").read(64).hex() in str(e.value)
    assert not os.path.exists(out)
    for path, cut in ((r1["challenge"], -1), (r1["challenge"], 1)):
        bad = _copy_with(path, str(tmp_path / "c.bin"), lambda b: b.__delitem__(-1) if cut < 0 else b.append(0))
        with pytest.raises(formats.FormatError):
            phase1.challenge_contribute(net, bad, str(tmp_path / "r.bin"), phase2.ChaCha(SEEDS[0]))
        assert not os.path.exists(str(tmp_path / "r.bin"))
    for cut in (-1, 1):
        bad = _copy_with(r1["response"], str(tmp_path / "r.bin"), lambda b: b.__delitem__(-1) if cut < 0 else b.append(0))
        with pytest.raises(formats.FormatError):
            phase1.import_response(net, rounds["p0"], bad, out)
        assert not os.path.exists(out)


@pytest.mark.gpu
def test_refuses_invalid_response_points(net, rounds, tmp_path):
    import challenge_oracle as co
    import phase1_oracle as po
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase1
    n = 1 << 15
    s3 = 64 + (2 * n - 1) * 32
    s6 = s3 + n * 64 + 2 * n * 32
    out = str(tmp_path / "out.ptau")
    x0 = bytes(32) + co.non_curve_x(True).to_bytes(32, "big")
    bad = _copy_with(rounds["r1"]["response"], str(tmp_path / "r.bin"), lambda b: b.__setitem__(slice(s3 + 17 * 64, s3 + 18 * 64), x0))
    with pytest.raises(formats.FormatError, match=r"section 3: 1 points .* point 17"):
        phase1.import_response(net, rounds["p0"], bad, out)
    assert not os.path.exists(out)
    rogue = po.c_g2(co.rogue_g2())
    bad = _copy_with(rounds["r1"]["response"], str(tmp_path / "r.bin"), lambda b: b.__setitem__(slice(s6, s6 + 64), rogue))
    with pytest.raises(formats.FormatError, match=r"section 6: .*subgroup.* point 0"):
        phase1.import_response(net, rounds["p0"], bad, out)
    assert not os.path.exists(out)


@pytest.mark.gpu
def test_flipped_flag_imports_and_verify_names_section_4(net, rounds, tmp_path):
    from distributed_groth16_b200.groth16 import phase1
    n = 1 << 15
    s4 = 64 + (2 * n - 1) * 32 + n * 64
    out = str(tmp_path / "flipped.ptau")
    bad = _copy_with(rounds["r1"]["response"], str(tmp_path / "r.bin"), lambda b: b.__setitem__(s4 + 3 * 32, b[s4 + 3 * 32] ^ 0x80))
    phase1.import_response(net, rounds["p0"], bad, out)
    rep = phase1.verify(net, out)
    assert not rep.ok and any("section 4" in f for f in rep.failures), rep.failures


@pytest.mark.gpu
def test_export_refuses_a_tampered_file(net, rounds, tmp_path):
    from distributed_groth16_b200.groth16 import phase1
    src = rounds["r1"]["imported"]
    buf = open(src, "rb").read()
    off = 12
    while struct.unpack_from("<I", buf, off)[0] != 5:
        off += 12 + struct.unpack_from("<Q", buf, off + 4)[0]
    off += 12
    # point 9 of section 5 replaced by the generator (a valid point, so only the hash can tell)
    bad = _copy_with(src, str(tmp_path / "t.ptau"), lambda b: b.__setitem__(slice(off + 9 * 64, off + 10 * 64),
                                                                          phase1.G1_GEN.astype("<u8").tobytes()))
    ch = str(tmp_path / "t.challenge")
    with pytest.raises(ValueError, match="current challenge"):
        phase1.export_challenge(net, bad, ch)
    assert not os.path.exists(ch)


@pytest.mark.gpu
def test_import_refuses_reduced_same_file_and_warns_on_prepared(net, rounds, tmp_path):
    from distributed_groth16_b200.groth16 import circom, phase1
    src, resp = rounds["r1"]["imported"], rounds["r2"]["response"]
    with pytest.raises(ValueError):
        phase1.import_response(net, src, resp, src)
    buf = bytearray(open(src, "rb").read())
    buf[12 + 12 + 40:12 + 12 + 44] = struct.pack("<I", 16)            # ceremonyPower 16 > power 15
    rp = str(tmp_path / "reduced.ptau")
    open(rp, "wb").write(bytes(buf))
    with pytest.raises(ValueError, match="reduced"):
        phase1.import_response(net, rp, resp, str(tmp_path / "x.ptau"))
    assert not os.path.exists(str(tmp_path / "x.ptau"))
    prep, out = str(tmp_path / "prep.ptau"), str(tmp_path / "after.ptau")
    circom.ptau_prepare_phase2(net, src, prep)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        circom.ptau_import_response(net, prep, resp, out, name="second remote")
    assert any("prepared" in str(w.message) for w in caught)
    assert open(out, "rb").read() == open(rounds["r2"]["imported"], "rb").read()
