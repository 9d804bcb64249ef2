"""snarkjs `powersoftau prepare phase2` on the GPU: the inverse NTT over points (b200zk_points_intt_dev) exact at every size
up to the top levels of a power-22 ceremony, its error codes and aliasing contract, prepared files byte for byte against
the test-side ptau writer (pure-Python oracle and pinned GPU building blocks), and the Lagrange check on good and tampered
files."""
import os
import struct
import sys

import numpy as np
import pytest

from distributed_groth16_b200 import _native
from distributed_groth16_b200._native import c_vp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")
TOXIC = (0x1234567890ABCDEF1234567890ABCDEF, 11111111111111111111, 22222222222222222223)
R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def _mont(net, ints):
    """canonical ints (any size < r) -> Montgomery limbs on the device (fr_convert)."""
    arr = np.array([[(int(v) % R >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] for v in ints], dtype=np.uint64)
    return net.fr_convert(net.to_device(arr.reshape(-1, 4)), to_mont=True)


def _mont_u64(net, logs):
    """(n,) uint64 -> Montgomery limbs on the device."""
    arr = np.zeros((len(logs), 4), dtype=np.uint64)
    arr[:, 0] = logs
    return net.fr_convert(net.to_device(arr), to_mont=True)


def _expected(net, scalars, g2):
    """fixed_base_mul(ntt(scalars, inverse)): the points of the inverse NTT of the logs, from pinned building blocks."""
    from distributed_groth16_b200.groth16.setup import _fixed_base
    return _fixed_base(net, net.ntt_dev(scalars, inverse=True), g2)


def _intt(net, pts, g2, out=None):
    from distributed_groth16_b200.groth16 import ptau
    r = ptau.points_intt(net, pts, g2, out=out)
    net.sync(0)
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("g2,log_n", [(False, k) for k in (0, 1, 2, 3, 5, 8, 11, 16, 20, 23)] +
                         [(True, k) for k in (0, 1, 2, 5, 8, 12, 18, 22)])
def test_points_intt_exact(net, g2, log_n):
    """Generated bases P_j = k_j G (known logs) with some set to infinity (log 0): the transform equals the generator times
    the field inverse NTT of the logs, point for point."""
    import torch
    import dlog_oracle
    n, seed = 1 << log_n, 0x1A7 + 31 * log_n + g2
    pts = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
    logs = dlog_oracle.base_logs(seed, n)
    inf = np.unique(np.random.default_rng(log_n).integers(0, n, size=min(n // 2, 5)))
    if n > 1:
        logs[inf] = 0
        pts[torch.from_numpy(inf).to(pts.device)] = 0
    want = _expected(net, _mont_u64(net, logs), g2)
    got = _intt(net, pts, g2)
    assert torch.equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("g2", [False, True])
@pytest.mark.parametrize("log_n", [1, 3, 8])
@pytest.mark.parametrize("kind", ["all_equal", "antipodal", "all_infinity"])
def test_points_intt_adversarial(net, g2, log_n, kind):
    """All points equal (every output but index 0 is infinity), P_{j + n/2} = -P_j (the first pass cancels to the
    identity), and all points infinity."""
    import torch
    from distributed_groth16_b200.groth16.setup import _fixed_base
    n = 1 << log_n
    rng = np.random.default_rng(n + 2 * g2)
    base = [int.from_bytes(rng.bytes(32), "little") % R for _ in range(n // 2)]
    logs = {"all_equal": [base[0]] * n, "antipodal": base + [R - v for v in base], "all_infinity": [0] * n}[kind]
    s = _mont(net, logs)
    pts = _fixed_base(net, s, g2)
    got = _intt(net, pts, g2)
    assert torch.equal(got, _expected(net, s, g2))
    if kind == "all_equal":
        assert not got[1:].any() and torch.equal(got[0], pts[0])
    if kind == "all_infinity":
        assert not got.any()


@pytest.mark.gpu
def test_points_intt_error_codes_and_aliasing(net):
    """log_n = 29: ERR_DOMAIN; a null pointer: ERR_ARG; nothing faults.  d_out == d_in (the documented in-place case)
    gives the out-of-place result."""
    import torch
    lib, h = net._lib, net._h
    pts = net.generate_g1(77, 1 << 10)
    buf = torch.empty_like(pts)
    assert lib.b200zk_points_intt_dev(h, 0, 0, c_vp(pts.data_ptr()), 29, c_vp(buf.data_ptr())) == _native.ERR_DOMAIN
    assert lib.b200zk_points_intt_dev(h, 0, 0, None, 10, c_vp(buf.data_ptr())) == _native.ERR_ARG
    assert lib.b200zk_points_intt_dev(h, 0, 1, c_vp(pts.data_ptr()), 10, None) == _native.ERR_ARG
    assert lib.b200zk_points_intt_dev(None, 0, 0, c_vp(pts.data_ptr()), 10, c_vp(buf.data_ptr())) == _native.ERR_ARG
    for g2, log_n in ((False, 10), (True, 6)):
        p = net.generate_g2(78, 1 << log_n) if g2 else net.generate_g1(78, 1 << log_n)
        inplace = p.clone()
        want = _intt(net, p, g2)
        assert torch.equal(p, inplace)                          # out of place: the input is left as it was
        _intt(net, inplace, g2, out=inplace)
        assert torch.equal(inplace, want) and not torch.equal(p, want)


# ---- prepared files ------------------------------------------------------------------------------------------------------
def _unprepared(secs: dict) -> dict:
    return {sid: secs[sid] for sid in range(1, 8)}


def _arbitrary_section7() -> bytes:
    rng = np.random.default_rng(17)
    return struct.pack("<I", 2) + rng.bytes(1000)


@pytest.fixture(scope="module")
def oracle_files(tmp_path_factory):
    """(a directory, power -> the oracle's sections of a prepared ceremony) for powers 1 and 3."""
    import ptau_writer as pw
    return tmp_path_factory.mktemp("prep"), {p: pw.sections_oracle(*TOXIC, p) for p in (1, 3)}


@pytest.mark.gpu
@pytest.mark.parametrize("power", [1, 3])
def test_prepare_equals_the_oracle_writer(net, oracle_files, power):
    import ptau_writer as pw
    from distributed_groth16_b200.groth16 import circom
    tmp, secs = oracle_files
    src = pw.write_ptau(str(tmp / ("u%d.ptau" % power)), _unprepared(secs[power]))
    dst = str(tmp / ("p%d.ptau" % power))
    circom.ptau_prepare_phase2(net, src, dst)
    assert open(dst, "rb").read() == pw.ptau_bytes(secs[power])
    assert circom.ptau_check_lagrange(net, dst).ok


@pytest.mark.gpu
def test_prepare_already_prepared_input_and_ceremony_power(net, oracle_files):
    """An input that is already prepared (with wrong Lagrange sections) and states ceremonyPower != power: sections 12-15
    are recomputed and section 1 is restated with ceremonyPower = power."""
    import artefact_writer as aw
    import ptau_writer as pw
    from distributed_groth16_b200.groth16 import circom
    tmp, secs = oracle_files
    s = dict(secs[3])
    s[1] = struct.pack("<I", 32) + aw.Q.to_bytes(32, "little") + struct.pack("<II", 3, 9)
    s[12] = s[12][64:] + s[12][:64]
    s[14] = bytes(len(s[14]))
    src = pw.write_ptau(str(tmp / "prepared_in.ptau"), s)
    dst = str(tmp / "prepared_out.ptau")
    circom.ptau_prepare_phase2(net, src, dst)
    assert open(dst, "rb").read() == pw.ptau_bytes(secs[3])
    with pytest.raises(ValueError, match="input file"):
        circom.ptau_prepare_phase2(net, src, src)


@pytest.mark.gpu
def test_prepare_at_power_17_equals_the_gpu_writer_and_feeds_zkey_new(net, tmp_path):
    import ptau_writer as pw
    from distributed_groth16_b200.groth16 import circom
    secs = pw.sections_gpu(net, *TOXIC, 17)
    secs[7] = _arbitrary_section7()
    src = pw.write_ptau(str(tmp_path / "u17.ptau"), _unprepared(secs))
    dst = str(tmp_path / "p17.ptau")
    timings = {}
    from distributed_groth16_b200.groth16 import ptau
    ptau.prepare_phase2(net, src, dst, timings=timings)
    ref = pw.write_ptau(str(tmp_path / "ref17.ptau"), secs)
    assert open(dst, "rb").read() == open(ref, "rb").read()
    assert set(timings) == {"intt_s", "transfer_s", "write_s"}
    rep = circom.ptau_check_lagrange(net, dst)
    assert rep.ok, rep.failures
    r1cs = open(os.path.join(G, "circom2_multiplier2.r1cs"), "rb").read()
    assert circom.zkey_new(net, r1cs, dst) == circom.zkey_new(net, r1cs, ref)


def _patch(path, sid, first_point, data, width):
    from distributed_groth16_b200 import formats
    with formats.PTau(path, prepared=False) as pt:
        off = pt.section_span(sid)[0] + first_point * width * 8
    with open(path, "r+b") as f:
        f.seek(off)
        f.write(data)


def _point(path, sid, idx, width):
    from distributed_groth16_b200 import formats
    with formats.PTau(path, prepared=False) as pt:
        return pt.points(sid, idx, 1, width).tobytes()


@pytest.fixture
def good3(net, oracle_files, tmp_path):
    import ptau_writer as pw
    _, secs = oracle_files
    return lambda name: pw.write_ptau(str(tmp_path / name), secs[3])


@pytest.mark.gpu
@pytest.mark.parametrize("sid", [12, 13, 14, 15])
def test_check_lagrange_rejects_a_replaced_point(net, good3, sid):
    """One Lagrange point replaced by another valid point (its neighbour), at level 1 and at the top level."""
    from distributed_groth16_b200.groth16 import circom
    width = 16 if sid == 13 else 8
    top = 3 + (1 if sid == 12 else 0)
    for level in (1, top):
        path = good3("repl_%d_%d.ptau" % (sid, level))
        first = (1 << level) - 1
        _patch(path, sid, first, _point(path, sid, first + 1, width), width)
        rep = circom.ptau_check_lagrange(net, path)
        assert not rep.ok
        assert rep.failures == [f for f in rep.failures if f.startswith("section %d level %d:" % (sid, level))]
        assert len(rep.failures) == 1, rep.failures


@pytest.mark.gpu
def test_check_lagrange_rejects_swapped_points_and_a_changed_tau_point(net, good3):
    from distributed_groth16_b200.groth16 import circom
    path = good3("swap.ptau")
    a, b = _point(path, 15, 3, 8), _point(path, 15, 5, 8)       # level 2 of section 15: points 3..6
    _patch(path, 15, 3, b, 8)
    _patch(path, 15, 5, a, 8)
    rep = circom.ptau_check_lagrange(net, path)
    assert not rep.ok and rep.failures == [f for f in rep.failures if f.startswith("section 15 level 2:")], rep.failures
    path = good3("tau.ptau")
    _patch(path, 3, 2, _point(path, 3, 3, 16), 16)              # tau^2 G2 := tau^3 G2
    rep = circom.ptau_check_lagrange(net, path)
    assert not rep.ok
    assert sorted(rep.failures) == sorted("section 13 level %d: the Lagrange points are not the inverse NTT of the first %d "
                                          "points of section 3" % (k, 1 << k) for k in (2, 3)), rep.failures
