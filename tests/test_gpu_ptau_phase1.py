"""Phase 1 of the ceremony on the GPU (snarkjs `powersoftau new / contribute / beacon / verify`): the geometric-sequence
kernel (b200zk_points_mul_powers_dev) exact at every size up to a power-22 ceremony's sections, the ffjavascript encodings
(b200zk_points_encode_dev), new -> contribute -> beacon byte for byte against the pure-Python phase1_oracle, a chain from
nothing to a verified proof, and verify on good and tampered files."""
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
R = 21888242871839275222246405745257275088548364400416034343698204186575808495617
Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
RINV = pow(1 << 256, -1, R)
SEEDS = ([0xA1, 2, 3, 4, 5, 6, 7, 8], [0xB2, 9, 10, 11, 12, 13, 14, 15])
BEACON = bytes.fromhex("0102030405060708090a0b0c0d0e0f101112131415161718191a1b1c1d1e1f")
RAND = int.from_bytes(np.random.default_rng(17).bytes(32), "little") % R


def _mont_u64(net, logs):
    arr = np.zeros((len(logs), 4), dtype=np.uint64)
    arr[:, 0] = logs
    return net.fr_convert(net.to_device(arr), to_mont=True)


def _expected(net, logs, first, ratio, g2):
    """fixed_base_mul(logs_i first ratio^i): fr_powers, a field product and the fixed-base multiplication (pinned)."""
    import torch
    from distributed_groth16_b200.groth16.setup import _fixed_base, _powers
    n = len(logs)
    pw = _powers(net, ratio % R, first % R, n)
    lm = _mont_u64(net, logs)
    prod = torch.empty_like(pw)
    zero = torch.zeros_like(pw)
    net.check(net._lib.b200zk_fr_mul_sub_dev(net._h, 0, c_vp(pw.data_ptr()), c_vp(lm.data_ptr()), c_vp(zero.data_ptr()),
                                             c_vp(prod.data_ptr()), n))
    return _fixed_base(net, prod, g2)


def _inputs(net, g2, n, seed):
    import torch
    import dlog_oracle
    pts = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
    logs = dlog_oracle.base_logs(seed, n)
    if n > 1:
        inf = np.unique(np.random.default_rng(n + g2).integers(0, n, size=min(n // 2, 5)))
        logs[inf] = 0
        pts[torch.from_numpy(inf).to(pts.device)] = 0
    return pts, logs


def _mul(net, pts, first, ratio, g2, out=None):
    from distributed_groth16_b200.groth16 import phase1
    r = phase1.points_mul_powers(net, pts, first, ratio, g2, out=out)
    net.sync(0)
    return r


FIRSTS = (0, 1, R - 1, RAND)
RATIOS = (0, 1, R - 1, RAND ^ 0x5A5A, R + 7, (1 << 256) - 1)
SIZES = [(False, n) for n in (0, 1, 2, 63, 64, 65, 1 << 10, 1 << 16, 1 << 20, 1 << 23)] + \
        [(True, n) for n in (0, 1, 31, 32, 33, 1 << 12, 1 << 18, 1 << 22)]


@pytest.mark.gpu
@pytest.mark.parametrize("g2,n", SIZES)
def test_points_mul_powers_exact(net, g2, n):
    """Generated points with known logs, some at infinity: out_i == (logs_i first ratio^i) G.  Every (first, ratio) pair
    up to 2^10 points, one random pair (and ratio = 0) above."""
    import torch
    pts, logs = _inputs(net, g2, n, 0x9A1 + 7 * n + g2)
    pairs = [(f, r) for f in FIRSTS for r in RATIOS] if n <= 1 << 10 else [(RAND, RAND ^ 0x5A5A), (RAND, 0)]
    for first, ratio in pairs:
        got = _mul(net, pts, first, ratio, g2)
        assert torch.equal(got, _expected(net, logs, first, ratio, g2)), (n, hex(first), hex(ratio))


@pytest.mark.gpu
@pytest.mark.parametrize("g2", [False, True])
def test_points_mul_powers_in_place_and_chunked(net, g2):
    """out == points works, and calls on [a, b) with first ratio^a equal the slices of one call."""
    import torch
    n = 3000
    pts, logs = _inputs(net, g2, n, 0x77 + g2)
    whole = _mul(net, pts, RAND, RAND ^ 0x5A5A, g2)
    ratio = RAND ^ 0x5A5A
    parts = []
    for a, b in ((0, 1), (1, 64), (64, 999), (999, 1000), (1000, 3000)):
        parts.append(_mul(net, pts[a:b].contiguous(), RAND * pow(ratio, a, R) % R, ratio, g2))
    assert torch.equal(torch.cat(parts), whole)
    inplace = pts.clone()
    _mul(net, inplace, RAND, ratio, g2, out=inplace)
    assert torch.equal(inplace, whole)


@pytest.mark.gpu
def test_points_mul_powers_error_codes(net):
    one = np.ones(4, dtype=np.uint64)
    lib = net._lib
    d = net.generate_g1(5, 4)
    call = lambda pts, n, f, r, out: lib.b200zk_points_mul_powers_dev(net._h, 0, 0, pts, n, f, r, out)
    assert call(None, 4, c_vp(one.ctypes.data), c_vp(one.ctypes.data), c_vp(d.data_ptr())) == _native.ERR_ARG
    assert call(c_vp(d.data_ptr()), 4, c_vp(one.ctypes.data), c_vp(one.ctypes.data), None) == _native.ERR_ARG
    assert call(c_vp(d.data_ptr()), 4, None, c_vp(one.ctypes.data), c_vp(d.data_ptr())) == _native.ERR_ARG
    assert lib.b200zk_points_mul_powers_dev(net._h, 3, 0, c_vp(d.data_ptr()), 4, c_vp(one.ctypes.data),
                                            c_vp(one.ctypes.data), c_vp(d.data_ptr())) == _native.ERR_ARG
    assert call(None, 0, c_vp(one.ctypes.data), c_vp(one.ctypes.data), None) == _native.OK          # n = 0: nothing
    # a workspace that cannot exist (4 TB of digits) is refused before any launch
    before = net.launch_count()
    assert call(c_vp(d.data_ptr()), 1 << 36, c_vp(one.ctypes.data), c_vp(one.ctypes.data), c_vp(d.data_ptr())) == _native.ERR_OOM
    assert net.launch_count() == before
    assert b"do not fit" in lib.b200zk_last_error(net._h)
    net.sync(0)                                                     # the context is still usable
    assert _mul(net, d, 1, 1, False).shape == (4, 8)


# ---- encodings -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("g2", [False, True])
def test_points_encode_matches_the_host_restatements(net, g2):
    import torch
    from distributed_groth16_b200.groth16 import phase1, phase2
    n = 300
    pts = (net.generate_g2(61, n) if g2 else net.generate_g1(61, n)).cpu().numpy().view(np.uint64).copy()
    w = 16 if g2 else 8
    for i in range(0, n, 2):                                         # -P: y -> q - y limb-wise in Montgomery form
        for k in range(w // 2, w, 4):
            v = sum(int(pts[i, k + j]) << (64 * j) for j in range(4))
            v = (Q - v) % Q
            pts[i, k:k + 4] = [(v >> (64 * j)) & 0xFFFFFFFFFFFFFFFF for j in range(4)]
    pts[[0, 7, n - 1]] = 0
    d = net.to_device(pts)
    u = phase1.points_encode(net, d, g2, compressed=False).cpu().numpy()
    c = phase1.points_encode(net, d, g2, compressed=True).cpu().numpy()
    uh, ch = (phase2.u_g2, phase1.c_g2) if g2 else (phase2.u_g1, phase1.c_g1)
    flags = set()
    for i in range(n):
        assert u[i].tobytes() == uh(pts[i]), i
        assert c[i].tobytes() == ch(pts[i]), i
        flags.add(c[i][0] & 0xC0)
    assert flags == {0x00, 0x80, 0x40}                               # both signs of y and infinity were covered
    assert phase1.points_encode(net, d[:0], g2).shape[0] == 0


# ---- against the pure-Python oracle ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("power", [1, 2])
def test_new_contribute_beacon_equal_the_oracle(net, tmp_path, power):
    import phase1_oracle as po
    from distributed_groth16_b200.groth16 import phase1, phase2
    p0, p1, p2 = (str(tmp_path / ("s%d.ptau" % k)) for k in range(3))
    phase1.new(p0, power)
    b0 = po.new(power)
    assert open(p0, "rb").read() == b0
    rh, nc = phase1.contribute(net, p0, p1, phase2.ChaCha(SEEDS[0]), name="first", chunk=1)
    b1, orh, onc = po.contribute(b0, phase2.ChaCha(SEEDS[0]), name="first")
    assert (rh, nc) == (orh, onc)
    assert open(p1, "rb").read() == b1
    rh, nc = phase1.beacon(net, p1, p2, BEACON, 10, name="final", chunk=1)
    b2, orh, onc = po.beacon(b1, BEACON, 10, name="final")
    assert (rh, nc) == (orh, onc)
    assert open(p2, "rb").read() == b2


# ---- a chain from nothing -------------------------------------------------------------------------------------------------
def _secrets(rng):
    from distributed_groth16_b200.groth16 import phase2
    return [phase2.field_from_rng(rng, R) * RINV % R for _ in range(3)]


def _tau_sections(path):
    from distributed_groth16_b200 import formats
    with formats.PTau(path, prepared=False) as pt:
        return {sid: b"".join(pt.section_chunks(sid)) for sid in (2, 3, 4, 5, 6)}


@pytest.fixture(scope="module")
def chain(net, tmp_path_factory):
    from distributed_groth16_b200.groth16 import circom, phase1, phase2
    d = tmp_path_factory.mktemp("phase1")
    paths = [str(d / ("c%d.ptau" % k)) for k in range(4)]
    circom.ptau_new(paths[0], 15)
    phase1.contribute(net, paths[0], paths[1], phase2.ChaCha(SEEDS[0]), name="first")
    phase1.contribute(net, paths[1], paths[2], phase2.ChaCha(SEEDS[1]), name="second")
    circom.ptau_beacon(net, paths[2], paths[3], BEACON, 10, name="final beacon")
    ks = [_secrets(phase2.ChaCha(SEEDS[0])), _secrets(phase2.ChaCha(SEEDS[1])), _secrets(phase2.rng_from_beacon(BEACON, 10))]
    tab = [ks[0][i] * ks[1][i] * ks[2][i] % R for i in range(3)]
    return dict(paths=paths, toxic=tab, dir=d)


@pytest.mark.gpu
def test_chain_equals_the_toxic_waste_sections(net, chain):
    import ptau_writer as pw
    want = pw.sections_gpu(net, *chain["toxic"], 15)
    got = _tau_sections(chain["paths"][3])
    for sid in (2, 3, 4, 5, 6):
        assert got[sid] == want[sid], sid


@pytest.mark.gpu
def test_chain_prepares_sets_up_and_proves(net, chain):
    import artefact_writer as aw
    from oracle import layout
    from distributed_groth16_b200 import ark_serialize as ark, formats
    from distributed_groth16_b200.groth16 import circom, verify
    x = np.load(os.path.join(HERE, "golden", "reference_artefacts.npz"))
    s = dict(np.load(os.path.join(HERE, "golden", "sha256_circuit.npz")))
    r1cs_secs = {1: x["sha256_r1cs_sec1"].tobytes(), 2: aw.r1cs_constraints(s, int(s["dims"][2])),
                 3: x["sha256_r1cs_sec3"].tobytes()}
    r1cs = aw.container(b"r1cs", [(int(sid), r1cs_secs[int(sid)]) for sid in x["sha256_r1cs_order"]])
    prepared = str(chain["dir"] / "prepared.ptau")
    circom.ptau_prepare_phase2(net, chain["paths"][3], prepared)
    assert circom.ptau_verify(net, prepared).ok
    z0 = circom.zkey_new(net, r1cs, prepared)
    z1, _ = circom.zkey_contribute(net, z0, name="phase 2", entropy=b"chain")
    z2, _ = circom.zkey_beacon(net, z1, BEACON, 10, name="phase 2 beacon")
    rep = circom.zkey_verify(net, r1cs, prepared, z2)
    assert rep.ok, rep.failures
    wit = [int.from_bytes(r.tobytes(), "little") for r in s["witness"]]
    proof, pub = circom.prove_zkey_wtns(net, z2, aw.write_wtns(wit))
    zk = formats.read_zkey(z2)
    vk = ark.ArkVerifyingKey(zk.alpha_g1, zk.beta_g2, zk.gamma_g2, zk.delta_g2, zk.ic)
    assert verify.verify_proof(net, vk, layout.fr_to_arr([wit[1]]), proof)
    assert not verify.verify_proof(net, vk, layout.fr_to_arr([wit[1] + 1]), proof)


@pytest.mark.gpu
def test_contribute_at_power_20(net, tmp_path):
    import ptau_writer as pw
    from distributed_groth16_b200.groth16 import phase1, phase2
    p0, p1 = str(tmp_path / "n20.ptau"), str(tmp_path / "c20.ptau")
    phase1.new(p0, 20)
    phase1.contribute(net, p0, p1, phase2.ChaCha(SEEDS[1]), chunk=3 << 18)
    tau, alpha, beta = _secrets(phase2.ChaCha(SEEDS[1]))
    want = pw.sections_gpu(net, tau, alpha, beta, 20)
    got = _tau_sections(p1)
    for sid in (2, 3, 4, 5, 6):
        assert got[sid] == want[sid], sid
    assert phase1.verify(net, p1).ok


# ---- verify ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_verify_accepts_every_stage_and_rejects_new(net, chain):
    from distributed_groth16_b200.groth16 import circom
    rep = circom.ptau_verify(net, chain["paths"][0])
    assert not rep.ok and "no contributions" in rep.failures[0]
    for k in (1, 2, 3):
        rep = circom.ptau_verify(net, chain["paths"][k])
        assert rep.ok, (k, rep.failures)
        assert [c[0] for c in rep.contributions] == ["first", "second", "final beacon"][:k]
        assert [c[1] for c in rep.contributions] == [0, 0, 1][:k]


def _file_sections(buf):
    off, out = 12, []
    while off < len(buf):
        sid, ln = struct.unpack_from("<IQ", buf, off)
        out.append((sid, off + 12, ln))
        off += 12 + ln
    return out


def _with_section(buf, sid, body):
    parts = [buf[:8], struct.pack("<I", struct.unpack_from("<I", buf, 8)[0])]
    for s, off, ln in _file_sections(buf):
        parts.append(struct.pack("<IQ", s, len(body) if s == sid else ln) + (body if s == sid else buf[off:off + ln]))
    return b"".join(parts)


def _with_point(buf, sid, idx, pt):
    off = dict((s, o) for s, o, _ in _file_sections(buf))[sid]
    raw = np.ascontiguousarray(pt, dtype="<u8").tobytes()
    b = bytearray(buf)
    b[off + idx * len(raw):off + (idx + 1) * len(raw)] = raw
    return bytes(b)


def _tampered(net, buf):
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase1, phase2
    g1x2 = phase2._scale_one(net, phase1.G1_GEN, 2)
    g2x2 = phase2._scale_one(net, phase1.G2_GEN, 2, g2=True)
    secs = {s: buf[o:o + ln] for s, o, ln in _file_sections(buf)}
    recs = lambda: formats.parse_ptau_contributions(secs[7])
    rec7 = lambda rs: _with_section(buf, 7, formats.ptau_contributions_bytes(rs))
    out = []
    out.append(("a tau point mid-section", _with_point(buf, 2, 1000, g1x2), "section 2"))
    s2 = bytearray(secs[2])
    s2[64 * 5:64 * 6], s2[64 * 6:64 * 7] = secs[2][64 * 6:64 * 7], secs[2][64 * 5:64 * 6]
    out.append(("two swapped points", _with_section(buf, 2, bytes(s2)), "section 2"))
    out.append(("tauG1[0] is not G1", _with_point(buf, 2, 0, g1x2), "section 2"))
    out.append(("a section-3 point", _with_point(buf, 3, 77, g2x2), "section 3"))
    s4 = phase2._scale_section(net, secs[4], 2)
    out.append(("section 4 scaled", _with_section(buf, 4, s4), "section 4"))
    out.append(("betaG2 replaced", _with_point(buf, 6, 0, g2x2), "section 6"))
    rs = recs(); rs[-1].key["tau"]["g1_sx"] = g1x2
    out.append(("a public-key point", rec7(rs), "contribution 3"))
    rs = recs(); rs[1].tau_g1 = g1x2
    out.append(("tauG1 of record 2 does not follow record 1", rec7(rs), "contribution 2"))
    rs = recs(); rs[-1].next_challenge = bytes(64)
    out.append(("nextChallenge", rec7(rs), "contribution 3"))
    rs = recs(); rs[-1].partial_hash = rs[-1].partial_hash[:5] + bytes([rs[-1].partial_hash[5] ^ 1]) + rs[-1].partial_hash[6:]
    out.append(("partialHash", rec7(rs), "contribution 3"))
    rs = recs(); rs[-1].beacon_hash = bytes([rs[-1].beacon_hash[0] ^ 1]) + rs[-1].beacon_hash[1:]
    out.append(("beacon parameters", rec7(rs), "contribution 3"))
    off5 = dict((s, o) for s, o, _ in _file_sections(buf))[5]
    out.append(("a truncated section", buf[:off5 + 1000], "section 5"))
    return out


@pytest.mark.gpu
def test_verify_rejects_tampered_files(net, chain, tmp_path):
    from distributed_groth16_b200.groth16 import circom
    buf = open(chain["paths"][3], "rb").read()
    for what, data, where in _tampered(net, buf):
        p = str(tmp_path / "t.ptau")
        open(p, "wb").write(data)
        rep = circom.ptau_verify(net, p)
        assert not rep.ok, what
        assert any(where in f for f in rep.failures), (what, rep.failures)


# ---- refusals ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals_and_prepared_input(net, chain, tmp_path):
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase1, phase2
    src = chain["paths"][1]
    with pytest.raises(ValueError):
        phase1.contribute(net, src, src, phase2.ChaCha(SEEDS[0]))
    buf = open(src, "rb").read()
    off1 = _file_sections(buf)[0][1]
    reduced = bytearray(buf)
    reduced[off1 + 40:off1 + 44] = struct.pack("<I", 16)               # ceremonyPower 16 > power 15
    rp = str(tmp_path / "reduced.ptau")
    open(rp, "wb").write(bytes(reduced))
    with pytest.raises(ValueError, match="reduced"):
        phase1.contribute(net, rp, str(tmp_path / "x.ptau"), phase2.ChaCha(SEEDS[0]))
    assert not os.path.exists(str(tmp_path / "x.ptau"))
    prep, out = str(tmp_path / "prep.ptau"), str(tmp_path / "after.ptau")
    from distributed_groth16_b200.groth16 import circom
    circom.ptau_prepare_phase2(net, src, prep)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        phase1.contribute(net, prep, out, phase2.ChaCha(SEEDS[1]))
    assert any("prepared" in str(w.message) for w in caught)
    assert [s for s, _, _ in _file_sections(open(out, "rb").read())] == [1, 2, 3, 4, 5, 6, 7]
    assert phase1.verify(net, out).ok
    with formats.PTau(out, prepared=False) as pt:
        assert len(phase1._read_records(pt)) == 2
