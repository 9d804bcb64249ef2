"""Phase 2 of the ceremony on the GPU (snarkjs `zkey contribute`, `zkey beacon`, `zkey verify`): the one-scalar-many-points
kernel (b200zk_points_scale_dev) and the same-ratio check against the oracle, a contribute / contribute / beacon chain on
sha256 against the toxic-waste setup with the accumulated delta, zkey_verify on every stage and on tampered keys, and the
tiny circuit byte for byte against the pure-Python phase2_oracle."""
import os
import sys

import numpy as np
import pytest

from distributed_groth16_b200._native import c_vp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")
TOXIC = dict(tau=0x1234567890ABCDEF1234567890ABCDEF, alpha=11111111111111111111, beta=22222222222222222223)
X1, X2 = 0x5EC12E7_0000_1111_2222_3333_4444_5555_6666_7777, 987654321987654321987654321
S1, S2 = 0xABCDEF0123456789, 0x1111222233334444555566667777
BEACON = bytes.fromhex("0102030405060708090a0b0c0d0e0f101112131415161718191a1b1c1d1e1f")


def _scale(net, pts, k, g2, in_place=False):
    import torch
    t = net.to_device(np.ascontiguousarray(pts, dtype=np.uint64))
    out = t if in_place else torch.full_like(t, -1)
    kl = np.array([(k >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)
    net.check(net._lib.b200zk_points_scale_dev(net._h, 0, int(g2), c_vp(t.data_ptr()), int(t.shape[0]), c_vp(kl.ctypes.data),
                                               c_vp(out.data_ptr())))
    return out.cpu().numpy().view(np.uint64)


@pytest.mark.gpu
def test_points_scale_g1_matches_the_oracle(net, cref):
    """Infinity points, k = 0, 1, r - 1, r, k > r (up to 2^256 - 1), random k, in place, n = 0 and n not a multiple of the
    block (64)."""
    from oracle import bn254 as o, layout
    n = 150
    pts = cref.g1_generate(41, n)
    pts[[0, 63, 64, 149]] = 0
    P = layout.arr_to_g1(pts)
    rng = np.random.default_rng(3)
    rand = int.from_bytes(rng.bytes(32), "little")
    for k in (0, 1, o.R - 1, o.R, o.R + 12345, (1 << 256) - 1, rand % o.R, rand):
        sel = range(n) if k in (rand, o.R - 1) else range(0, n, 7)
        got = _scale(net, pts, k, False, in_place=(k == rand))
        want = layout.g1_to_arr([o.G1.mul(P[i], k) for i in sel])
        assert (got[list(sel)] == want).all(), hex(k)
    assert _scale(net, pts[:0], 5, False).shape == (0, 8)


@pytest.mark.gpu
def test_points_scale_g2_matches_the_oracle_and_clears_the_cofactor(net, cref):
    import phase2_oracle
    from oracle import bn254 as o, layout
    from distributed_groth16_b200.groth16.phase2 import G2_COFACTOR
    pts = cref.g2_generate(43, 5)
    pts[2] = 0
    P = layout.arr_to_g2(pts)
    times = lambda p, k: phase2_oracle.g2_times(p, k)
    rand = int.from_bytes(np.random.default_rng(4).bytes(32), "little")
    for k in (0, 1, o.R - 1, o.R, o.R + 3, rand):
        got = _scale(net, pts, k, True, in_place=(k == 1))
        assert (got == layout.g2_to_arr([times(p, k) for p in P])).all(), hex(k)
    # a twist point outside the order-r subgroup: the cofactor brings it in
    x = 5
    while True:
        x += 1
        try:
            q = o.g2_decompress(x.to_bytes(32, "little") + (7).to_bytes(32, "little"))
        except ValueError:
            continue
        if o.G2.from_jac(o.G2.jac_mul(o.G2.to_jac(q), o.R)) is not None:
            break
    got = _scale(net, layout.g2_to_arr([q]), G2_COFACTOR, True)
    assert (got == layout.g2_to_arr([times(q, G2_COFACTOR)])).all()
    enc = net.points_compress(net.to_device(got), g2=True)
    back = net.points_decompress(enc, g2=True, check_subgroup=True).cpu().numpy().view(np.uint64)
    assert (back == got).all()


@pytest.mark.gpu
def test_same_ratio_agrees_with_the_oracle_pairing(net):
    from oracle import bn254 as o, layout
    from distributed_groth16_b200.groth16.phase2 import _same_ratio
    a, b, c = 12345678901234567, 98765432109876543, 555555555555555555
    g1 = lambda k: layout.g1_to_arr([o.G1.mul(o.G1_GEN, k)])[0]
    g2 = lambda k: layout.g2_to_arr([o.G2.mul(o.G2_GEN, k)])[0]
    cases = [(a, a * b, c, b * c), (a, a * b + 1, c, b * c), (1, b, 1, b), (a, a * b, c, c)]
    for p1, p2, q1, q2 in cases:
        want = o.pairing(o.G1.mul(o.G1_GEN, p1), o.G2.mul(o.G2_GEN, q2)) == o.pairing(o.G1.mul(o.G1_GEN, p2),
                                                                                   o.G2.mul(o.G2_GEN, q1))
        assert _same_ratio(net, g1(p1), g1(p2), g2(q1), g2(q2)) == want, (p1, p2, q1, q2)
    assert _same_ratio(net, g1(a), g1(a * b), g2(c), g2(b * c))
    assert not _same_ratio(net, g1(a), g1(a * b), g2(c), g2(b * c + 1))


# ---- sha256: contribute, contribute, beacon ----------------------------------------------------------------------------
def _sha256():
    import artefact_writer as aw
    x = np.load(os.path.join(G, "reference_artefacts.npz"))
    s = dict(np.load(os.path.join(G, "sha256_circuit.npz")))         # in memory: the writer slices it per constraint
    secs = {1: x["sha256_r1cs_sec1"].tobytes(), 2: aw.r1cs_constraints(s, int(s["dims"][2])), 3: x["sha256_r1cs_sec3"].tobytes()}
    return s, aw.container(b"r1cs", [(int(sid), secs[int(sid)]) for sid in x["sha256_r1cs_order"]])


def _toxic_key(net, s, delta):
    """circuit_specific_setup(tau, alpha, beta, 1, delta) with its query tensors captured at the upload."""
    from distributed_groth16_b200.groth16 import setup
    from distributed_groth16_b200.groth16.proving_key import ProvingKey
    captured = {}
    orig = ProvingKey.from_device.__func__

    def capture(cls, net_, a, b1, b2, l, h, n_inputs, vk_points):
        captured.update(l_query=l.cpu().numpy().view(np.uint64).copy(), h_query=h.cpu().numpy().view(np.uint64).copy(),
                        vk_points=np.array(vk_points))
        return orig(cls, net_, a, b1, b2, l, h, n_inputs, vk_points)

    n_wires, n_pub, n_cons = (int(v) for v in s["dims"])
    coo = lambda k: (s[k + "_rows"], s[k + "_cols"], s[k + "_vals"])
    mp = pytest.MonkeyPatch()
    mp.setattr(ProvingKey, "from_device", classmethod(capture))
    try:
        pk, vk, mats = setup.circuit_specific_setup(net, n_wires, n_pub + 1, n_cons, coo("a"), coo("b"), coo("c"),
                                                    (TOXIC["tau"], TOXIC["alpha"], TOXIC["beta"], 1, delta))
    finally:
        mp.undo()
    return pk, vk, mats, captured


@pytest.fixture(scope="module")
def chain(net, tmp_path_factory):
    import ptau_writer as pw
    from oracle import bn254 as o, layout
    from distributed_groth16_b200.groth16 import circom, phase2
    s, r1cs = _sha256()
    path = pw.write_ptau(str(tmp_path_factory.mktemp("ptau") / "p15.ptau"),
                         pw.sections_gpu(net, TOXIC["tau"], TOXIC["alpha"], TOXIC["beta"], 15))
    z0 = circom.zkey_new(net, r1cs, path)
    g1 = lambda k: layout.g1_to_arr([o.G1.mul(o.G1_GEN, k)])[0]
    z1, h1 = phase2.contribute(net, z0, X1, g1(S1), name="first")
    z2, h2 = phase2.contribute(net, z1, X2, g1(S2), name="second")
    z3, h3 = circom.zkey_beacon(net, z2, BEACON, 10, name="final beacon")
    xb, _ = phase2.beacon_secrets(net, BEACON, 10)
    deltas = [1, X1 % o.R, X1 * X2 % o.R, X1 * X2 * xb % o.R]
    return dict(s=s, r1cs=r1cs, ptau=path, zkeys=[z0, z1, z2, z3], hashes=[h1, h2, h3], deltas=deltas)


def _sections(z):
    from distributed_groth16_b200.groth16 import phase2
    return {sid: z[off:off + ln] for sid, off, ln in phase2._section_table(z)}


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [1, 2, 3])
def test_sha256_chain_equals_the_toxic_waste_key_and_proves(net, chain, stage):
    import artefact_writer as aw
    from oracle import layout
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import circom, verify
    from distributed_groth16_b200.groth16.phase2 import _HDR_DELTA
    z, z0, s = chain["zkeys"][stage], chain["zkeys"][0], chain["s"]
    pk, vk, mats, t = _toxic_key(net, s, chain["deltas"][stage])
    try:
        zk = formats.read_zkey(z)
        assert (zk.l_query == t["l_query"]).all() and (zk.h_query == t["h_query"]).all()
        assert (zk.vk_points() == t["vk_points"]).all()                      # alpha_1 beta_1 delta_1 beta_2 delta_2
        a, b = _sections(z), _sections(z0)
        assert list(a) == list(b)
        for sid in (1, 3, 4, 5, 6, 7):
            assert a[sid] == b[sid], sid
        assert a[2][:_HDR_DELTA] == b[2][:_HDR_DELTA] and a[2][_HDR_DELTA + 192:] == b[2][_HDR_DELTA + 192:]
        mpc = formats.read_mpc_params(z)
        assert len(mpc.contributions) == stage and mpc.cs_hash == bytes(64)
        assert [c.name for c in mpc.contributions] == ["first", "second", "final beacon"][:stage]
        wit = [int.from_bytes(r.tobytes(), "little") for r in s["witness"]]
        proof, _ = circom.prove_zkey_wtns(net, z, aw.write_wtns(wit))
        zt = net.fr_convert(net.to_device(s["witness"]), to_mont=True)
        assert proof == circom.prove_from_matrices(pk, mats, zt)
        assert verify.verify_proof(net, vk, layout.fr_to_arr([wit[1]]), proof)
        assert not verify.verify_proof(net, vk, layout.fr_to_arr([wit[1] + 1]), proof)
    finally:
        pk.free()


@pytest.mark.gpu
def test_zkey_verify_accepts_every_stage(net, chain):
    from distributed_groth16_b200.groth16 import circom
    for i, z in enumerate(chain["zkeys"]):
        rep = circom.zkey_verify(net, chain["r1cs"], chain["ptau"], z)
        assert rep.ok, (i, rep.failures)
        assert [c[0] for c in rep.contributions] == ["first", "second", "final beacon"][:i]
        assert [c[1] for c in rep.contributions] == [0, 0, 1][:i]
        assert [c[2] for c in rep.contributions] == chain["hashes"][:i]
        assert rep.cs_hash == bytes(64)


def _tampered(net, chain):
    """(what, zkey bytes) pairs zkey_verify must reject."""
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase2
    from distributed_groth16_b200.groth16.phase2 import _HDR_DELTA, _replace_sections
    z1, z2, z3 = chain["zkeys"][1:]
    sec = _sections(z3)
    pts = lambda sid: np.frombuffer(sec[sid], dtype="<u8").reshape(-1, 8 if sid != 7 else 16).copy()

    def with_point(sid, i, j):                       # point i of section sid replaced by point j
        p = pts(sid)
        p[i] = p[j]
        return _replace_sections(z3, {sid: p.tobytes()})

    def mpc_edit(z, fn):
        m = formats.read_mpc_params(z)
        fn(m)
        return _replace_sections(z, {10: formats.mpc_params_bytes(m)})

    def scaled(z, k):                                # L and H times k, delta untouched
        s = _sections(z)
        out = {}
        for sid in (8, 9):
            t = net.to_device(np.frombuffer(s[sid], dtype="<u8").reshape(-1, 8))
            out[sid] = phase2.points_scale(net, t, k).cpu().numpy().tobytes()
        return _replace_sections(z, out)

    hdr = sec[2]
    d2 = np.frombuffer(hdr, dtype="<u8", count=16, offset=_HDR_DELTA + 64)
    d2x = phase2._scale_one(net, d2, 2, g2=True)
    bad_d2 = _replace_sections(z3, {2: hdr[:_HDR_DELTA + 64] + d2x.astype("<u8").tobytes() + hdr[_HDR_DELTA + 192:]})

    def sx(m):
        m.contributions[0].g1_sx = phase2._scale_one(net, m.contributions[0].g1_sx, 3)

    def tr(m):
        t = bytearray(m.contributions[1].transcript)
        t[5] ^= 1
        m.contributions[1].transcript = bytes(t)

    def exp(m):
        m.contributions[2].num_iterations_exp = 11

    return [("one L point", with_point(8, 3, 4)), ("one H point", with_point(9, 10, 11)),
            ("L and H scaled by another x", scaled(z1, 7)), ("delta_2 inconsistent with delta_1", bad_d2),
            ("g1_sx", mpc_edit(z3, sx)), ("transcript", mpc_edit(z3, tr)),
            ("dropped contribution", mpc_edit(z2, lambda m: m.contributions.pop(0))),
            ("beacon parameters", mpc_edit(z3, exp)), ("A section", with_point(5, 2, 3))]


@pytest.mark.gpu
def test_zkey_verify_rejects_tampered_keys(net, chain):
    from distributed_groth16_b200.groth16 import circom
    for what, z in _tampered(net, chain):
        rep = circom.zkey_verify(net, chain["r1cs"], chain["ptau"], z)
        assert not rep.ok and rep.failures, what


@pytest.mark.gpu
@pytest.mark.parametrize("power", [2, 3])
def test_tiny_circuit_contribute_and_beacon_equal_the_oracle(net, tmp_path, power):
    import phase2_oracle
    import ptau_writer as pw
    from oracle import bn254 as o, layout
    from distributed_groth16_b200.groth16 import circom, phase2
    r1cs = open(os.path.join(G, "circom2_multiplier2.r1cs"), "rb").read()
    path = pw.write_ptau(str(tmp_path / "tiny.ptau"), pw.sections_oracle(0x1234567890ABCDEF, 1111111111111111111,
                                                                            2222222222222222223, power))
    z0 = circom.zkey_new(net, r1cs, path)
    s_pt = o.G1.mul(o.G1_GEN, S1)
    z1, h1 = phase2.contribute(net, z0, X1, layout.g1_to_arr([s_pt])[0], name="tiny")
    w1, g1 = phase2_oracle.contribute(z0, X1, s_pt, name="tiny")
    assert z1 == w1 and h1 == g1
    z2, h2 = circom.zkey_beacon(net, z1, BEACON, 10)
    w2, g2 = phase2_oracle.beacon(w1, BEACON, 10)
    assert z2 == w2 and h2 == g2
    assert circom.zkey_verify(net, r1cs, path, z2).ok
