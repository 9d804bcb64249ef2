"""Phase 2 by challenge and response on the GPU (snarkjs `zkey export bellman`, `zkey bellman contribute`, `zkey import
bellman`): the forward point NTT (b200zk_points_ntt_dev) against fixed-base multiplication of the field NTT, the export of
the snarkjs-written complex-circuit key against the circuit hash snarkjs wrote, the exported H against the toxic waste on
synthetic ceremonies, a bellman round against the direct phase2.contribute, the tiny circuit byte for byte against the
pure-Python bellman_oracle, the refusals of import, and the widened H check of zkey_verify."""
import functools
import hashlib
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
TOXIC = dict(tau=0x2468ACE013579BDF2468ACE013579BDF, alpha=31415926535897932384, beta=27182818284590452353)
TINY = dict(tau=0x1234567890ABCDEF, alpha=1111111111111111111, beta=2222222222222222223)
X = [0x5EC12E7_0000_1111_2222_3333_4444_5555_6666_7777, 987654321987654321987654321, 0xC0FFEE_1234567, 0xBEEF_77777777]
S = [0xABCDEF0123456789, 0x1111222233334444555566667777, 0x3141592653589793, 0x2718281828459045]
BEACON = bytes.fromhex("0102030405060708090a0b0c0d0e0f101112131415161718191a1b1c1d1e1f")
R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def _g1(k):
    from oracle import bn254 as o, layout
    return layout.g1_to_arr([o.G1.mul(o.G1_GEN, k)])[0]


def _sections(z):
    from distributed_groth16_b200.groth16 import phase2
    return {sid: z[off:off + ln] for sid, off, ln in phase2._section_table(z)}


def _span(buf, part):
    from distributed_groth16_b200 import formats
    off, ln = formats.parse_bellman(buf).spans[part]
    return buf[off:off + ln]


# ---- the kernel ----------------------------------------------------------------------------------------------------------
def _mont(net, ints):
    arr = np.array([[(int(v) % R >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] for v in ints], dtype=np.uint64)
    return net.fr_convert(net.to_device(arr.reshape(-1, 4)), to_mont=True)


def _ntt(net, pts, g2, out=None):
    from distributed_groth16_b200.groth16 import ptau
    r = ptau.points_ntt(net, pts, g2, out=out)
    net.sync(0)
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("g2,log_n", [(False, k) for k in (0, 1, 2, 3, 5, 9, 14, 18, 22)] + [(True, k) for k in (0, 1, 3, 6, 10)])
def test_points_ntt_exact(net, g2, log_n):
    """P_j = k_j G with some k_j = 0 (infinity): points_ntt(P) == fixed_base_mul(ntt(k)) point for point, and the point iNTT
    takes it back to P."""
    import torch
    from distributed_groth16_b200.groth16 import ptau
    from distributed_groth16_b200.groth16.setup import _fixed_base
    n = 1 << log_n
    k = net.generate_fr(0xB311 + 7 * log_n + g2, n)
    if n > 1:
        k[torch.from_numpy(np.unique(np.random.default_rng(log_n).integers(0, n, size=min(n // 2, 5)))).to(k.device)] = 0
    pts = _fixed_base(net, k, g2)
    got = _ntt(net, pts, g2)
    assert torch.equal(got, _fixed_base(net, net.ntt_dev(k), g2))
    back = ptau.points_intt(net, got, g2)
    net.sync(0)
    assert torch.equal(back, pts)


@pytest.mark.gpu
@pytest.mark.parametrize("g2", [False, True])
@pytest.mark.parametrize("log_n", [1, 3, 8])
@pytest.mark.parametrize("kind", ["all_equal", "antipodal", "all_infinity"])
def test_points_ntt_adversarial(net, g2, log_n, kind):
    """All points equal (only output 0 is not infinity: n P_0), P_(j + n/2) = -P_j (the first pass cancels to the identity)
    and all points infinity, out of place and in place."""
    import torch
    from distributed_groth16_b200.groth16.setup import _fixed_base
    n = 1 << log_n
    rng = np.random.default_rng(n + 2 * g2 + 1)
    base = [int.from_bytes(rng.bytes(32), "little") % R for _ in range(n // 2)]
    logs = {"all_equal": [base[0]] * n, "antipodal": base + [R - v for v in base], "all_infinity": [0] * n}[kind]
    s = _mont(net, logs)
    pts = _fixed_base(net, s, g2)
    want = _fixed_base(net, net.ntt_dev(s), g2)
    assert torch.equal(_ntt(net, pts, g2), want)
    _ntt(net, pts, g2, out=pts)
    assert torch.equal(pts, want)
    if kind == "all_equal":
        assert not want[1:].any() and torch.equal(want[0], _fixed_base(net, _mont(net, [n * base[0]]), g2)[0])
    if kind == "all_infinity":
        assert not want.any()


@pytest.mark.gpu
def test_points_ntt_error_codes_and_aliasing(net):
    import torch
    lib, h = net._lib, net._h
    pts = net.generate_g1(77, 1 << 10)
    buf = torch.empty_like(pts)
    assert lib.b200zk_points_ntt_dev(h, 0, 0, c_vp(pts.data_ptr()), 29, c_vp(buf.data_ptr())) == _native.ERR_DOMAIN
    assert lib.b200zk_points_ntt_dev(h, 0, 0, None, 10, c_vp(buf.data_ptr())) == _native.ERR_ARG
    assert lib.b200zk_points_ntt_dev(h, 0, 1, c_vp(pts.data_ptr()), 10, None) == _native.ERR_ARG
    assert lib.b200zk_points_ntt_dev(None, 0, 0, c_vp(pts.data_ptr()), 10, c_vp(buf.data_ptr())) == _native.ERR_ARG
    assert lib.b200zk_points_ntt_dev(h, 99, 0, c_vp(pts.data_ptr()), 10, c_vp(buf.data_ptr())) == _native.ERR_ARG
    for g2, log_n in ((False, 10), (True, 6)):
        p = net.generate_g2(78, 1 << log_n) if g2 else net.generate_g1(78, 1 << log_n)
        inplace = p.clone()
        want = _ntt(net, p, g2)
        assert torch.equal(p, inplace)
        _ntt(net, inplace, g2, out=inplace)
        assert torch.equal(inplace, want) and not torch.equal(p, want)


# ---- against snarkjs ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_export_of_the_snarkjs_key_hashes_to_the_cs_hash_snarkjs_wrote(net):
    """The reference's complex-circuit zkey (snarkjs `zkey new`, no contributions, domain 2^14), rebuilt byte for byte:
    Blake2b-512 of its export up to the csHash is the csHash in its section 10."""
    import artefact_writer as aw
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import circom
    x = np.load(os.path.join(G, "reference_artefacts.npz"))
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    secs = aw.zkey_sections(d)
    secs[10] = x["zkey_sec10"].tobytes()
    zkey = aw.container(b"zkey", [(int(sid), secs[int(sid)]) for sid in x["zkey_order"]])
    assert hashlib.sha256(zkey).hexdigest() == str(x["zkey_sha256"])
    buf = circom.zkey_export_bellman(net, zkey)
    n_vars, n_public, n = (int(v) for v in d["dims"][:3])
    b = formats.parse_bellman(buf)
    assert len(buf) == formats.bellman_size(n_public + 1, n - 1, n_vars - n_public - 1, n_vars)
    assert hashlib.blake2b(buf[:b.params_end], digest_size=64).digest() == secs[10][:64]
    assert buf[b.params_end:] == secs[10][:64] + struct.pack(">I", 0)


# ---- synthetic ceremonies -------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def _sha256():
    import artefact_writer as aw
    x = np.load(os.path.join(G, "reference_artefacts.npz"))
    s = dict(np.load(os.path.join(G, "sha256_circuit.npz")))
    secs = {1: x["sha256_r1cs_sec1"].tobytes(), 2: aw.r1cs_constraints(s, int(s["dims"][2])), 3: x["sha256_r1cs_sec3"].tobytes()}
    return s, aw.container(b"r1cs", [(int(sid), secs[int(sid)]) for sid in x["sha256_r1cs_order"]])


def _tiny_r1cs():
    return open(os.path.join(G, "circom2_multiplier2.r1cs"), "rb").read()


@pytest.fixture(scope="module")
def ceremonies(net, tmp_path_factory):
    import ptau_writer as pw
    tmp = tmp_path_factory.mktemp("ptau")
    return {p: pw.write_ptau(str(tmp / ("p%d.ptau" % p)), pw.sections_gpu(net, TOXIC["tau"], TOXIC["alpha"], TOXIC["beta"], p))
            for p in (15, 17)}


@pytest.mark.gpu
@pytest.mark.parametrize("circuit", ["sha256", "tiny"])
@pytest.mark.parametrize("power", [15, 17])
def test_exported_h_is_the_tau_basis_after_0_1_and_2_contributions(net, ceremonies, power, circuit):
    from distributed_groth16_b200.groth16 import bellman, circom, phase1, phase2, setup
    r1cs = _sha256()[1] if circuit == "sha256" else _tiny_r1cs()
    z = circom.zkey_new(net, r1cs, ceremonies[power], cs_hash=True)
    t, delta = TOXIC["tau"], 1
    for stage in range(3):
        if stage:
            z, _ = phase2.contribute(net, z, X[stage - 1], _g1(S[stage - 1]))
            delta = delta * X[stage - 1] % R
        n = struct.unpack_from("<I", phase2._section(z, 2), 80)[0]
        assert n == (1 << 15 if circuit == "sha256" else 4)
        buf = bellman.export(net, z)
        want = setup._fixed_base(net, setup._powers(net, t, (pow(t, n, R) - 1) * pow(delta, -1, R) % R, n - 1))
        assert _span(buf, "h") == phase1.points_encode(net, want).cpu().numpy().tobytes(), stage
        if stage == 0:
            b = bellman.formats.parse_bellman(buf)
            assert hashlib.blake2b(buf[:b.params_end], digest_size=64).digest() == phase2._section(z, 10)[:64] == b.cs_hash


@pytest.fixture(scope="module")
def rounds(net, ceremonies):
    """On the sha256 key with the csHash: one contribution by the direct path and the same contribution (x, s, name) by
    a bellman round."""
    from distributed_groth16_b200.groth16 import bellman, circom, phase2
    r1cs = _sha256()[1]
    z0 = circom.zkey_new(net, r1cs, ceremonies[15], cs_hash=True)
    direct, hd = phase2.contribute(net, z0, X[0], _g1(S[0]), name="one")
    challenge = circom.zkey_export_bellman(net, z0)
    t = {}
    resp, hb = bellman.contribute(net, challenge, X[0], _g1(S[0]), timings=t)
    assert set(t) == {"ntt_s", "mul_powers_s", "decode_s", "scale_s", "encode_s", "transfer_s", "host_s"}
    imported = circom.zkey_import_bellman(net, z0, resp, name="one")
    return dict(r1cs=r1cs, ptau=ceremonies[15], z0=z0, direct=direct, hd=hd, challenge=challenge, resp=resp, hb=hb,
                imported=imported)


@pytest.mark.gpu
def test_a_bellman_round_equals_the_direct_contribution(net, rounds):
    import artefact_writer as aw
    from oracle import layout
    from distributed_groth16_b200.groth16 import circom
    assert rounds["hb"] == rounds["hd"]
    a, b = _sections(rounds["imported"]), _sections(rounds["direct"])
    assert list(a) == list(b)
    for sid in (1, 2, 3, 4, 5, 6, 7, 8, 10):
        assert a[sid] == b[sid], sid
    assert a[9] != b[9]                              # they differ in the unused tau component
    e = circom.zkey_export_bellman(net, rounds["imported"])
    assert e == circom.zkey_export_bellman(net, rounds["direct"]) == rounds["resp"]
    s = _sha256()[0]
    wtns = aw.write_wtns([int.from_bytes(r.tobytes(), "little") for r in s["witness"]])
    r_, s_ = layout.fr_to_arr([12345])[0], layout.fr_to_arr([67890])[0]
    proofs = [circom.groth16_prove(net, z, wtns, r=r_, s=s_) for z in (rounds["imported"], rounds["direct"])]
    assert proofs[0] == proofs[1]
    for z in (rounds["imported"], rounds["direct"]):
        assert circom.groth16_verify(net, circom.zkey_export_verificationkey(net, z), proofs[0][1], proofs[0][0])


@pytest.mark.gpu
def test_a_chain_of_direct_and_bellman_rounds_verifies(net, rounds):
    from distributed_groth16_b200.groth16 import bellman, circom, phase2
    z1 = rounds["direct"]
    r2, h2 = bellman.contribute(net, circom.zkey_export_bellman(net, z1), X[1], _g1(S[1]))
    z2 = circom.zkey_import_bellman(net, z1, r2, name="bellman")
    r3, h3 = bellman.contribute(net, circom.zkey_export_bellman(net, z2), X[2], _g1(S[2]))
    r4, h4 = bellman.contribute(net, r3, X[3], _g1(S[3]))
    z3 = circom.zkey_import_bellman(net, z2, r4, name="pair")
    z4, h5 = circom.zkey_beacon(net, z3, BEACON, 10, name="beacon")
    hashes = [rounds["hd"], h2, h3, h4, h5]
    for i, z in enumerate([z1, z2, z3, z4]):
        rep = circom.zkey_verify(net, rounds["r1cs"], rounds["ptau"], z, check_cs_hash=True)
        assert rep.ok, (i, rep.failures)
    assert [c[0] for c in rep.contributions] == ["one", "bellman", "pair", "pair", "beacon"]
    assert [c[1] for c in rep.contributions] == [0, 0, 0, 0, 1]
    assert [c[2] for c in rep.contributions] == hashes
    assert circom.zkey_export_bellman(net, z3) == r4


@pytest.mark.gpu
def test_zkey_verify_checks_every_tau_component_of_h(net, rounds):
    """The imported key (H_(n-1) = infinity) and the direct one (H_(n-1) scaled) verify; a key whose H_(n-1) is another
    point, or whose H is altered in one of the first n - 1 tau components, does not."""
    from distributed_groth16_b200.groth16 import bellman, phase1, phase2
    assert phase2.verify(net, rounds["r1cs"], rounds["ptau"], rounds["imported"]).ok
    resp = rounds["resp"]
    h = phase1.points_decode(net, _span(resp, "h"))
    n = h.shape[0] + 1
    other = net.generate_g1(5, 1)

    def with_tau(pts):
        sec9 = bellman._h_from_tau(net, pts, n, bellman._timings()).cpu().numpy().tobytes()
        return phase2._replace_sections(rounds["imported"], {9: sec9})

    import torch
    last = with_tau(torch.cat([h, other]))
    rep = phase2.verify(net, rounds["r1cs"], rounds["ptau"], last)
    assert not rep.ok and rep.failures == ["the last tau component of the H section is neither infinity nor the initial one "
                                           "times delta^-1"], rep.failures
    for i in (0, 7, n - 2):
        bad = h.clone()
        bad[i] = other[0]
        rep = phase2.verify(net, rounds["r1cs"], rounds["ptau"], with_tau(bad))
        assert not rep.ok and rep.failures == ["the H section is not the initial one times delta^-1 in its first n - 1 tau "
                                               "components"], (i, rep.failures)


@pytest.mark.gpu
def test_import_refuses_responses_that_do_not_answer_the_key(net, rounds, ceremonies):
    from oracle import bn254 as o
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import bellman, circom, phase2
    import phase2_oracle
    z0, resp = rounds["z0"], rounds["resp"]
    b = formats.parse_bellman(resp)
    imp = lambda z, r: bellman.import_response(net, z, r, name="x")

    def put(part, i, w, new):
        off = b.spans[part][0] + w * i
        assert resp[off:off + w] != new
        return resp[:off] + new + resp[off + w:]

    def point(part, i, w):
        off = b.spans[part][0] + w * i
        return resp[off:off + w]

    zero_key = circom.zkey_new(net, rounds["r1cs"], rounds["ptau"])
    with pytest.raises(ValueError, match="csHash"):
        imp(zero_key, resp)
    with pytest.raises(ValueError, match="no new contribution"):
        imp(z0, rounds["challenge"])
    # an altered earlier record: a round on the key with one record, the record's transcript changed
    z1 = rounds["direct"]
    r2, _ = bellman.contribute(net, circom.zkey_export_bellman(net, z1), X[1], _g1(S[1]))
    b2 = formats.parse_bellman(r2)
    off = b2.records_offset + 330
    with pytest.raises(ValueError, match="record 0 differs"):
        imp(z1, r2[:off] + bytes([r2[off] ^ 1]) + r2[off + 1:])
    a_i = next(i for i in range(b.counts["a"] - 1) if point("a", i, 64) != point("a", i + 1, 64))
    b1_i = next(i for i in range(b.counts["b1"] - 1) if point("b1", i, 64) != point("b1", i + 1, 64))
    b2_i = next(i for i in range(b.counts["b2"] - 1) if point("b2", i, 128) != point("b2", i + 1, 128))
    changed = {"alpha_g1 point 0": put("alpha_g1", 0, 64, point("beta_g1", 0, 64)),
               "beta_g1 point 0": put("beta_g1", 0, 64, point("alpha_g1", 0, 64)),
               "beta_g2 point 0": put("beta_g2", 0, 128, point("delta_g2", 0, 128)),
               "gamma_g2 point 0": put("gamma_g2", 0, 128, point("beta_g2", 0, 128)),
               "ic point 1": put("ic", 1, 64, point("ic", 0, 64)),
               "a point %d" % a_i: put("a", a_i, 64, point("a", a_i + 1, 64)),
               "b1 point %d" % b1_i: put("b1", b1_i, 64, point("b1", b1_i + 1, 64)),
               "b2 point %d" % b2_i: put("b2", b2_i, 128, point("b2", b2_i + 1, 128))}
    for what, r in changed.items():
        with pytest.raises(ValueError, match=what + " differs"):
            imp(z0, r)
    # another circuit's response: the counts differ
    tiny = circom.zkey_new(net, _tiny_r1cs(), ceremonies[15])
    tr, _ = bellman.contribute(net, circom.zkey_export_bellman(net, tiny), X[0], _g1(S[0]))
    with pytest.raises(ValueError, match="IC holds 2 points|H holds 3 points"):
        imp(z0, tr)
    for r in (resp[:-1], resp + b"\0", resp[:b.spans["h"][0] - 4] + struct.pack(">I", b.counts["h"] - 1) + resp[b.spans["h"][0]:]):
        with pytest.raises(formats.FormatError):
            imp(z0, r)
    # off the curve: y + 1
    for part, i in (("h", 5), ("l", 3)):
        p = point(part, i, 64)
        y = int.from_bytes(p[32:], "big")
        with pytest.raises(formats.FormatError, match="%s point %d is not a valid" % (part.upper(), i)):
            imp(z0, put(part, i, 64, p[:32] + ((y + 1) % o.P).to_bytes(32, "big")))
    # delta_2 on the twist, outside the order-r subgroup
    x = 5
    while True:
        x += 1
        try:
            q = o.g2_decompress(x.to_bytes(32, "little") + (7).to_bytes(32, "little"))
        except ValueError:
            continue
        if o.G2.from_jac(o.G2.jac_mul(o.G2.to_jac(q), o.R)) is not None:
            break
    with pytest.raises(formats.FormatError, match="delta_g2 point 0 is not a valid uncompressed G2 point of the order-r"):
        imp(z0, put("delta_g2", 0, 128, phase2_oracle.u_g2(q)))
    assert phase2.verify(net, rounds["r1cs"], rounds["ptau"], imp(z0, resp)).ok


@pytest.mark.gpu
@pytest.mark.parametrize("power", [2, 3])
def test_tiny_circuit_equals_the_oracle(net, tmp_path, power):
    import bellman_oracle as bo
    import ptau_writer as pw
    from oracle import bn254 as o, layout
    from distributed_groth16_b200.groth16 import bellman, circom
    r1cs = _tiny_r1cs()
    path = pw.write_ptau(str(tmp_path / "tiny.ptau"), pw.sections_oracle(TINY["tau"], TINY["alpha"], TINY["beta"], power))
    z0 = circom.zkey_new(net, r1cs, path, cs_hash=True)
    e = bellman.export(net, z0)
    assert e == bo.export(z0)
    s_pt = o.G1.mul(o.G1_GEN, S[0])
    resp, h = bellman.contribute(net, e, X[0], layout.g1_to_arr([s_pt])[0])
    assert (resp, h) == bo.contribute(e, X[0], s_pt)
    z1 = bellman.import_response(net, z0, resp, name="tiny")
    assert z1 == bo.import_response(z0, resp, name="tiny")
    assert circom.zkey_verify(net, r1cs, path, z1, check_cs_hash=True).ok


@pytest.mark.gpu
def test_round_trip_at_domain_2_22(net):
    """A synthetic key with a 2^22 domain: export(import(response)) == response."""
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import bellman, phase1
    n, n_vars, n_public = 1 << 22, 12, 1
    host = lambda t: t.cpu().numpy().view(np.uint64)
    g1, g2 = phase1.G1_GEN, phase1.G2_GEN
    zk = formats.ZKey(n_vars=n_vars, n_public=n_public, domain_size=n, alpha_g1=g1, beta_g1=g1, beta_g2=g2, gamma_g2=g2,
                      delta_g1=g1, delta_g2=g2, ic=host(net.generate_g1(1, n_public + 1)), a_query=host(net.generate_g1(2, n_vars)),
                      b_g1_query=host(net.generate_g1(3, n_vars)), b_g2_query=host(net.generate_g2(4, n_vars)),
                      l_query=host(net.generate_g1(5, n_vars - n_public - 1)), h_query=host(net.generate_g1(6, n)),
                      coef_matrix=np.zeros(0, np.uint32), coef_row=np.zeros(0, np.uint32), coef_col=np.zeros(0, np.uint32),
                      coef_val_r2=np.zeros((0, 4), np.uint64))
    z0 = formats.write_zkey(zk)
    e = bellman.export(net, z0)
    resp, _ = bellman.contribute(net, e, X[0], _g1(S[0]))
    z1 = bellman.import_response(net, z0, resp)
    assert bellman.export(net, z1) == resp
    assert formats.read_zkey(z1).h_query.shape == (n, 8)
