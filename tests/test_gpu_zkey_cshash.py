"""The circuit hash (csHash) of snarkjs `zkey new` on the GPU: the pointwise-difference kernel (b200zk_points_sub_dev)
against fixed-base multiplication, the product path against the hash snarkjs wrote into the reference's complex-circuit
zkey, the H points by subtraction against the H points by the Lagrange identity on synthetic ceremonies, chunking, the
tiny circuit byte for byte against the pure-Python restatement, and `zkey_new(cs_hash=True)` / `zkey_verify(check_cs_hash=
True)` through a contribute / contribute / beacon chain."""
import functools
import os
import struct
import sys

import numpy as np
import pytest

from distributed_groth16_b200._native import c_vp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")
TOXIC = dict(tau=0x2468ACE013579BDF2468ACE013579BDF, alpha=31415926535897932384, beta=27182818284590452353)
TINY = dict(tau=0x1234567890ABCDEF, alpha=1111111111111111111, beta=2222222222222222223)
X1, X2 = 0x5EC12E7_0000_1111_2222_3333_4444_5555_6666_7777, 987654321987654321987654321
S1, S2 = 0xABCDEF0123456789, 0x1111222233334444555566667777
BEACON = bytes.fromhex("0102030405060708090a0b0c0d0e0f101112131415161718191a1b1c1d1e1f")


def _lincomb(net, a, b, s0: int, s1: int):
    """a s0 + b s1 over Montgomery Fr tensors (b200zk_fr_lincomb_dev)."""
    import torch
    from distributed_groth16_b200.groth16.setup import _mont_limbs
    s = np.concatenate([_mont_limbs(s0), _mont_limbs(s1), _mont_limbs(0), _mont_limbs(1)])
    out = torch.empty_like(a)
    net.check(net._lib.b200zk_fr_lincomb_dev(net._h, c_vp(a.data_ptr()), c_vp(b.data_ptr()), c_vp(a.data_ptr()),
                                             c_vp(s.ctypes.data), int(a.shape[0]), c_vp(out.data_ptr())))
    return out


class _TauG1:
    """What the circuit hash reads of a ceremony, section 2 (tau^i G1), from a host array."""

    def __init__(self, pts):
        self.pts = np.ascontiguousarray(pts, dtype=np.uint64).reshape(-1, 8)

    def has_section(self, sid):
        return sid == 2

    def section_span(self, sid):
        return 0, self.pts.shape[0] * 64

    def points(self, sid, first, count, width):
        assert sid == 2 and width == 8
        return self.pts[first:first + count].copy()


def _h_by_identity(net, h_query):
    """H_i = -2n w_2n^i iNTT(h)_((n - i) mod n), i < n - 1, from the n points of zkey section 9 (CUDA) on the device."""
    import torch
    from oracle import bn254 as o
    from distributed_groth16_b200.groth16 import phase1, ptau
    n = int(h_query.shape[0])
    y = ptau.points_intt(net, h_query)
    idx = (n - torch.arange(n - 1, device=y.device)) % n
    return phase1.points_mul_powers(net, y[idx].contiguous(), (-2 * n) % o.R, o.fr_root_of_unity(2 * n))


# ---- the kernel ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("g2,n", [(False, 1), (False, 200), (False, (1 << 20) + 77), (False, 1 << 23),
                                  (True, 1), (True, 200), (True, 1 << 22)])
def test_points_sub_equals_fixed_base_mul_of_the_difference(net, g2, n):
    """a_i - b_i == (x_i - y_i) G for random logs, with a = b (infinity), a = -b (a doubling), a, b or both at infinity,
    n not a multiple of the block (128), and calls in place on either input."""
    import torch
    from distributed_groth16_b200.groth16 import phase1
    from distributed_groth16_b200.groth16.setup import _fixed_base
    x, y = net.generate_fr(1000 + n, n), net.generate_fr(2000 + n, n)
    if n >= 8:
        x[[2, 4]] = 0                                             # a at infinity (and both at 4)
        negx = _lincomb(net, x, x, -1, 0)
        y[[0, n - 1]] = x[[0, n - 1]]                             # a = b
        y[[1, n - 2]] = negx[[1, n - 2]]                          # a = -b
        y[[3, 4]] = 0                                             # b at infinity
    d = _lincomb(net, x, y, 1, -1)
    a, b, want = _fixed_base(net, x, g2), _fixed_base(net, y, g2), _fixed_base(net, d, g2)
    if n >= 8:
        inf = torch.zeros_like(want[0])
        assert torch.equal(want[0], inf) and torch.equal(want[n - 1], inf) and not torch.equal(want[1], inf)
    out = phase1.points_sub(net, a, b, g2)
    net.sync(0)
    assert torch.equal(out, want)
    b_copy = b.clone()
    phase1.points_sub(net, a, b_copy, g2, out=b_copy)
    phase1.points_sub(net, a, b, g2, out=a)
    net.sync(0)
    assert torch.equal(b_copy, want) and torch.equal(a, want)


@pytest.mark.gpu
def test_points_sub_argument_errors(net):
    import torch
    from distributed_groth16_b200 import _native
    from distributed_groth16_b200.groth16 import phase1
    lib, t = net._lib, net.generate_g1(7, 4)
    p = c_vp(t.data_ptr())
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert lib.b200zk_points_sub_dev(net._h, 0, 0, *args[:2], 4, args[2]) == _native.ERR_ARG
    assert lib.b200zk_points_sub_dev(net._h, 0, 1, None, None, 0, None) == _native.OK
    assert lib.b200zk_points_sub_dev(net._h, 99, 0, p, p, 4, p) == _native.ERR_ARG
    assert lib.b200zk_points_sub_dev(None, 0, 0, p, p, 4, p) == _native.ERR_ARG
    with pytest.raises(ValueError, match="shapes"):
        phase1.points_sub(net, t, t[:3])
    net.sync(0)
    assert torch.equal(phase1.points_sub(net, t, t), torch.zeros_like(t))       # the context still works


# ---- against snarkjs ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_product_path_reproduces_the_cs_hash_snarkjs_wrote_into_the_reference_zkey(net):
    """H from section 9 by the identity on the device, then cshash.cs_hash with those points as tau^(n+i) G1 and
    infinity as tau^i G1 (so the sub kernel passes them through): the 64 bytes of the reference file's section 10."""
    from distributed_groth16_b200.groth16 import cshash
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    want = np.load(os.path.join(G, "reference_artefacts.npz"))["zkey_sec10"].tobytes()[:64]
    n = int(d["dims"][2])
    h = _h_by_identity(net, net.to_device(d["h_query"])).cpu().numpy().view(np.uint64)
    dev = lambda k: net.to_device(np.ascontiguousarray(d[k]))
    q = dict(domain_size=n, alpha_g1=d["vk_g1"][0], beta_g1=d["vk_g1"][1], beta_g2=d["vk_g2"][0], gamma_g2=d["vk_g2"][2],
             delta_g1=d["vk_g1"][2], delta_g2=d["vk_g2"][1], ic=dev("ic"), l_query=dev("l_query"), a_query=dev("a_query"),
             b_g1_query=dev("b_g1_query"), b_g2_query=dev("b_g2_query"))
    tau = _TauG1(np.concatenate([np.zeros((n, 8), dtype=np.uint64), h]))
    assert cshash.cs_hash(net, q, tau) == want
    assert cshash.cs_hash(net, q, tau, chunk=1000) == want


# ---- synthetic ceremonies -------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def _sha256_r1cs():
    import artefact_writer as aw
    x = np.load(os.path.join(G, "reference_artefacts.npz"))
    s = dict(np.load(os.path.join(G, "sha256_circuit.npz")))         # in memory: the writer slices it per constraint
    secs = {1: x["sha256_r1cs_sec1"].tobytes(), 2: aw.r1cs_constraints(s, int(s["dims"][2])), 3: x["sha256_r1cs_sec3"].tobytes()}
    return aw.container(b"r1cs", [(int(sid), secs[int(sid)]) for sid in x["sha256_r1cs_order"]])


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
def test_h_by_subtraction_equals_h_by_the_identity_and_the_toxic_waste(net, ceremonies, power, circuit):
    import torch
    from oracle import bn254 as o
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase1, setup
    r1 = formats.read_r1cs(_sha256_r1cs() if circuit == "sha256" else _tiny_r1cs())
    with formats.read_ptau(ceremonies[power]) as pt:
        q = setup.ptau_key_points(net, r1, pt)
        n = q["domain_size"]
        by_sub = phase1.points_sub(net, net.to_device(pt.points(2, n, n - 1, 8)), net.to_device(pt.points(2, 0, n - 1, 8)))
    by_identity = _h_by_identity(net, q["h_query"])
    t = TOXIC["tau"]
    want = setup._fixed_base(net, setup._powers(net, t, pow(t, n, o.R) - 1, n - 1))           # tau^i (tau^n - 1)
    net.sync(0)
    assert n == (1 << 15 if circuit == "sha256" else 4)
    assert torch.equal(by_sub, want) and torch.equal(by_identity, want)


@pytest.mark.gpu
def test_chunked_hash_equals_one_chunk_at_domain_2_20(net):
    from distributed_groth16_b200.groth16 import cshash
    from distributed_groth16_b200.groth16.phase1 import G1_GEN, G2_GEN
    n, n_vars, n_public = 1 << 20, (1 << 20) - 9, 2
    tau = _TauG1(net.generate_g1(31, 2 * n - 1).cpu().numpy().view(np.uint64))
    a = net.generate_g1(33, n_vars)
    a[[0, 5, n_vars - 1]] = 0                                      # points at infinity are hashed too
    q = dict(domain_size=n, alpha_g1=G1_GEN, beta_g1=G1_GEN, beta_g2=G2_GEN, gamma_g2=G2_GEN, delta_g1=G1_GEN,
             delta_g2=G2_GEN, ic=net.generate_g1(32, n_public + 1), l_query=net.generate_g1(34, n_vars - n_public - 1),
             a_query=a, b_g1_query=net.generate_g1(35, n_vars), b_g2_query=net.generate_g2(36, n_vars))
    t = {}
    one = cshash.cs_hash(net, q, tau, chunk=1 << 22, timings=t)
    assert set(t) == {"sub_s", "encode_s", "copy_s", "hash_s", "file_s"}
    assert cshash.cs_hash(net, q, tau, chunk=1 << 18) == one
    assert cshash.cs_hash(net, q, tau, chunk=(1 << 18) + 3) == one
    short = _TauG1(tau.pts[:2 * n - 2])
    from distributed_groth16_b200 import formats
    with pytest.raises(formats.FormatError, match="section 2 holds"):
        cshash.cs_hash(net, q, short)


@pytest.mark.gpu
def test_tiny_circuit_zkey_with_cs_hash_equals_the_oracle(net, tmp_path):
    """circom2_multiplier2 with a power-3 ceremony: zkey_new(cs_hash=True) is the pure-Python zkey new with the pure-Python
    csHash in section 10, byte for byte."""
    import cshash_oracle as co
    import ptau_writer as pw
    import zkey_oracle
    from distributed_groth16_b200.groth16 import circom, phase2
    secs = pw.sections_oracle(TINY["tau"], TINY["alpha"], TINY["beta"], 3)
    path = pw.write_ptau(str(tmp_path / "tiny.ptau"), secs)
    zk = zkey_oracle.zkey_new(_tiny_r1cs(), pw.ptau_bytes(secs))
    cs = co.cs_hash(zk, co.h_from_tau(secs[2], 4))
    assert circom.zkey_new(net, _tiny_r1cs(), path, cs_hash=True) == phase2._replace_sections(zk, {10: cs + struct.pack("<I", 0)})
    assert circom.zkey_cs_hash(net, _tiny_r1cs(), path) == cs


# ---- the public interface through a ceremony ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def chains(net, ceremonies):
    """contribute / contribute / beacon on the sha256 key with the csHash and on the default (zero-hash) key."""
    from oracle import bn254 as o, layout
    from distributed_groth16_b200.groth16 import circom, phase2
    r1cs, path = _sha256_r1cs(), ceremonies[15]
    g1 = lambda k: layout.g1_to_arr([o.G1.mul(o.G1_GEN, k)])[0]
    out = dict(r1cs=r1cs, ptau=path, hash=circom.zkey_cs_hash(net, r1cs, path))
    for name, flag in (("cs", True), ("zero", False)):
        z0 = circom.zkey_new(net, r1cs, path, cs_hash=flag)
        z1, h1 = phase2.contribute(net, z0, X1, g1(S1), name="first")
        z2, h2 = phase2.contribute(net, z1, X2, g1(S2), name="second")
        z3, h3 = circom.zkey_beacon(net, z2, BEACON, 10, name="final beacon")
        out[name] = dict(zkeys=[z0, z1, z2, z3], hashes=[h1, h2, h3])
    return out


@pytest.mark.gpu
def test_zkey_new_with_cs_hash_differs_only_in_the_hash(chains):
    from distributed_groth16_b200.groth16 import phase2
    a, b = chains["cs"]["zkeys"][0], chains["zero"]["zkeys"][0]
    off = next(o_ for sid, o_, _ in phase2._section_table(b) if sid == 10)
    assert len(a) == len(b) and a[:off] == b[:off] and a[off + 64:] == b[off + 64:]
    assert a[off:off + 64] == chains["hash"] != bytes(64) and b[off:off + 64] == bytes(64)


@pytest.mark.gpu
def test_zkey_verify_with_the_check_accepts_every_stage(net, chains):
    from distributed_groth16_b200.groth16 import circom
    for i, z in enumerate(chains["cs"]["zkeys"]):
        rep = circom.zkey_verify(net, chains["r1cs"], chains["ptau"], z, check_cs_hash=True)
        assert rep.ok, (i, rep.failures)
        assert rep.cs_hash == rep.cs_hash_expected == chains["hash"]
        assert [c[2] for c in rep.contributions] == chains["cs"]["hashes"][:i]
    # every transcript starts from the csHash: the chain's contribution hashes all change
    assert all(x != y for x, y in zip(chains["cs"]["hashes"], chains["zero"]["hashes"]))


@pytest.mark.gpu
def test_zkey_verify_without_the_check_is_unchanged(net, chains):
    from distributed_groth16_b200.groth16 import circom
    for name in ("cs", "zero"):
        z = chains[name]["zkeys"][3]
        rep = circom.zkey_verify(net, chains["r1cs"], chains["ptau"], z)
        assert rep.ok, rep.failures
        assert rep.cs_hash == (chains["hash"] if name == "cs" else bytes(64)) and rep.cs_hash_expected == b""
        assert [c[0] for c in rep.contributions] == ["first", "second", "final beacon"]
        assert [c[2] for c in rep.contributions] == chains[name]["hashes"]


@pytest.mark.gpu
def test_zkey_verify_with_the_check_rejects_a_wrong_cs_hash(net, chains):
    from distributed_groth16_b200.groth16 import circom, phase2
    z0 = chains["cs"]["zkeys"][0]
    sec10 = phase2._section(z0, 10)
    flipped = bytes([sec10[0] ^ 0x01]) + sec10[1:]
    other = circom.zkey_cs_hash(net, _tiny_r1cs(), chains["ptau"])
    assert other != chains["hash"]
    cases = {"default": chains["zero"]["zkeys"][0], "bit flipped": phase2._replace_sections(z0, {10: flipped}),
             "another circuit's": phase2._replace_sections(z0, {10: other + struct.pack("<I", 0)})}
    for what, z in cases.items():
        rep = circom.zkey_verify(net, chains["r1cs"], chains["ptau"], z, check_cs_hash=True)
        assert not rep.ok, what
        assert len(rep.failures) == 1 and "circuit hash" in rep.failures[0], (what, rep.failures)
        assert rep.cs_hash_expected == chains["hash"]
