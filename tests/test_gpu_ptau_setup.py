"""Groth16 setup from a Powers-of-Tau file on the GPU (snarkjs `zkey new`): the CSR product over points
(b200zk_points_spmv_dev) against the oracle, the key from a synthetic ceremony against the toxic-waste setup with the same
(tau, alpha, beta) and gamma = delta = 1, proofs through the written zkey, and the tiny circuit byte for byte against the
pure-Python zkey new."""
import os
import sys

import numpy as np
import pytest

from distributed_groth16_b200._native import c_vp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")
TOXIC = dict(tau=0x1234567890ABCDEF1234567890ABCDEF, alpha=11111111111111111111, beta=22222222222222222223)


def _spmv(net, ptr, idx, val, points, n_rows, g2):
    import torch
    out = torch.full((n_rows, 16 if g2 else 8), -1, dtype=torch.int64, device=points.device)
    d = lambda a: net.to_device(np.ascontiguousarray(a).view(np.int32) if a.dtype == np.uint32 else a)
    ptr_d, idx_d, val_d = d(ptr), d(idx), d(val)
    net.check(net._lib.b200zk_points_spmv_dev(net._h, 0, int(g2), c_vp(ptr_d.data_ptr()), c_vp(idx_d.data_ptr()),
                                              c_vp(val_d.data_ptr()), c_vp(points.data_ptr()), n_rows, c_vp(out.data_ptr())))
    return out.cpu().numpy().view(np.uint64)


@pytest.mark.gpu
@pytest.mark.parametrize("g2", [False, True])
def test_points_spmv_matches_the_oracle(net, cref, g2):
    """Empty rows, one row longer than the MSM threshold (256), zero and r - 1 coefficients, short (< 2^64) and full ones,
    r - short ones (the signed path) and infinity points."""
    from oracle import bn254 as o, layout
    rng = np.random.default_rng(7 + g2)
    n_pts, w = 96, 16 if g2 else 8
    pts = (cref.g2_generate if g2 else cref.g1_generate)(31 + g2, n_pts)
    pts[[5, 17, 60]] = 0                                                    # infinity
    lens = rng.integers(0, 7, size=48)
    lens[[0, 9, 30, 47]] = 0
    lens[13] = 300
    ptr = np.zeros(len(lens) + 1, dtype=np.uint32)
    ptr[1:] = np.cumsum(lens)
    nnz = int(ptr[-1])
    idx = rng.integers(0, n_pts, size=nnz).astype(np.uint32)
    idx[ptr[13]:ptr[13] + 10] = 5                                           # infinity inside the long row
    full = [int.from_bytes(r.tobytes(), "little") for r in cref.fr_generate(99 + g2, nnz)]
    kinds = rng.integers(0, 6, size=nnz)
    vals = []
    for k, f in zip(kinds, full):
        short = int(rng.integers(1, 1 << 62)) << int(rng.integers(0, 3))
        vals.append([0, o.R - 1, short, o.R - short, f % o.R, 1][k])
    vals = [v % o.R for v in vals]
    val_limbs = layout.fr_to_arr(vals)
    got = _spmv(net, ptr, idx, val_limbs, net.to_device(pts), len(lens), g2)
    msm = cref.msm_g2 if g2 else cref.msm_g1
    for r in range(len(lens)):
        b, e = int(ptr[r]), int(ptr[r + 1])
        if b == e:
            assert not got[r].any(), r
            continue
        exp, inf = msm(pts[idx[b:e]], val_limbs[b:e])
        assert (got[r] == (np.zeros(w, dtype=np.uint64) if inf else exp)).all(), (r, e - b)


def _sha256():
    import artefact_writer as aw
    x = np.load(os.path.join(G, "reference_artefacts.npz"))
    s = np.load(os.path.join(G, "sha256_circuit.npz"))
    secs = {1: x["sha256_r1cs_sec1"].tobytes(), 2: aw.r1cs_constraints(s, int(s["dims"][2])), 3: x["sha256_r1cs_sec3"].tobytes()}
    return s, aw.container(b"r1cs", [(int(sid), secs[int(sid)]) for sid in x["sha256_r1cs_order"]])


@pytest.fixture(scope="module")
def sha256_keys(net, tmp_path_factory):
    """zkey_new on the sha256 circuit with synthetic ceremonies of power 15 (= the circuit's) and 16, and the toxic-waste
    key of the same (tau, alpha, beta) with gamma = delta = 1 (its query tensors captured at the upload)."""
    import ptau_writer as pw
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import circom, setup
    from distributed_groth16_b200.groth16.proving_key import ProvingKey
    s, r1cs = _sha256()
    out = {"s": s, "r1cs": r1cs}
    tmp = tmp_path_factory.mktemp("ptau")
    for p in (15, 16):
        path = pw.write_ptau(str(tmp / ("p%d.ptau" % p)), pw.sections_gpu(net, TOXIC["tau"], TOXIC["alpha"], TOXIC["beta"], p))
        out["zkey%d" % p] = circom.zkey_new(net, r1cs, path)
        out["ptau%d" % p] = path
    with formats.read_ptau(out["ptau15"]) as pt:
        out["pk15"], out["vk15"], out["mats15"] = setup.setup_from_ptau(net, formats.read_r1cs(r1cs), pt)
    captured = {}
    orig = ProvingKey.from_device.__func__

    def capture(cls, net_, a, b1, b2, l, h, n_inputs, vk_points):
        captured.update(a_query=a, b_g1_query=b1, b_g2_query=b2, l_query=l, h_query=h, vk_points=np.array(vk_points))
        return orig(cls, net_, a, b1, b2, l, h, n_inputs, vk_points)

    n_wires, n_pub, n_cons = (int(v) for v in s["dims"])
    coo = lambda k: (s[k + "_rows"], s[k + "_cols"], s[k + "_vals"])
    mp = pytest.MonkeyPatch()
    mp.setattr(ProvingKey, "from_device", classmethod(capture))
    try:
        out["pk_toxic"], out["vk_toxic"], out["mats_toxic"] = setup.circuit_specific_setup(
            net, n_wires, n_pub + 1, n_cons, coo("a"), coo("b"), coo("c"), (TOXIC["tau"], TOXIC["alpha"], TOXIC["beta"], 1, 1))
    finally:
        mp.undo()
    out["toxic"] = {k: (v.cpu().numpy().view(np.uint64) if hasattr(v, "cpu") else v) for k, v in captured.items()}
    yield out
    out["pk15"].free()
    out["pk_toxic"].free()


@pytest.mark.gpu
def test_sha256_key_from_a_power_15_ceremony_equals_the_toxic_waste_key(sha256_keys):
    from distributed_groth16_b200 import formats
    k, t = sha256_keys, sha256_keys["toxic"]
    zk = formats.read_zkey(k["zkey15"])
    for name in ("a_query", "b_g1_query", "b_g2_query", "l_query", "h_query"):
        assert (getattr(zk, name) == t[name]).all(), name
    assert (zk.vk_points() == t["vk_points"]).all()
    vk, vt = k["vk15"], k["vk_toxic"]
    assert (zk.ic == vt.gamma_abc_g1).all() and (vk.gamma_abc_g1 == vt.gamma_abc_g1).all()
    for name in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2"):
        assert (np.asarray(getattr(vk, name)) == np.asarray(getattr(vt, name))).all(), name
    assert (zk.gamma_g2 == vt.gamma_g2).all() and (zk.delta_g2 == vt.delta_g2).all()


def _prove_and_check(net, k, zkey):
    import artefact_writer as aw
    from oracle import layout
    from distributed_groth16_b200.groth16 import circom, verify
    s = k["s"]
    wit = [int.from_bytes(r.tobytes(), "little") for r in s["witness"]]
    proof, pub = circom.prove_zkey_wtns(net, zkey, aw.write_wtns(wit))
    z = net.fr_convert(net.to_device(s["witness"]), to_mont=True)
    assert proof == circom.prove_from_matrices(k["pk_toxic"], k["mats_toxic"], z)
    x = layout.fr_to_arr([wit[1]])
    assert verify.verify_proof(net, k["vk15"], x, proof)
    assert not verify.verify_proof(net, k["vk15"], layout.fr_to_arr([wit[1] + 1]), proof)
    return proof


@pytest.mark.gpu
def test_sha256_zkey_proves_like_the_toxic_waste_key_and_verifies(net, sha256_keys):
    from distributed_groth16_b200.groth16 import circom
    k = sha256_keys
    proof = _prove_and_check(net, k, k["zkey15"])
    z = net.fr_convert(net.to_device(k["s"]["witness"]), to_mont=True)
    assert circom.prove_from_matrices(k["pk15"], k["mats15"], z) == proof       # setup_from_ptau's device key


@pytest.mark.gpu
def test_sha256_power_16_ceremony_changes_only_h(net, sha256_keys):
    """A larger ceremony has the real tau^(2m-1) term in the doubled domain: H changes, A, B1, B2, C and IC do not, and
    the proof bytes of a satisfying witness do not either (that term multiplies a zero coefficient of A B - C)."""
    from distributed_groth16_b200 import formats
    k = sha256_keys
    z15, z16 = formats.read_zkey(k["zkey15"]), formats.read_zkey(k["zkey16"])
    for name in ("a_query", "b_g1_query", "b_g2_query", "l_query", "ic"):
        assert (getattr(z15, name) == getattr(z16, name)).all(), name
    assert not (z15.h_query == z16.h_query).all()
    assert _prove_and_check(net, k, k["zkey16"]) == _prove_and_check(net, k, k["zkey15"])


@pytest.mark.gpu
@pytest.mark.parametrize("power", [2, 3])
def test_tiny_circuit_zkey_equals_the_oracle_zkey_new(net, tmp_path, power):
    import ptau_writer as pw
    import zkey_oracle
    from distributed_groth16_b200.groth16 import circom
    r1cs = open(os.path.join(G, "circom2_multiplier2.r1cs"), "rb").read()
    secs = pw.sections_oracle(0x1234567890ABCDEF, 1111111111111111111, 2222222222222222223, power)
    path = pw.write_ptau(str(tmp_path / "tiny.ptau"), secs)
    assert circom.zkey_new(net, r1cs, path) == zkey_oracle.zkey_new(r1cs, pw.ptau_bytes(secs))
    assert pw.sections_gpu(net, 0x1234567890ABCDEF, 1111111111111111111, 2222222222222222223, power) == secs
