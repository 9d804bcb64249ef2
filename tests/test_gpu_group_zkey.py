"""snarkjs `groth16 prove` on a group (b200zk_group_r1cs_upload / b200zk_group_groth16_prove_r1cs_dev, group.load_zkey,
circom.prove_zkey_wtns_group / groth16_prove_group): the constraint matrices sharded by QAP output slot, each GPU computing
its column-layout slice of a, b, c from the witness on device 0.

Worlds as in test_gpu_group.py: world1 (one context), emu2 / emu4 / emu8 (`Group([0] * P)`: every index of the sharding, the
peer copies of z and the event ordering between contexts run at P ranks on one GPU; the NVLink transport and event ordering
across real devices are not covered there) and all (every GPU of the box; skips on a single-GPU box).

Expected bytes: the reference's own sha256 proof, snarkjs's complex-circuit proofs, and for keys of known discrete logs
(prove_dlog_oracle.KeySpec) the exponents of the CPU twin's QAP and h; every case also equals the one-GPU prover."""
import ctypes
import os
import sys

import numpy as np
import pytest

from distributed_groth16_b200._native import ERR_ARG, ERR_DOMAIN, B200zkError, c_vp
from oracle import bn254 as o, layout

HERE = os.path.dirname(os.path.abspath(__file__))
G = os.path.join(HERE, "golden")
sys.path.insert(0, HERE)
import artefact_writer as aw                    # noqa: E402
import prove_dlog_oracle as po                  # noqa: E402
from test_gpu_qap_setup_exact import RS_RANDOM, coo, host, make_csr, mont, witness  # noqa: E402

pytestmark = pytest.mark.gpu
_memo = {}


def _cached(key, fn):
    if key not in _memo:
        _memo[key] = fn()
    return _memo[key]


def _n_gpus():
    import torch
    n, w = torch.cuda.device_count(), 1
    while w * 2 <= min(n, 8):
        w *= 2
    return w


@pytest.fixture(scope="module", params=["world1", "emu2", "emu4", "emu8", "all"])
def group(request):
    from distributed_groth16_b200.group import Group
    if request.param == "all":
        if _n_gpus() < 2:
            pytest.skip("needs >= 2 GPUs")
        devices = list(range(_n_gpus()))
    elif request.param == "world1":
        devices = [0]
    else:
        devices = [0] * int(request.param[3:])
    g = Group(devices)
    yield g
    g.close()


def _launches(grp) -> int:
    lib = grp._lib
    return sum(int(lib.b200zk_launch_count(lib.b200zk_group_ctx(grp._h, r))) for r in range(grp.size()))


def _raises_before_launch(grp, fn, code, text):
    before = _launches(grp)
    with pytest.raises(B200zkError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)
    assert text in e.value.message, e.value.message
    assert _launches(grp) == before


def _canonical(z):
    return layout.arr_to_fr(np.asarray(z, dtype=np.uint64).reshape(-1, 4))


# ---- the reference's own proof ------------------------------------------------------------------------------------------------
def _sha256():
    from oracle import cref
    from test_oracle_reference_proof import reference_sha256_instance
    return _cached("sha256", lambda: reference_sha256_instance(cref))


def _prove_sha256(grp):
    from distributed_groth16_b200.group import GroupConstraintMatrices, GroupProvingKey
    pk, vk, z, _, _, _, (n_vars, n_inputs, m) = _sha256()
    d = np.load(os.path.join(G, "sha256_circuit.npz"))
    nc = int(d["dims"][2])
    gpk = GroupProvingKey(grp, pk["a_query"], pk["b_g1_query"], pk["b_g2_query"], pk["l_query"], pk["h_query"], n_inputs,
                          vk["alpha_g1"], vk["beta_g1"], vk["delta_g1"], vk["beta_g2"], vk["delta_g2"])
    mats = GroupConstraintMatrices(grp, n_inputs, nc, (d["a_rows"], d["a_cols"], d["a_vals"]), (d["b_rows"], d["b_cols"], d["b_vals"]),
                                   values_montgomery_depth=-1, log_m=m.bit_length() - 1, n_vars=n_vars)
    try:
        return gpk.create_proof_r1cs(mats, grp.witness_to_device(d["witness"])), gpk.table_bytes
    finally:
        mats.free()
        gpk.free()


def test_reference_sha256_proof_from_its_matrices_and_witness(group, monkeypatch):
    gold = open(os.path.join(G, "sha256_proof.bin"), "rb").read()
    got, table_bytes = _prove_sha256(group)
    assert table_bytes > 0
    assert got == gold
    from distributed_groth16_b200.group import Group
    monkeypatch.setenv("B200ZK_PK_TABLES", "0")        # read by every key upload: the generic MSM on every shard
    fresh = Group(group.devices)
    try:
        got, table_bytes = _prove_sha256(fresh)
        assert table_bytes == 0
        assert got == gold
    finally:
        fresh.close()


# ---- a snarkjs-made zkey -------------------------------------------------------------------------------------------------------
def test_complex_circuit_zkey_texts_equal_the_one_gpu_prover_and_verify(group, net):
    import json
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import circom
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    exp = json.load(open(os.path.join(G, "complex_circuit_proof.json")))
    zkey, wtns = aw.write_zkey(d), aw.write_wtns(aw.f1_witness(int(d["dims"][0])))
    vk_json = _cached("complex_vk", lambda: circom.zkey_export_verificationkey(net, zkey))
    for key in ("r_s", "r0s0"):
        r, s = layout.fr_to_arr([exp[key]["r"]])[0], layout.fr_to_arr([exp[key]["s"]])[0]
        proof, _ = circom.prove_zkey_wtns_group(group, zkey, wtns, r=r, s=s)
        assert proof.hex() == exp[key]["proof_hex"], key
        texts = circom.groth16_prove_group(group, zkey, wtns, r=r, s=s)
        assert texts == _cached(("complex", key), lambda: circom.groth16_prove(net, zkey, wtns, r=r, s=s)), key
        A, B, C = o.proof_decompress(proof)
        assert texts[0] == formats.write_proof_json(formats.SnarkjsProof(A, B, C))
        assert circom.groth16_verify(net, vk_json, texts[1], texts[0]), key


# ---- exact proofs at size, by discrete logs -------------------------------------------------------------------------------------
# name -> (log_m, nc, n_inputs, n_vars, witness kind, worlds (None: every world), through zkey bytes)
#   2^15: odd log m (rows = 2 cols), a row of 2^16 terms (make_csr's long row) and empty rows
#   2^16 full: nc + n_inputs = m exactly, n_inputs = 1
#   2^6 sparse: 2 constraints and 31 inputs, all public: at P = 8 (one column per GPU) GPU g holds global rows g, 8 + g, ...,
#         so GPUs 2..7 own only instance and padding rows
#   2^20: the thread kernel in each shard at P = 2 (2^19 slots), the warp kernel at P = 8 (2^17 slots).  Written straight into
#         GroupConstraintMatrices: the Python zkey writer would take minutes at this size, and the smaller cases cover the
#         reader.
DLOG_CASES = {
    "2^10": (10, 1000, 3, 700, "random", None, True),
    "2^15 odd": (15, 30000, 2, 20000, "0/1", None, True),
    "2^16 full n_inputs=1": (16, (1 << 16) - 1, 1, 40000, "random", None, True),
    "2^6 sparse all public": (6, 2, 31, 31, "random", None, True),
    "2^20 P=2": (20, 1000000, 3, 1 << 19, "0/1", (2,), False),
    "2^20 P=8": (20, 1000000, 3, 1 << 19, "0/1", (8,), False),
}


def _dlog_instance(name):
    from oracle import cref
    log_m, nc, ni, n_vars, kind, _, _ = DLOG_CASES[name]
    m = 1 << log_m

    def f():
        seed = 0x62A0 + log_m * 7 + nc % 1000
        rng = np.random.default_rng(seed)
        a_csr = make_csr(rng, nc, n_vars, long_row=nc >= 1024)
        b_csr = make_csr(rng, nc, n_vars, long_row=False, empty_rows=[nc - 1] if nc > 1 else [])
        z = witness(rng, n_vars, kind, seed)
        h = po.expected_h(cref, *cref.qap(a_csr, b_csr, z, nc, ni, m))
        spec = po.KeySpec(m, n_vars, ni, seed << 8)
        return dict(a_csr=a_csr, b_csr=b_csr, z=z, spec=spec, e=po.exponents(spec, z, h))
    return _cached(("dlog",) + DLOG_CASES[name][:5], f)


def _key_arrays(net, spec):
    pts = spec.device_points(net)
    return {k: v if isinstance(v, np.ndarray) else host(v) for k, v in pts.items()}


def _zkey_bytes(net, cref, name):
    def f():
        I = _dlog_instance(name)
        log_m, nc, ni, n_vars = DLOG_CASES[name][:4]
        pts = _key_arrays(net, I["spec"])
        d = dict(dims=np.array([n_vars, ni - 1, 1 << log_m, nc]), vk_g1=pts["vk1"], ic=cref.g1_generate(0x1C, ni),
                 vk_g2=np.concatenate([pts["vk2"], layout.g2_to_arr([o.G2_GEN])]), a_query=pts["a"], b_g1_query=pts["b1"],
                 b_g2_query=pts["b2"], l_query=pts["l"], h_query=pts["h"])
        for k, csr in (("a", I["a_csr"]), ("b", I["b_csr"])):
            d[k + "_rows"], d[k + "_cols"], d[k + "_vals"] = coo(csr)
        return aw.write_zkey(d), aw.write_wtns(_canonical(I["z"]))
    return _cached(("zkey", name), f)


def _one_gpu(net, cref, name, rs):
    from distributed_groth16_b200.groth16 import circom
    from distributed_groth16_b200.groth16.proving_key import ProvingKey
    from distributed_groth16_b200.groth16.qap import ConstraintMatrices

    def f():
        I = _dlog_instance(name)
        r, s = mont([rs[0]])[0], mont([rs[1]])[0]
        if DLOG_CASES[name][6]:
            return circom.prove_zkey_wtns(net, *_zkey_bytes(net, cref, name), r, s)[0]
        import torch
        pts = I["spec"].device_points(net)
        pk = ProvingKey.from_device(net, pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], I["spec"].n_inputs, po.vk_array(pts))
        mats = ConstraintMatrices(net, I["spec"].n_inputs, DLOG_CASES[name][1], coo(I["a_csr"]), coo(I["b_csr"]), values_montgomery_depth=0)
        try:
            return circom.prove_from_matrices(pk, mats, net.to_device(I["z"]), r, s)
        finally:
            pk.free()
            del pts, mats
            torch.cuda.empty_cache()
    return _cached(("one",) + DLOG_CASES[name][:5] + (rs,), f)


def _group_proofs(group, net, cref, name):
    from distributed_groth16_b200.group import GroupConstraintMatrices, GroupProvingKey
    from distributed_groth16_b200.groth16 import circom
    I = _dlog_instance(name)
    out = {}
    if DLOG_CASES[name][6]:
        zkey, wtns = _zkey_bytes(net, cref, name)
        for rs in ((0, 0), RS_RANDOM):
            out[rs] = circom.prove_zkey_wtns_group(group, zkey, wtns, mont([rs[0]])[0], mont([rs[1]])[0])[0]
        return out
    import torch
    log_m, nc, ni, n_vars = DLOG_CASES[name][:4]
    pts = _key_arrays(net, I["spec"])
    gpk = GroupProvingKey(group, pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], ni, pts["vk1"][0], pts["vk1"][1], pts["vk1"][2],
                          pts["vk2"][0], pts["vk2"][1])
    mats = GroupConstraintMatrices(group, ni, nc, coo(I["a_csr"]), coo(I["b_csr"]), values_montgomery_depth=0, log_m=log_m, n_vars=n_vars)
    try:
        z_dev = torch.from_numpy(I["z"].view(np.int64)).to(torch.device("cuda", group.devices[0]))
        for rs in ((0, 0), RS_RANDOM):
            out[rs] = gpk.create_proof_r1cs(mats, z_dev, mont([rs[0]])[0], mont([rs[1]])[0])
    finally:
        mats.free()
        gpk.free()
        torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("name", list(DLOG_CASES))
def test_exact_proofs_by_discrete_logs(group, net, cref, name):
    worlds = DLOG_CASES[name][5]
    if worlds is not None and group.size() not in worlds:
        pytest.skip("%s runs at P in %s" % (name, worlds))
    e = _dlog_instance(name)["e"]
    for rs, got in _group_proofs(group, net, cref, name).items():
        assert got == po.proof_bytes(e, *rs), (name, rs)
        assert got == _one_gpu(net, cref, name, rs), (name, rs)


# ---- one key and matrices, several witnesses, other group calls in between -----------------------------------------------------
def test_reuse_across_witnesses_and_other_group_calls(group, net, cref):
    import torch
    from distributed_groth16_b200.group import load_zkey
    name = "2^10"
    I = _dlog_instance(name)
    log_m, nc, ni, n_vars = DLOG_CASES[name][:4]
    m = 1 << log_m
    gpk, mats, zk = load_zkey(group, _zkey_bytes(net, cref, name)[0])
    try:
        for k, kind in enumerate(("random", "0/1", "random")):
            rng = np.random.default_rng(0x2E05 + k)
            z = witness(rng, n_vars, kind, 0x2E05 + k)
            a, b, c = cref.qap(I["a_csr"], I["b_csr"], z, nc, ni, m)
            want = po.proof_bytes(po.exponents(I["spec"], z, po.expected_h(cref, a, b, c)), *RS_RANDOM)
            r, s = mont([RS_RANDOM[0]])[0], mont([RS_RANDOM[1]])[0]
            z_dev = torch.from_numpy(z.view(np.int64)).to(torch.device("cuda", group.devices[0]))
            assert gpk.create_proof_r1cs(mats, z_dev, r, s) == want, k
            bases, scalars = cref.g1_generate(0x2E10 + k, 300), cref.fr_generate(0x2E10 + k, 300)
            got = group.d_msm(bases, scalars)
            exp, inf = cref.msm_g1(bases, scalars)
            assert got.infinity == inf and (got.limbs == exp).all(), k
            assert gpk.create_proof(z, a, b, c, r, s) == want, k          # the host-vector entry on the same key
            assert (group.h(a, b, c) == po.expected_h(cref, a, b, c)).all(), k
    finally:
        mats.free()
        gpk.free()


# ---- refusals -------------------------------------------------------------------------------------------------------------------
def _upload(grp, a_csr, b_csr, nc, ni, n_vars, log_m):
    lib = grp._lib
    (ap, ac, av), (bp, bc, bv) = a_csr, b_csr
    h = c_vp()
    p = lambda x: np.ascontiguousarray(x).ctypes.data
    grp.check(lib.b200zk_group_r1cs_upload(grp._h, p(ap), p(ac), p(av), p(bp), p(bc), p(bv), nc, ni, n_vars, log_m, 0, ctypes.byref(h)))
    return h


def test_refusals_leave_a_working_group(group, net, cref):
    import torch
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.group import Group, GroupConstraintMatrices, load_zkey
    from distributed_groth16_b200.groth16 import circom
    name = "2^10"
    I = _dlog_instance(name)
    log_m, nc, ni, n_vars = DLOG_CASES[name][:4]
    P = group.size()
    a_csr, b_csr = I["a_csr"], I["b_csr"]
    bad_col = b_csr[1].copy()
    bad_col[5] = n_vars
    _raises_before_launch(group, lambda: _upload(group, a_csr, (b_csr[0], bad_col, b_csr[2]), nc, ni, n_vars, log_m), ERR_ARG,
                          "matrix B: term 5")
    bad_ptr = a_csr[0].copy()
    bad_ptr[7] = bad_ptr[6] - 1 if bad_ptr[6] else bad_ptr[8] + 1
    _raises_before_launch(group, lambda: _upload(group, (bad_ptr, a_csr[1], a_csr[2]), b_csr, nc, ni, n_vars, log_m), ERR_ARG,
                          "matrix A: row_ptr decreases")
    _raises_before_launch(group, lambda: _upload(group, a_csr, b_csr, nc, 30, n_vars, log_m), ERR_DOMAIN,
                          "num_constraints + num_inputs exceeds the domain size")
    empty = (np.zeros(1, dtype=np.uint32), np.zeros(1, dtype=np.uint32), np.zeros((1, 4), dtype=np.uint64))
    _raises_before_launch(group, lambda: _upload(group, empty, empty, 0, 1, 1, 28), ERR_DOMAIN, "log_m > 27")
    if P > 1:
        small = 2 * (P.bit_length() - 1) - 1                               # cols = P / 2
        _raises_before_launch(group, lambda: _upload(group, empty, empty, 0, 1, 1, small), ERR_ARG, "domain too small")

    zkey, wtns = _zkey_bytes(net, cref, name)
    gpk, mats, _ = load_zkey(group, zkey)
    other = Group([0] * (2 if P != 2 else 4))
    try:
        z_dev = torch.from_numpy(I["z"].view(np.int64)).to(torch.device("cuda", group.devices[0]))
        o_pk, o_mats, _ = load_zkey(other, zkey)
        try:
            out = (ctypes.c_uint8 * 128)()
            zero = np.zeros(4, dtype=np.uint64)
            prove = lambda pk_h, mats_h: group.check(group._lib.b200zk_group_groth16_prove_r1cs_dev(
                group._h, pk_h, mats_h, c_vp(z_dev.data_ptr()), zero.ctypes.data, zero.ctypes.data, out))
            _raises_before_launch(group, lambda: prove(o_pk._h, mats._h), ERR_ARG, "proving key was uploaded to a different group")
            _raises_before_launch(group, lambda: prove(gpk._h, o_mats._h), ERR_ARG,
                                  "constraint matrices were uploaded to a different group")
            assert bytes(out) == bytes(128)
        finally:
            o_mats.free()
            o_pk.free()
        wrong_m = GroupConstraintMatrices(group, ni, nc, coo(a_csr), coo(b_csr), 0, log_m + 1, n_vars)
        wrong_ni = GroupConstraintMatrices(group, ni + 1, nc, coo(a_csr), coo(b_csr), 0, log_m, n_vars)
        try:
            _raises_before_launch(group, lambda: gpk.create_proof_r1cs(wrong_m, z_dev), ERR_DOMAIN, "domain")
            _raises_before_launch(group, lambda: gpk.create_proof_r1cs(wrong_ni, z_dev), ERR_ARG, "inputs")
        finally:
            wrong_m.free()
            wrong_ni.free()
        with pytest.raises(formats.FormatError):
            circom.prove_zkey_wtns_group(group, zkey, aw.write_wtns(_canonical(I["z"])[:-1]))
        assert gpk.create_proof_r1cs(mats, z_dev) == po.proof_bytes(I["e"], 0, 0)     # the group still proves
    finally:
        other.close()
        mats.free()
        gpk.free()
