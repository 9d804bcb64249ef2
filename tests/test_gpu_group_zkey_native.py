"""The native prover on a group (b200zk_group_zkey_load / _prove, groth16.native_prover.GroupZKeyProver, `b200zk-prove --devices`)
against the one-GPU native prover (ZKeyProver), the Python group path (circom.groth16_prove_group: read_zkey, coo_to_csr and
the host reorder of GroupConstraintMatrices) and exact bytes.

Worlds as in test_gpu_group_zkey.py: world1, emu2 / emu4 / emu8 (`Group([0] * P)`: every index of the owner-major sort, the
slices' peer copies and the event ordering between contexts run at P ranks on one GPU; the NVLink transport and event
ordering across real devices are not covered there) and all (every GPU of the box; skips on a single-GPU box).  Every key is
loaded with the automatic table policy and without tables, and proves at (r, s) = (0, 0) and at random non-zero values."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from distributed_groth16_b200 import formats
from distributed_groth16_b200._native import ERR_ARG, ERR_LENGTH, ERR_SHORT_BUFFER, B200zkError
from distributed_groth16_b200.context import MpcNetError
from distributed_groth16_b200.groth16 import circom
from distributed_groth16_b200.groth16.native_prover import NO_TABLES, PROOF_JSON_MAX, GroupZKeyProver, ZKeyProver
from oracle import bn254 as o, layout

HERE = os.path.dirname(os.path.abspath(__file__))
G = os.path.join(HERE, "golden")
sys.path.insert(0, HERE)
import prove_dlog_oracle as po                  # noqa: E402
import test_gpu_group_zkey as gz                # noqa: E402
import test_gpu_zkey_native as zn               # noqa: E402
from test_gpu_qap_setup_exact import RS_RANDOM, host, witness  # noqa: E402

pytestmark = pytest.mark.gpu
TABLES = {"auto tables": 0, "no tables": NO_TABLES}
_memo = {}


def _cached(key, fn):
    if key not in _memo:
        _memo[key] = fn()
    return _memo[key]


def _m(v):
    return zn._m(v)


@pytest.fixture(scope="module")
def net():
    """This module's own GPU party, closed when the module ends (as test_gpu_prove_exact.py's): the one-GPU reference proofs at
    2^20 and 2^22 grow its slot workspaces to several GB, which on the session's Net would stay allocated for the rest of the
    run and shrink the table budget (60% of the free HBM) of every later key.  The handles cached here go with it."""
    import torch
    from distributed_groth16_b200 import Net
    n = Net(0)
    n.use_torch_stream(0)
    yield n
    torch.cuda.synchronize()
    for k in list(_memo):
        v = _memo.pop(k)
        if isinstance(v, ZKeyProver):
            v.free()
    n.close()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=["world1", "emu2", "emu4", "emu8", "all"])
def group(request):
    from distributed_groth16_b200.group import Group
    if request.param == "all":
        if gz._n_gpus() < 2:
            pytest.skip("needs >= 2 GPUs")
        devices = list(range(gz._n_gpus()))
    elif request.param == "world1":
        devices = [0]
    else:
        devices = [0] * int(request.param[3:])
    g = Group(devices)
    yield g
    g.close()


def _launches(grp) -> int:
    return gz._launches(grp)


def _check(group, net, name, zkey, wtns, want=None, rs_cases=((0, 0), RS_RANDOM)):
    """every table policy and (r, s): texts and bytes equal ZKeyProver's on one GPU and circom.groth16_prove_group's texts
    (and want[rs] when given); info() equals ZKeyProver's; no tables gives table_bytes 0"""
    one = _cached(("one", name), lambda: ZKeyProver(net, zkey, NO_TABLES))
    for tname, tw in TABLES.items():
        with GroupZKeyProver(group, zkey, table_window=tw) as gp:
            assert gp.info() == one.info(), name
            if tw == NO_TABLES:
                assert gp.table_bytes == 0
            for rs in rs_cases:
                r, s = (_m(rs[0]), _m(rs[1])) if isinstance(rs[0], int) else rs
                got = gp.prove(wtns, r, s)
                key = rs if isinstance(rs[0], int) else tuple(bytes(np.asarray(v, np.uint64)) for v in rs)
                assert got == _cached(("one", name, key), lambda: one.prove(wtns, r, s)), (name, tname, rs)
                py = _cached(("py", name, group.size(), key), lambda: circom.groth16_prove_group(group, zkey, wtns, r, s))
                assert got[:2] == py, (name, tname, rs)
                if want is not None:
                    assert got[2] == want[key], (name, tname, rs)


def _drop(name):
    one = _memo.pop(("one", name), None)
    if one is not None:
        one.free()
    for k in [k for k in _memo if k[1] == name]:
        del _memo[k]


# ---- the reference's proof and snarkjs's complex circuit ------------------------------------------------------------------------
def _sha256_key(net, cref):
    def f():
        from test_oracle_reference_proof import reference_sha256_instance
        pk, vk, _, _, _, _, (n_vars, n_inputs, m) = reference_sha256_instance(cref)
        d = np.load(os.path.join(G, "sha256_circuit.npz"))
        nc = int(d["dims"][2])
        to_mont = lambda v: host(net.fr_convert(net.to_device(np.ascontiguousarray(v, dtype=np.uint64)), to_mont=True))
        csr = [formats.coo_to_csr(d[k + "_rows"], d[k + "_cols"], to_mont(d[k + "_vals"]), nc) for k in "ab"]
        pts = dict(a=pk["a_query"], b1=pk["b_g1_query"], b2=pk["b_g2_query"], l=pk["l_query"], h=pk["h_query"],
                   vk1=np.stack([vk["alpha_g1"], vk["beta_g1"], vk["delta_g1"]]), vk2=np.stack([vk["beta_g2"], vk["delta_g2"]]))
        zkey = zn._zkey_of(net, pts, n_inputs - 1, m, nc, csr[0], csr[1], ic=vk["gamma_abc_g1"], gamma2=vk["gamma_g2"])
        return zkey, zn._wtns(d["witness"])
    return _cached("sha256 key", f)


def test_reference_sha256_key_gives_proof_bin(group, net, cref):
    zkey, wtns = _sha256_key(net, cref)
    gold = open(os.path.join(G, "sha256_proof.bin"), "rb").read()
    zero = np.zeros(4, np.uint64)
    _check(group, net, "sha256", zkey, wtns, want={(zero.tobytes(), zero.tobytes()): gold}, rs_cases=((zero, zero),))
    _check(group, net, "sha256", zkey, wtns, rs_cases=(RS_RANDOM,))


def test_complex_circuit_key_both_entries_verify(group, net):
    zkey, wtns, exp = zn._complex()
    vk = _cached("complex vk", lambda: circom.zkey_export_verificationkey(net, zkey))
    rs = {key: (layout.fr_to_arr([exp[key]["r"]])[0], layout.fr_to_arr([exp[key]["s"]])[0]) for key in ("r_s", "r0s0")}
    want = {tuple(bytes(np.asarray(v, np.uint64)) for v in rs[k]): bytes.fromhex(exp[k]["proof_hex"]) for k in rs}
    _check(group, net, "complex", zkey, wtns, want=want, rs_cases=tuple(rs.values()))
    with GroupZKeyProver(group, zkey) as gp:
        for key, (r, s) in rs.items():
            pj, uj, _ = gp.prove(wtns, r, s)
            assert circom.groth16_verify(net, vk, uj, pj), key


# ---- keys of known discrete logs ------------------------------------------------------------------------------------------------
# name -> (builder, worlds (None: every world)); the builders are test_gpu_group_zkey's (gz) and test_gpu_zkey_native's (zn)
#   2^6 sparse all public: at P = 8 GPUs 2..7 own only instance and padding rows
DLOG = {
    "2^10": ("gz", None), "2^15 odd": ("gz", None), "2^16 full n_inputs=1": ("gz", None), "2^6 sparse all public": ("gz", None),
    "2^18": ("zn", None), "2^20": ("zn", (2, 8)), "2^22": ("zn", (8,)), "n_public=0": ("zn", None),
}


def _dlog(net, cref, name):
    """-> zkey, wtns, exponents of the exact proof"""
    if DLOG[name][0] == "gz":
        zkey, wtns = gz._zkey_bytes(net, cref, name)
        return zkey, wtns, gz._dlog_instance(name)["e"]
    inst, wit = zn._instance(net, cref, name)
    return inst["zkey"], wit["wtns"], wit["e"]


@pytest.mark.parametrize("name", list(DLOG))
def test_known_log_keys(group, net, cref, name):
    worlds = DLOG[name][1]
    if worlds is not None and group.size() not in worlds:
        pytest.skip("%s runs at P in %s" % (name, worlds))
    zkey, wtns, e = _dlog(net, cref, name)
    try:
        _check(group, net, name, zkey, wtns, want={rs: po.proof_bytes(e, *rs) for rs in ((0, 0), RS_RANDOM)})
    finally:
        _drop(name)
        if name in ("2^20", "2^22") and group.size() == max(DLOG[name][1]):   # GBs of host memory: the last world to use it
            for k in [k for k in zn._memo if name in k]:
                del zn._memo[k]


def test_shuffled_records_with_public_rows_interleaved(group, net, cref):
    inst, wit = zn._instance(net, cref, "2^16")
    log_m, nc, n_public, _, _ = zn.DLOG["2^16"]

    def f():
        pts = {k: v if isinstance(v, np.ndarray) else host(v) for k, v in inst["spec"].device_points(net).items()}
        n_rec = int(inst["a_csr"][0][-1]) + int(inst["b_csr"][0][-1]) + n_public + 1
        order = np.random.default_rng(5).permutation(n_rec)
        return zn._zkey_of(net, pts, n_public, 1 << log_m, nc, inst["a_csr"], inst["b_csr"], order=order)
    zkey = _cached("shuffled", f)
    _check(group, net, "shuffled", zkey, wit["wtns"], want={rs: po.proof_bytes(wit["e"], *rs) for rs in ((0, 0), RS_RANDOM)})


def test_zkey_without_coefficient_records(group, net, cref):
    def f():
        spec = po.KeySpec(4, 20, 3, 0x5151 << 8)
        pts = {k: v if isinstance(v, np.ndarray) else host(v) for k, v in spec.device_points(net).items()}
        empty = (np.zeros(1, np.uint32), np.zeros(0, np.uint32), np.zeros((0, 4), np.uint64))
        zk = formats.read_zkey(zn._zkey_of(net, pts, 2, 4, 0, empty, empty))
        zkey = formats.write_zkey(formats.ZKey(**{**zk.__dict__, "coef_matrix": zk.coef_matrix[:0], "coef_row": zk.coef_row[:0],
                                                  "coef_col": zk.coef_col[:0], "coef_val_r2": zk.coef_val_r2[:0]}))
        return zkey, zn._wtns(zn._canonical(net, witness(np.random.default_rng(3), 20, "random", 3)))
    zkey, wtns = _cached("no records", f)
    if group.size() > 2:            # domain 4: cols = 2
        with pytest.raises(B200zkError, match="domain too small"):
            GroupZKeyProver(group, zkey)
        return
    _check(group, net, "no records", zkey, wtns)
    with GroupZKeyProver(group, zkey) as gp:
        assert gp.info()["num_constraints"] == 0


@pytest.mark.parametrize("name", list(zn.TINY))
def test_tiny_domains_agree_with_the_python_group_path(group, net, cref, name):
    zkey, wtns, e = _cached(("tiny", name), lambda: zn._tiny(net, cref, name))
    for rs in ((0, 0), RS_RANDOM):
        r, s = _m(rs[0]), _m(rs[1])
        try:
            py = circom.groth16_prove_group(group, zkey, wtns, r, s)
        except B200zkError as err:
            py = err
        before = _launches(group)
        try:
            with GroupZKeyProver(group, zkey) as gp:
                got = gp.prove(wtns, r, s)
        except B200zkError as err:
            assert isinstance(py, B200zkError), (name, rs, err.message)
            assert (err.code, err.message) == (py.code, py.message), (name, rs)
            if "domain too small for this many GPUs" in err.message:
                assert err.code == ERR_ARG and _launches(group) == before
            continue
        assert not isinstance(py, B200zkError), (name, rs, py)
        assert got[:2] == py and got[2] == po.proof_bytes(e, *rs), (name, rs)


# ---- refusals -------------------------------------------------------------------------------------------------------------------
def _refusal(fn):
    with pytest.raises((B200zkError, MpcNetError)) as e:
        fn()
    return e.value


def test_refusals_match_the_one_gpu_prover(group, net):
    zkey, wtns, _ = zn._complex()
    zk = formats.read_zkey(zkey)
    P = group.size()

    def same(one_fn, grp_fn, host_detectable):
        one = _refusal(one_fn)
        before = _launches(group)
        got = _refusal(grp_fn)
        assert type(got) is type(one)
        assert getattr(got, "code", ERR_LENGTH) == getattr(one, "code", ERR_LENGTH), (got, one)
        assert got.message.endswith(one.message), (got.message, one.message)
        if host_detectable:
            assert _launches(group) == before, one.message

    bad = [b"zkez" + zkey[4:],
           zn._edit_section(zkey, 5, lambda p: p).replace(struct_pack("<IQ", 5, zk.n_vars * 64), struct_pack("<IQ", 11, zk.n_vars * 64), 1),
           zn._edit_section(zkey, 1, lambda p: struct_pack("<I", 2)),
           zn._edit_section(zkey, 2, lambda p: p[:4] + (formats.FQ_MODULUS + 2).to_bytes(32, "little") + p[36:]),
           zn._edit_section(zkey, 2, lambda p: p[:80] + struct_pack("<I", 12) + p[84:]),
           zn._edit_section(zkey, 9, lambda p: p[:-64]),
           zkey[:len(zkey) - 100]]
    for buf in bad:
        same(lambda: ZKeyProver(net, buf), lambda: GroupZKeyProver(group, buf), True)
    rec = lambda k, field, v: (lambda p: p[:4 + 44 * k + 4 * field] + struct_pack("<I", v) + p[8 + 44 * k + 4 * field:])
    two_bad = zn._edit_section(zn._edit_section(zkey, 4, rec(7, 0, 2)), 4, rec(3, 2, zk.n_vars))
    same(lambda: ZKeyProver(net, two_bad), lambda: GroupZKeyProver(group, two_bad), False)

    w = formats.read_wtns(wtns)
    big = w.copy()
    for i in (9, 4):
        big[i] = [(o.R >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(4)]
    with ZKeyProver(net, zkey) as zp, GroupZKeyProver(group, zkey) as gp:
        for wb, host_detectable in ((zn._wtns(w[:-1]), True), (b"wtnx" + wtns[4:], True), (wtns[:-8], True), (zn._wtns(big), False)):
            same(lambda: zp.prove(wb), lambda: gp.prove(wb), host_detectable)

        # short buffers: refused before any launch with both sizes needed, then proved at exactly those sizes
        lib = group._lib
        proof = (ctypes.c_uint8 * 128)()
        zero = np.zeros(4, np.uint64)
        want = zp.prove(wtns, zero, zero)
        for plen0, ulen0 in ((PROOF_JSON_MAX - 1, 1000), (PROOF_JSON_MAX, len(want[1])), (10, 0)):
            plen, ulen = ctypes.c_size_t(plen0), ctypes.c_size_t(ulen0)
            pbuf, ubuf = ctypes.create_string_buffer(max(plen0, 1)), ctypes.create_string_buffer(max(ulen0, 1))
            before = _launches(group)
            rc = lib.b200zk_group_zkey_prove(group._h, gp._h, wtns, len(wtns), zero.ctypes.data, zero.ctypes.data, proof, pbuf,
                                             ctypes.byref(plen), ubuf, ctypes.byref(ulen))
            assert rc == ERR_SHORT_BUFFER and _launches(group) == before
            assert (plen.value, ulen.value) == (PROOF_JSON_MAX, len(want[1]) + 1)
            pbuf, ubuf = ctypes.create_string_buffer(plen.value), ctypes.create_string_buffer(ulen.value)
            assert lib.b200zk_group_zkey_prove(group._h, gp._h, wtns, len(wtns), zero.ctypes.data, zero.ctypes.data, proof, pbuf,
                                               ctypes.byref(plen), ubuf, ctypes.byref(ulen)) == 0
            assert (pbuf.raw[:plen.value].decode(), ubuf.raw[:ulen.value].decode(), bytes(proof)) == want

        # a key loaded on another group
        from distributed_groth16_b200.group import Group
        other = Group([0] * (2 if P != 2 else 1))
        try:
            with GroupZKeyProver(other, zkey) as og:
                before = _launches(group)
                err = _refusal(lambda: group.check(lib.b200zk_group_zkey_prove(group._h, og._h, wtns, len(wtns), None, None, proof,
                                                                              None, None, None, None)))
                assert err.code == ERR_ARG and "different group" in err.message
                assert _launches(group) == before
        finally:
            other.close()
        assert gp.prove(wtns, zero, zero) == want                    # the group still proves after every refusal


def struct_pack(fmt, *v):
    import struct
    return struct.pack(fmt, *v)


# ---- reuse, memory, randomness --------------------------------------------------------------------------------------------------
def test_reuse_two_handles_and_memory_returns(group, net, cref):
    import gc
    import torch
    inst, _ = zn._instance(net, cref, "2^16")
    wits = [zn._instance(net, cref, "2^16", z_seed=0x33 + k)[1] for k in range(3)]
    zkey_c, wtns_c, _ = zn._complex()
    want_c = circom.groth16_prove(net, zkey_c, wtns_c, _m(0), _m(0))
    rs = tuple(_m(v) for v in RS_RANDOM)

    def rounds(a, b):
        """the witnesses on one handle, interleaved with the other handle and with the group's d_msm / d_fft"""
        for k, wit in enumerate(wits):
            assert a.prove(wit["wtns"], *rs)[2] == po.proof_bytes(wit["e"], *RS_RANDOM), k
            bases, scalars = cref.g1_generate(0x2E10 + k, 300), cref.fr_generate(0x2E10 + k, 300)
            got = group.d_msm(bases, scalars)
            exp, inf = cref.msm_g1(bases, scalars)
            assert got.infinity == inf and (got.limbs == exp).all(), k
            assert b.prove(wtns_c, _m(0), _m(0))[:2] == want_c, k
            x = cref.fr_generate(0x2E20 + k, 1 << 10)
            assert (group.d_ifft(group.d_fft(x)) == x).all(), k

    # one pass on the very same inputs first: the contexts' grow-only workspaces reach their size for these calls
    with GroupZKeyProver(group, inst["zkey"]) as a, GroupZKeyProver(group, zkey_c) as b:
        rounds(a, b)
    gc.collect()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    a, b = GroupZKeyProver(group, inst["zkey"]), GroupZKeyProver(group, zkey_c)
    try:
        rounds(a, b)
    finally:
        a.free()
        b.free()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


def test_random_r_s_are_fresh_and_verify(group, net):
    zkey, wtns, _ = zn._complex()
    vk = _cached("complex vk", lambda: circom.zkey_export_verificationkey(net, zkey))
    with GroupZKeyProver(group, zkey) as gp:
        p1, u1, b1 = gp.prove(wtns)
        p2, u2, b2 = gp.prove(wtns)
    assert b1 != b2 and p1 != p2 and u1 == u2
    assert circom.groth16_verify(net, vk, u1, p1) and circom.groth16_verify(net, vk, u2, p2)


# ---- the command ----------------------------------------------------------------------------------------------------------------
def test_command_devices(group, net, tmp_path):
    from distributed_groth16_b200 import build
    zkey, wtns, _ = zn._complex()
    (tmp_path / "c.zkey").write_bytes(zkey)
    (tmp_path / "w.wtns").write_bytes(wtns)
    devices = ",".join(str(d) for d in (group.devices if group.size() > 1 else [0, 0, 0, 0]))
    run = lambda *a: subprocess.run([build.PROVE_EXE, "--devices", devices] + [str(tmp_path / x) for x in a], capture_output=True,
                                    text=True)
    r = run("c.zkey", "w.wtns", "proof.json", "public.json")
    assert r.returncode == 0, r.stderr
    proof, public = (tmp_path / "proof.json").read_text(), (tmp_path / "public.json").read_text()
    with ZKeyProver(net, zkey, NO_TABLES) as zp:
        assert public == zp.prove(wtns)[1]
    assert circom.groth16_verify(net, _cached("complex vk", lambda: circom.zkey_export_verificationkey(net, zkey)), public, proof)
    (tmp_path / "bad.wtns").write_bytes(b"wtnx" + wtns[4:])
    r = run("c.zkey", "bad.wtns", "p2.json", "u2.json")
    assert r.returncode == 1 and "bad magic" in r.stderr, r.stderr
    assert sorted(os.listdir(tmp_path)) == ["bad.wtns", "c.zkey", "proof.json", "public.json", "w.wtns"]
