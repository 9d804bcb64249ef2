"""The native prover (b200zk_zkey_load / b200zk_zkey_prove, groth16.native_prover.ZKeyProver, the b200zk-prove command) against
the Python path (circom.groth16_prove: read_zkey, coo_to_csr, ConstraintMatrices, proof_to_json) and exact bytes.

Keys: the reference's sha256 key (its proof must be proof.bin), snarkjs's complex-circuit key, and keys of known discrete
logs (prove_dlog_oracle.KeySpec) written as zkeys by formats.write_zkey at 2^16 (one warp per row in the QAP) up to 2^22 (one
thread per row), whose proofs must be prove_dlog_oracle.expected_proof.  Every key is loaded with the automatic table policy
and without tables, and proves at (r, s) = (0, 0) and at random non-zero values."""
import ctypes
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from distributed_groth16_b200 import formats
from distributed_groth16_b200._native import ERR_ARG, ERR_LENGTH, ERR_SHORT_BUFFER, B200zkError
from distributed_groth16_b200.context import MpcNetError
from distributed_groth16_b200.groth16 import circom
from distributed_groth16_b200.groth16.native_prover import NO_TABLES, PROOF_JSON_MAX, ZKeyProver
from oracle import bn254 as o, layout

HERE = os.path.dirname(os.path.abspath(__file__))
G = os.path.join(HERE, "golden")
sys.path.insert(0, HERE)
import artefact_writer as aw                    # noqa: E402
import prove_dlog_oracle as po                  # noqa: E402
from test_gpu_qap_setup_exact import RS_RANDOM, coo, host, make_csr, mont, witness  # noqa: E402

pytestmark = pytest.mark.gpu
R = o.R
TABLES = {"auto tables": 0, "no tables": NO_TABLES}
_memo = {}


def _cached(key, fn):
    if key not in _memo:
        _memo[key] = fn()
    return _memo[key]


def _m(v):
    return mont([v])[0]


def _wtns(canon: np.ndarray) -> bytes:
    """a .wtns of canonical (n, 4) limbs"""
    w = np.ascontiguousarray(canon, dtype="<u8").reshape(-1, 4)
    s1 = struct.pack("<I", 32) + R.to_bytes(32, "little") + struct.pack("<I", w.shape[0])
    return aw.container(b"wtns", [(1, s1), (2, w.tobytes())], version=2)


def _times_r(net, vals_mont: np.ndarray) -> np.ndarray:
    """Montgomery values v R -> v R^2, the zkey's coefficient words (on the device)"""
    if vals_mont.shape[0] == 0:
        return np.zeros((0, 4), dtype=np.uint64)
    return host(net.fr_convert(net.to_device(np.ascontiguousarray(vals_mont, dtype=np.uint64)), to_mont=True))


def _canonical(net, z_mont: np.ndarray) -> np.ndarray:
    return host(net.fr_convert(net.to_device(np.ascontiguousarray(z_mont, dtype=np.uint64)), to_mont=False))


def _zkey_of(net, pts: dict, n_public: int, m: int, nc: int, a_csr, b_csr, ic=None, gamma2=None, order=None) -> bytes:
    """a Groth16 zkey in snarkjs's record order (order: a permutation of the records instead)"""
    ca, cb = coo(a_csr), coo(b_csr)
    mi, ci, si, vi = formats.zkey_coefficients(n_public, nc, (ca[0], ca[1], _times_r(net, ca[2])), (cb[0], cb[1], _times_r(net, cb[2])))
    if order is not None:
        mi, ci, si, vi = mi[order], ci[order], si[order], vi[order]
    vk1, vk2 = np.asarray(pts["vk1"]).reshape(3, 8), np.asarray(pts["vk2"]).reshape(2, 16)
    n_vars = pts["a"].shape[0]
    zk = formats.ZKey(n_vars=n_vars, n_public=n_public, domain_size=m, alpha_g1=vk1[0], beta_g1=vk1[1], beta_g2=vk2[0],
                      gamma_g2=layout.g2_to_arr([o.G2_GEN])[0] if gamma2 is None else gamma2, delta_g1=vk1[2], delta_g2=vk2[1],
                      ic=layout.g1_to_arr([o.G1_GEN] * (n_public + 1)) if ic is None else ic, a_query=pts["a"], b_g1_query=pts["b1"],
                      b_g2_query=pts["b2"], l_query=pts["l"], h_query=pts["h"], coef_matrix=mi, coef_row=ci, coef_col=si,
                      coef_val_r2=vi)
    return formats.write_zkey(zk)


# ---- known-log instances ----------------------------------------------------------------------------------------------------
# name -> (log_m, nc, n_public, n_vars, witness kind)
DLOG = {
    "2^16": (16, 40000, 2, 30000, "random"),
    "2^18": (18, 200000, 3, 150000, "0/1"),
    "2^20": (20, 1000000, 3, 1 << 19, "0/1"),
    "2^22": (22, 4000000, 3, 1 << 21, "0/1"),
    "n_public=0": (8, 200, 0, 150, "random"),
    "all public": (6, 2, 30, 31, "random"),
}


def _instance(net, cref, name, z_seed=None):
    log_m, nc, n_public, n_vars, kind = DLOG[name]
    m = 1 << log_m

    def f():
        seed = 0x7A00 + log_m * 11 + n_public
        rng = np.random.default_rng(seed)
        a_csr = make_csr(rng, nc, n_vars, long_row=nc >= 1024)
        b_csr = make_csr(rng, nc, n_vars, long_row=False, empty_rows=[nc - 1] if nc > 1 else [])
        spec = po.KeySpec(m, n_vars, n_public + 1, seed << 8)
        pts = {k: v if isinstance(v, np.ndarray) else host(v) for k, v in spec.device_points(net).items()}
        return dict(a_csr=a_csr, b_csr=b_csr, spec=spec, zkey=_zkey_of(net, pts, n_public, m, nc, a_csr, b_csr))
    inst = _cached(("inst", name), f)

    def g():
        zs = 0x9100 + log_m if z_seed is None else z_seed
        z = witness(np.random.default_rng(zs), n_vars, kind, zs)
        h = po.expected_h(cref, *cref.qap(inst["a_csr"], inst["b_csr"], z, nc, n_public + 1, m))
        return dict(z=z, wtns=_wtns(_canonical(net, z)), e=po.exponents(inst["spec"], z, h))
    return inst, _cached(("wit", name, z_seed), g)


def _texts(proof: bytes, z_canon_public) -> tuple:
    A, B, C = o.proof_decompress(proof)
    return formats.write_proof_json(formats.SnarkjsProof(A, B, C)), formats.write_public_json(z_canon_public)


def _check_against_python(net, zkey, wtns, rs_cases, want_proofs=None):
    """every table policy and (r, s): texts and bytes equal circom.groth16_prove (and want_proofs[rs] when given)"""
    for tname, tw in TABLES.items():
        with ZKeyProver(net, zkey, table_window=tw) as zp:
            for rs in rs_cases:
                r, s = _m(rs[0]), _m(rs[1])
                pj, uj, proof = zp.prove(wtns, r, s)
                py = _cached(("py", hash(zkey), hash(wtns), rs), lambda: circom.groth16_prove(net, zkey, wtns, r, s))
                assert (pj, uj) == py, (tname, rs)
                if want_proofs is not None:
                    assert proof == want_proofs[rs], (tname, rs)
                assert pj == _texts(proof, [])[0], (tname, rs)


@pytest.mark.parametrize("name", ["2^16", "2^18", "2^20", "2^22"])
def test_known_log_keys_equal_the_oracle_and_the_python_path(net, cref, name):
    try:
        inst, wit = _instance(net, cref, name)
        rs_cases = ((0, 0), RS_RANDOM)
        _check_against_python(net, inst["zkey"], wit["wtns"], rs_cases, {rs: po.proof_bytes(wit["e"], *rs) for rs in rs_cases})
        with ZKeyProver(net, inst["zkey"], NO_TABLES) as zp:
            assert zp.info() == dict(n_vars=DLOG[name][3], n_public=DLOG[name][2], domain_size=1 << DLOG[name][0],
                                     num_constraints=DLOG[name][1])
    finally:
        if name != "2^16":                  # the other tests reuse only the 2^16 instance; the larger ones are GBs of host memory
            zh = hash(_memo[("inst", name)]["zkey"]) if ("inst", name) in _memo else None
            for key in [k for k in _memo if k[1] == name or (k[0] == "py" and k[1] == zh)]:
                del _memo[key]


# ---- the smallest keys, in a context of their own -------------------------------------------------------------------------------
# (domain, n_vars, A, B): domain 2 is what snarkjs gives a one-constraint circuit without public signals; domain 1 has no
# constraint at all.  z, a, b, c of these keys take less device memory than the proof's JSON step uses as scratch.
TINY = {"m=2": (2, 3, ([0, 2], [0, 2], [5, 7]), ([0, 1], [1], [3])),
        "m=1": (1, 1, ([0], [], []), ([0], [], []))}


def _tiny(net, cref, name):
    m, n_vars, a, b = TINY[name]
    csr = lambda t: (np.array(t[0], np.uint32), np.array(t[1], np.uint32), mont(t[2]).reshape(-1, 4))
    a_csr, b_csr = csr(a), csr(b)
    nc = len(a[0]) - 1
    spec = po.KeySpec(m, n_vars, 1, 0x7171 << 8)
    pts = {k: v if isinstance(v, np.ndarray) else host(v) for k, v in spec.device_points(net).items()}
    z = mont([1, 3, 9][:n_vars])
    h = po.expected_h(cref, *cref.qap(a_csr, b_csr, z, nc, 1, m))
    return _zkey_of(net, pts, 0, m, nc, a_csr, b_csr), _wtns(_canonical(net, z)), po.exponents(spec, z, h)


@pytest.mark.parametrize("name", list(TINY))
def test_smallest_keys_in_a_fresh_context(net, cref, name, tmp_path):
    from distributed_groth16_b200 import Net, build
    zkey, wtns, e = _tiny(net, cref, name)
    fresh = Net(0)                          # its slots' workspaces have never grown
    try:
        for tw in TABLES.values():
            with ZKeyProver(fresh, zkey, tw) as zp:
                for rs in ((0, 0), RS_RANDOM):
                    pj, uj, proof = zp.prove(wtns, _m(rs[0]), _m(rs[1]))
                    assert proof == po.proof_bytes(e, *rs), (tw, rs)
                    assert (pj, uj) == circom.groth16_prove(net, zkey, wtns, _m(rs[0]), _m(rs[1])), (tw, rs)
    finally:
        fresh.close()
    # the command: a process and a context of its own, r and s from the OS
    (tmp_path / "k.zkey").write_bytes(zkey)
    (tmp_path / "w.wtns").write_bytes(wtns)
    r = subprocess.run([build.PROVE_EXE] + [str(tmp_path / f) for f in ("k.zkey", "w.wtns", "proof.json", "public.json")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert (tmp_path / "public.json").read_text() == circom.groth16_prove(net, zkey, wtns)[1] == "[]"
    from distributed_groth16_b200.groth16 import snarkjs
    p = formats.read_proof_json((tmp_path / "proof.json").read_text())
    snarkjs.points_from_ints(net, [p.pi_a, p.pi_c])                     # raises for a point off the curve
    snarkjs.points_from_ints(net, [p.pi_b], g2=True)


def test_reference_sha256_key_gives_proof_bin(net, cref):
    from test_oracle_reference_proof import reference_sha256_instance
    pk, vk, _, _, _, _, (n_vars, n_inputs, m) = reference_sha256_instance(cref)
    d = np.load(os.path.join(G, "sha256_circuit.npz"))
    nc = int(d["dims"][2])
    to_mont = lambda v: host(net.fr_convert(net.to_device(np.ascontiguousarray(v, dtype=np.uint64)), to_mont=True))
    csr = [formats.coo_to_csr(d[k + "_rows"], d[k + "_cols"], to_mont(d[k + "_vals"]), nc) for k in "ab"]
    pts = dict(a=pk["a_query"], b1=pk["b_g1_query"], b2=pk["b_g2_query"], l=pk["l_query"], h=pk["h_query"],
               vk1=np.stack([vk["alpha_g1"], vk["beta_g1"], vk["delta_g1"]]), vk2=np.stack([vk["beta_g2"], vk["delta_g2"]]))
    zkey = _zkey_of(net, pts, n_inputs - 1, m, nc, csr[0], csr[1], ic=vk["gamma_abc_g1"], gamma2=vk["gamma_g2"])
    wtns = _wtns(d["witness"])
    gold = open(os.path.join(G, "sha256_proof.bin"), "rb").read()
    _check_against_python(net, zkey, wtns, ((0, 0), RS_RANDOM))
    for tw in TABLES.values():
        with ZKeyProver(net, zkey, tw) as zp:
            assert zp.prove(wtns, np.zeros(4, np.uint64), np.zeros(4, np.uint64))[2] == gold


def _complex():
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    exp = json.load(open(os.path.join(G, "complex_circuit_proof.json")))
    return aw.write_zkey(d), aw.write_wtns(aw.f1_witness(int(d["dims"][0]))), exp


def test_complex_circuit_key(net):
    zkey, wtns, exp = _complex()
    rs = {key: (layout.fr_to_arr([exp[key]["r"]])[0], layout.fr_to_arr([exp[key]["s"]])[0]) for key in ("r_s", "r0s0")}
    for tw in TABLES.values():
        with ZKeyProver(net, zkey, tw) as zp:
            for key, (r, s) in rs.items():
                pj, uj, proof = zp.prove(wtns, r, s)
                assert proof.hex() == exp[key]["proof_hex"], key
                assert (pj, uj) == circom.groth16_prove(net, zkey, wtns, r=r, s=s), key


# ---- edge cases ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["n_public=0", "all public"])
def test_public_input_extremes(net, cref, name):
    inst, wit = _instance(net, cref, name)
    rs_cases = ((0, 0), RS_RANDOM)
    _check_against_python(net, inst["zkey"], wit["wtns"], rs_cases, {rs: po.proof_bytes(wit["e"], *rs) for rs in rs_cases})
    if DLOG[name][2] == 0:
        with ZKeyProver(net, inst["zkey"]) as zp:
            assert zp.prove(wit["wtns"], _m(0), _m(0))[1] == "[]"


def test_shuffled_records_with_public_rows_interleaved(net, cref):
    inst, wit = _instance(net, cref, "2^16")
    log_m, nc, n_public, n_vars, _ = DLOG["2^16"]
    spec = inst["spec"]
    pts = {k: v if isinstance(v, np.ndarray) else host(v) for k, v in spec.device_points(net).items()}
    n_rec = int(inst["a_csr"][0][-1]) + int(inst["b_csr"][0][-1]) + n_public + 1
    order = np.random.default_rng(5).permutation(n_rec)
    zkey = _zkey_of(net, pts, n_public, 1 << log_m, nc, inst["a_csr"], inst["b_csr"], order=order)
    rows = formats.read_zkey(zkey).coef_row
    assert rows.size == n_rec
    assert (np.flatnonzero(rows >= nc) < n_rec - n_public - 1).any()      # public-input rows among the constraints' records
    with ZKeyProver(net, zkey, NO_TABLES) as zp:
        assert zp.info()["num_constraints"] == nc
        for rs in ((0, 0), RS_RANDOM):
            assert zp.prove(wit["wtns"], _m(rs[0]), _m(rs[1]))[2] == po.proof_bytes(wit["e"], *rs), rs


def test_zkey_without_coefficient_records(net, cref):
    # the domain snarkjs gives such a circuit: the n_public + 1 input rows, rounded up to a power of two
    spec = po.KeySpec(4, 20, 3, 0x5151 << 8)
    pts = {k: v if isinstance(v, np.ndarray) else host(v) for k, v in spec.device_points(net).items()}
    empty = (np.zeros(1, np.uint32), np.zeros(0, np.uint32), np.zeros((0, 4), np.uint64))
    zkey = _zkey_of(net, pts, 2, 4, 0, empty, empty)
    zk = formats.read_zkey(zkey)
    zkey = formats.write_zkey(formats.ZKey(**{**zk.__dict__, "coef_matrix": zk.coef_matrix[:0], "coef_row": zk.coef_row[:0],
                                              "coef_col": zk.coef_col[:0], "coef_val_r2": zk.coef_val_r2[:0]}))
    z = witness(np.random.default_rng(3), 20, "random", 3)
    wtns = _wtns(_canonical(net, z))
    _check_against_python(net, zkey, wtns, ((0, 0), RS_RANDOM))
    with ZKeyProver(net, zkey) as zp:
        assert zp.info()["num_constraints"] == 0


def test_designed_randomisers_give_infinity_json(net, cref):
    inst, wit = _instance(net, cref, "2^16")
    with ZKeyProver(net, inst["zkey"]) as zp:
        for case, (r, s) in po.designed_cases(wit["e"]).items():
            pj, _, proof = zp.prove(wit["wtns"], _m(r), _m(s))
            assert proof == po.proof_bytes(wit["e"], r, s), case
            obj = json.loads(pj)
            if case == "A_inf":
                assert obj["pi_a"] == ["0", "1", "0"]
            elif case == "B_inf":
                assert obj["pi_b"] == [["0", "0"], ["1", "0"], ["0", "0"]]
            else:
                assert obj["pi_c"] == ["0", "1", "0"]
            assert pj == circom.groth16_prove(net, inst["zkey"], wit["wtns"], _m(r), _m(s))[0], case


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def _refused(net, fn, code, text):
    """Net.check raises B200zkError with the code, and MpcNetError for ERR_LENGTH (the reference's Generic error)"""
    before = net.launch_count()
    with pytest.raises(MpcNetError if code == ERR_LENGTH else B200zkError) as e:
        fn()
    assert code == ERR_LENGTH or e.value.code == code, (e.value.code, e.value.message)
    assert text in e.value.message, e.value.message
    return net.launch_count() - before


def _edit_section(buf, sid, fn):
    pre = buf[:8]
    nsec = struct.unpack_from("<I", buf, 8)[0]
    off, secs = 12, []
    for _ in range(nsec):
        s, ln = struct.unpack_from("<IQ", buf, off)
        secs.append((s, fn(buf[off + 12:off + 12 + ln]) if s == sid else buf[off + 12:off + 12 + ln]))
        off += 12 + ln
    return pre + struct.pack("<I", len(secs)) + b"".join(struct.pack("<IQ", s, len(p)) + p for s, p in secs)


def test_refusals(net, cref):
    zkey, wtns, _ = _complex()
    zk = formats.read_zkey(zkey)
    # host-detectable zkey faults: the message of read_zkey (or the native reader's own), and no launch
    bad = {"bad magic b'zkez' (expected b'zkey')": b"zkez" + zkey[4:],
           "zkey section 5 missing": _edit_section(zkey, 5, lambda p: p).replace(struct.pack("<IQ", 5, zk.n_vars * 64),
                                                                                 struct.pack("<IQ", 11, zk.n_vars * 64), 1),
           "zkey protocol 2 is not Groth16 (1)": _edit_section(zkey, 1, lambda p: struct.pack("<I", 2)),
           "zkey is not over BN254": _edit_section(zkey, 2, lambda p: p[:4] + (formats.FQ_MODULUS + 2).to_bytes(32, "little") + p[36:]),
           "zkey header: domain size 12 is not a power of two": _edit_section(zkey, 2, lambda p: p[:80] + struct.pack("<I", 12) + p[84:]),
           "zkey section 9 too short": _edit_section(zkey, 9, lambda p: p[:-64]),
           "runs past the end of the file": zkey[:len(zkey) - 100]}
    for text, buf in bad.items():
        assert _refused(net, lambda: ZKeyProver(net, buf), ERR_ARG, text) == 0, text
    # bad coefficient records: found on the device, the count and the first index named
    rec = lambda k, field, v: (lambda p: p[:4 + 44 * k + 4 * field] + struct.pack("<I", v) + p[8 + 44 * k + 4 * field:])
    two_bad = _edit_section(_edit_section(zkey, 4, rec(7, 0, 2)), 4, rec(3, 2, zk.n_vars))
    _refused(net, lambda: ZKeyProver(net, two_bad), ERR_ARG, "2 of %d records have matrix index > 1" % zk.coef_row.size)
    _refused(net, lambda: ZKeyProver(net, two_bad), ERR_ARG, "the first at index 3")

    w = formats.read_wtns(wtns)
    with ZKeyProver(net, zkey) as zp:
        assert _refused(net, lambda: zp.prove(_wtns(w[:-1])), ERR_LENGTH,
                        "witness has %d entries, the key expects %d" % (w.shape[0] - 1, w.shape[0])) == 0
        assert _refused(net, lambda: zp.prove(b"wtnx" + wtns[4:]), ERR_ARG, "bad magic b'wtnx' (expected b'wtns')") == 0
        assert _refused(net, lambda: zp.prove(wtns[:-8]), ERR_ARG, "runs past the end of the file") == 0
        big = w.copy()
        for i in (9, 4):
            big[i] = [(R >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(4)]
        _refused(net, lambda: zp.prove(_wtns(big)), ERR_ARG, "witness: 2 of %d entries are not below r, the first is w[4]" % w.shape[0])

        # short buffers: refused before any launch with the sizes needed, then proved at exactly those sizes
        lib = net._lib
        proof = (ctypes.c_uint8 * 128)()
        zero = np.zeros(4, np.uint64)
        want = circom.groth16_prove(net, zkey, wtns, zero, zero)
        for plen0, ulen0 in ((PROOF_JSON_MAX - 1, 1000), (PROOF_JSON_MAX, len(want[1])), (10, 0)):
            plen, ulen = ctypes.c_size_t(plen0), ctypes.c_size_t(ulen0)
            pbuf, ubuf = ctypes.create_string_buffer(max(plen0, 1)), ctypes.create_string_buffer(max(ulen0, 1))
            before = net.launch_count()
            rc = lib.b200zk_zkey_prove(net._h, zp._h, wtns, len(wtns), zero.ctypes.data, zero.ctypes.data, proof, pbuf,
                                       ctypes.byref(plen), ubuf, ctypes.byref(ulen))
            assert rc == ERR_SHORT_BUFFER and net.launch_count() == before
            assert (plen.value, ulen.value) == (PROOF_JSON_MAX, len(want[1]) + 1)
            pbuf, ubuf = ctypes.create_string_buffer(plen.value), ctypes.create_string_buffer(ulen.value)
            assert lib.b200zk_zkey_prove(net._h, zp._h, wtns, len(wtns), zero.ctypes.data, zero.ctypes.data, proof, pbuf,
                                         ctypes.byref(plen), ubuf, ctypes.byref(ulen)) == 0
            assert (pbuf.raw[:plen.value].decode(), ubuf.raw[:ulen.value].decode()) == want
        # no outputs asked for at all: still proves
        assert lib.b200zk_zkey_prove(net._h, zp._h, wtns, len(wtns), None, None, proof, None, None, None, None) == 0
        assert zp.prove(wtns, zero, zero)[0] == want[0]           # the handle still works after every refusal


# ---- randomness, reuse, memory --------------------------------------------------------------------------------------------------
def test_random_r_s_are_fresh_and_verify(net):
    zkey, wtns, _ = _complex()
    vk = circom.zkey_export_verificationkey(net, zkey)
    with ZKeyProver(net, zkey) as zp:
        p1, u1, b1 = zp.prove(wtns)
        p2, u2, b2 = zp.prove(wtns)
    assert b1 != b2 and p1 != p2 and u1 == u2
    assert circom.groth16_verify(net, vk, u1, p1) and circom.groth16_verify(net, vk, u2, p2)


def test_reuse_two_handles_and_memory_returns(net, cref):
    import torch
    inst, _ = _instance(net, cref, "2^16")
    wits = [_instance(net, cref, "2^16", z_seed=0x33 + k)[1] for k in range(3)]
    zkey_c, wtns_c, _ = _complex()
    want_c = circom.groth16_prove(net, zkey_c, wtns_c, _m(0), _m(0))
    with ZKeyProver(net, inst["zkey"]) as a, ZKeyProver(net, zkey_c) as b:    # warm the context's workspaces
        a.prove(wits[0]["wtns"], *(_m(v) for v in RS_RANDOM))
        b.prove(wtns_c, _m(0), _m(0))
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    a, b = ZKeyProver(net, inst["zkey"]), ZKeyProver(net, zkey_c)
    try:
        for k, wit in enumerate(wits):
            assert a.prove(wit["wtns"], *(_m(v) for v in RS_RANDOM))[2] == po.proof_bytes(wit["e"], *RS_RANDOM), k
            assert b.prove(wtns_c, _m(0), _m(0))[:2] == want_c, k
    finally:
        a.free()
        b.free()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


# ---- the command ----------------------------------------------------------------------------------------------------------------
def test_command(net, tmp_path):
    from distributed_groth16_b200 import build
    zkey, wtns, _ = _complex()
    (tmp_path / "c.zkey").write_bytes(zkey)
    (tmp_path / "w.wtns").write_bytes(wtns)
    exe = build.PROVE_EXE
    run = lambda *a: subprocess.run([exe] + [str(tmp_path / x) for x in a], capture_output=True, text=True)
    r = run("c.zkey", "w.wtns", "proof.json", "public.json")
    assert r.returncode == 0, r.stderr
    proof, public = (tmp_path / "proof.json").read_text(), (tmp_path / "public.json").read_text()
    assert public == circom.groth16_prove(net, zkey, wtns)[1]
    assert circom.groth16_verify(net, circom.zkey_export_verificationkey(net, zkey), public, proof)
    (tmp_path / "bad.zkey").write_bytes(zkey[:-100])
    (tmp_path / "bad.wtns").write_bytes(b"wtnx" + wtns[4:])
    for args, text in ((("bad.zkey", "w.wtns"), "runs past the end of the file"), (("c.zkey", "bad.wtns"), "bad magic"),
                       (("missing.zkey", "w.wtns"), "No such file")):
        r = run(*args, "p2.json", "u2.json")
        assert r.returncode != 0 and text in r.stderr, (args, r.stderr)
        assert sorted(os.listdir(tmp_path)) == ["bad.wtns", "bad.zkey", "c.zkey", "proof.json", "public.json", "w.wtns"], args
