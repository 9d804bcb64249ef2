"""snarkjs's Groth16 files on the GPU: `zkey export verificationkey`, `groth16 prove` / `groth16 verify` on proof.json and
public.json, and `wtns check` (groth16/snarkjs.py, groth16/circom.py, b200zk_vk_alphabeta_12, b200zk_r1cs_check_dev).

Pinned against the files snarkjs wrote for the reference's million-constraint circuit (tests/golden/snarkjs_million/), the
snarkjs-made complex-circuit key, and the oracle (oracle/bn254.py)."""
import ctypes
import hashlib
import json
import lzma
import os
import sys

import numpy as np
import pytest

from distributed_groth16_b200 import B200zkError, formats
from distributed_groth16_b200._native import ERR_ARG
from distributed_groth16_b200.groth16 import circom, snarkjs

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")
M = os.path.join(G, "snarkjs_million")
U = 4965661367192848881
SNARKJS_M = 2 * U * (6 * U * U + 3 * U + 1)


def _text(name):
    return open(os.path.join(M, name)).read()


def _snarkjs_nesting(f):
    """Oracle Fq12 (12 Fq coefficients of w^0..w^11, u = w^6 - 9) -> snarkjs's [[c0.a, c0.b, c0.c], [c1.a, c1.b, c1.c]]."""
    out = [[None] * 3 for _ in range(2)]
    for (h, k), i in zip(((0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (1, 2)), (0, 2, 4, 1, 3, 5)):
        y = f[i + 6]
        out[h][k] = [(f[i] + 9 * y) % formats.FQ_MODULUS, y]
    return out


# ---- zkey export verificationkey ---------------------------------------------------------------------------------------

def test_vk_export_of_the_million_key_equals_the_snarkjs_file_byte_for_byte(net):
    from oracle import bn254 as o
    want = _text("verification_key.json")
    vk = formats.read_vk_json(want)
    avk = snarkjs.read_vk_json(net, want)
    ab = snarkjs.alphabeta_12(net, avk.alpha_g1, avk.beta_g2)
    out = formats.SnarkjsVerificationKey(vk.n_public, vk.alpha_1, vk.beta_2, vk.gamma_2, vk.delta_2, ab,
                                         snarkjs.points_to_ints(net, avk.gamma_abc_g1))
    assert formats.write_vk_json(out) == want
    # the test would catch a device value without the m exponent, or with the Fq6 halves swapped
    plain = _snarkjs_nesting(o.pairing(vk.alpha_1, vk.beta_2))
    assert plain != ab and _snarkjs_nesting(o.fq12_pow(o.pairing(vk.alpha_1, vk.beta_2), SNARKJS_M)) == ab
    for mutant in (plain, [ab[1], ab[0]]):
        out.alphabeta_12 = mutant
        assert formats.write_vk_json(out) != want


# ---- groth16 verify ----------------------------------------------------------------------------------------------------

def _proof_with(fn):
    obj = json.loads(_text("proof.json"))
    fn(obj)
    return json.dumps(obj, indent=1)


def test_snarkjs_million_proof_verifies_and_tampering_is_rejected(net):
    from oracle import bn254 as o
    vk, pub, proof = _text("verification_key.json"), _text("public.json"), _text("proof.json")
    assert circom.groth16_verify(net, vk, pub, proof)
    assert not circom.groth16_verify(net, vk, '["999993"]', proof)
    assert not circom.groth16_verify(net, vk, json.dumps([str(999992 + o.R)]), proof)        # no aliasing mod r
    assert not circom.groth16_verify(net, vk, '[]', proof)
    assert not circom.groth16_verify(net, vk, '["999992", "1"]', proof)

    def off_curve(obj):
        obj["pi_a"][1] = str((int(obj["pi_a"][1]) + 1) % o.P)
    assert not circom.groth16_verify(net, vk, pub, _proof_with(off_curve))

    x = (1, 0)                                                         # a twist point outside the order-r subgroup
    while True:
        y = o.fq2_sqrt(o.fq2_add(o.fq2_mul(o.fq2_sqr(x), x), o.B_G2))
        if y is not None:
            break
        x = (x[0] + 1, 0)
    assert o.G2.is_on_curve((x, y)) and o.G2.from_jac(o.G2.jac_mul(o.G2.to_jac((x, y)), o.R)) is not None

    def outside(obj):
        obj["pi_b"] = [[str(x[0]), str(x[1])], [str(y[0]), str(y[1])], ["1", "0"]]
    assert not circom.groth16_verify(net, vk, pub, _proof_with(outside))

    bad_vk = json.loads(vk)
    bad_vk["IC"].append(bad_vk["IC"][0])
    with pytest.raises(formats.FormatError, match="IC"):
        circom.groth16_verify(net, json.dumps(bad_vk, indent=1), pub, proof)
    bad_vk = json.loads(vk)
    bad_vk["vk_alpha_1"][1] = str((int(bad_vk["vk_alpha_1"][1]) + 1) % o.P)                  # a vk point off the curve
    with pytest.raises(formats.FormatError):
        circom.groth16_verify(net, json.dumps(bad_vk, indent=1), pub, proof)
    with pytest.raises(formats.FormatError):
        circom.groth16_verify(net, vk, "not json", proof)


# ---- complex circuit: groth16 prove -> JSON -> groth16 verify ------------------------------------------------------------

def test_complex_circuit_prove_export_and_verify_through_json(net):
    import artefact_writer as aw
    from oracle import bn254 as o, layout
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    exp = json.load(open(os.path.join(G, "complex_circuit_proof.json")))
    n_vars, n_public = int(d["dims"][0]), int(d["dims"][1])
    zkey, z = aw.write_zkey(d), aw.f1_witness(n_vars)
    wtns = aw.write_wtns(z)

    vk_json = circom.zkey_export_verificationkey(net, zkey)
    alpha, (beta, delta, gamma) = layout.arr_to_g1(d["vk_g1"])[0], layout.arr_to_g2(d["vk_g2"])
    want_vk = formats.SnarkjsVerificationKey(n_public, alpha, beta, gamma, delta,
                                             _snarkjs_nesting(o.fq12_pow(o.pairing(alpha, beta), SNARKJS_M)),
                                             layout.arr_to_g1(d["ic"]))
    assert vk_json == formats.write_vk_json(want_vk)

    for key in ("r_s", "r0s0"):
        r, s = layout.fr_to_arr([exp[key]["r"]])[0], layout.fr_to_arr([exp[key]["s"]])[0]        # 12345, 67890 and 0, 0
        proof_json, public_json = circom.groth16_prove(net, zkey, wtns, r=r, s=s)
        A, B, C = o.proof_decompress(bytes.fromhex(exp[key]["proof_hex"]))
        assert proof_json == formats.write_proof_json(formats.SnarkjsProof(A, B, C)), key
        assert public_json == '[\n "%s"\n]' % exp["public_input"]
        assert circom.groth16_verify(net, vk_json, public_json, proof_json), key
        assert not circom.groth16_verify(net, vk_json, json.dumps([str(z[1] + 1)]), proof_json)


# ---- wtns check on real circuits ------------------------------------------------------------------------------------------

def _r1cs_constraints(d, n_constraints) -> bytes:
    """artefact_writer.r1cs_constraints without the per-constraint loop: per constraint and matrix a u32 term count, then
    the (u32 wire, 32-byte value) terms."""
    cnt = np.stack([np.bincount(d[k + "_rows"].astype(np.int64), minlength=n_constraints) for k in "abc"], axis=1).reshape(-1)
    start = np.concatenate([[0], np.cumsum(4 + 36 * cnt)])
    buf = np.zeros(int(start[-1]), dtype=np.uint8)
    buf[start[:-1, None] + np.arange(4)] = cnt.astype("<u4").view(np.uint8).reshape(-1, 4)
    for m, k in enumerate("abc"):
        rows = d[k + "_rows"].astype(np.int64)
        block = 3 * rows + m
        rank = np.arange(rows.size) - np.searchsorted(rows, rows)      # the term's place in its (sorted) row
        pos = start[block] + 4 + 36 * rank
        buf[pos[:, None] + np.arange(4)] = d[k + "_cols"].astype("<u4").view(np.uint8).reshape(-1, 4)
        buf[pos[:, None] + 4 + np.arange(32)] = np.ascontiguousarray(d[k + "_vals"], dtype="<u8").view(np.uint8).reshape(-1, 32)
    return buf.tobytes()


_SHA256 = []


def _sha256():
    """The reference's sha256 r1cs, rebuilt from the goldens (test_formats checks the SHA-256 of this rebuild), and its
    witness."""
    import artefact_writer as aw
    if not _SHA256:
        x = np.load(os.path.join(G, "reference_artefacts.npz"))
        s = np.load(os.path.join(G, "sha256_circuit.npz"))
        secs = {1: x["sha256_r1cs_sec1"].tobytes(), 2: _r1cs_constraints(s, int(s["dims"][2])), 3: x["sha256_r1cs_sec3"].tobytes()}
        r1cs = aw.container(b"r1cs", [(int(sid), secs[int(sid)]) for sid in x["sha256_r1cs_order"]])
        assert hashlib.sha256(r1cs).hexdigest() == str(x["sha256_r1cs_sha256"])
        _SHA256.append((r1cs, [int.from_bytes(r.tobytes(), "little") for r in s["witness"]], s))
    r1cs, w, s = _SHA256[0]
    return r1cs, list(w), s


def test_wtns_check_accepts_the_witnesses_of_real_circuits(net):
    import artefact_writer as aw
    x = np.load(os.path.join(G, "reference_artefacts.npz"))
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    rep = circom.wtns_check(net, lzma.decompress(x["complex_r1cs_xz"].tobytes()), aw.write_wtns(aw.f1_witness(int(d["dims"][0]))))
    assert rep.ok and rep.n_failed == 0 and rep.lines == []
    r1cs, w, _ = _sha256()
    rep = circom.wtns_check(net, r1cs, aw.write_wtns(w))
    assert rep.ok and rep.n_failed == 0 and rep.first_failed == 30134 and rep.lines == []


def test_wtns_check_reports_exactly_the_constraints_a_changed_entry_breaks(net):
    import artefact_writer as aw
    from oracle import bn254 as o
    r1cs, w, s = _sha256()
    n_cons = int(s["dims"][2])
    w[777] = (w[777] + 1) % o.R
    acc = {}
    for k in "abc":
        vals = [int.from_bytes(r.tobytes(), "little") for r in s[k + "_vals"]]
        v = [0] * n_cons
        for r_, c_, val in zip(s[k + "_rows"], s[k + "_cols"], vals):
            v[int(r_)] = (v[int(r_)] + val * w[int(c_)]) % o.R
        acc[k] = v
    bad = [i for i in range(n_cons) if acc["a"][i] * acc["b"][i] % o.R != acc["c"][i]]
    assert bad
    rep = circom.wtns_check(net, r1cs, aw.write_wtns(w))
    i = bad[0]
    assert not rep.ok and (rep.n_failed, rep.first_failed) == (len(bad), i) and len(rep.lines) == 1
    assert "constraint %d " % i in rep.lines[0]
    assert "<A,w> = %d, <B,w> = %d, <C,w> = %d" % (acc["a"][i], acc["b"][i], acc["c"][i]) in rep.lines[0]


def test_wtns_check_rejects_a_malformed_witness_with_one_line(net):
    import artefact_writer as aw
    from oracle import bn254 as o
    r1cs, w, _ = _sha256()
    for bad, where in ((w[:-1], "29822 entries"), ([2] + w[1:], "w[0] = 2"), (w[:500] + [o.R + 3] + w[501:], "w[500]")):
        rep = circom.wtns_check(net, r1cs, aw.write_wtns(bad))
        assert not rep.ok and len(rep.lines) == 1 and where in rep.lines[0], (where, rep.lines)
        assert rep.n_failed == 0


# ---- wtns check at scale, through the device entry ----------------------------------------------------------------------

def _synthetic(rng, n, n_wires=1 << 16, long_row=1 << 20, empty=97):
    """CSR A, B, C over small values, so that every product is exact in u64, on which every row holds.  Rows 3, 3 + empty,
    3 + 2 empty, ... are empty in all three matrices; row 5 of A has `long_row` terms."""
    w = rng.integers(1, 1 << 16, n_wires, dtype=np.uint64)
    w[0] = 1
    mats, sums = [], []
    for m in range(2):
        cnt = rng.choice(np.array([0, 1, 2], dtype=np.int64), n, p=[0.25, 0.5, 0.25])
        cnt[5] = long_row if m == 0 else 1
        cnt[3::empty] = 0
        ptr = np.zeros(n + 1, dtype=np.uint64)
        ptr[1:] = np.cumsum(cnt)
        nnz = int(ptr[-1])
        col = rng.integers(0, n_wires, nnz, dtype=np.uint32)
        val = rng.integers(0, 1 << 8, nnz, dtype=np.uint64)
        if m == 1:
            col[int(ptr[5])], val[int(ptr[5])] = 0, 1                  # B_5 = w[0] = 1
        cs = np.zeros(nnz + 1, dtype=np.uint64)
        np.cumsum(val * w[col], out=cs[1:])
        sums.append(cs[ptr[1:]] - cs[ptr[:-1]])
        mats.append((ptr.astype(np.uint32), col, val))
    cnt = np.ones(n, dtype=np.int64)
    cnt[3::empty] = 0
    ptr = np.zeros(n + 1, dtype=np.uint32)
    ptr[1:] = np.cumsum(cnt)
    c_val = (sums[0] * sums[1])[cnt == 1]                              # < 2^52; < 2^44 on the long row, where B_5 = 1
    mats.append((ptr, np.zeros(int(ptr[-1]), dtype=np.uint32), c_val))
    return mats, w, cnt == 1


def _check_dev(net, mats, w, n):
    def limbs(v):
        out = np.zeros((v.shape[0], 4), dtype=np.uint64)
        out[:, 0] = v
        return net.fr_convert(net.to_device(out), to_mont=True) if v.shape[0] else None
    dev = [(net.to_device(p.view(np.int32)), net.to_device(c.view(np.int32)) if c.size else None, limbs(v)) for p, c, v in mats]
    return snarkjs.r1cs_check(net, dev, limbs(w), n)


@pytest.mark.parametrize("log_n", [16, 20, 24])
def test_r1cs_check_at_scale_counts_and_locates_planted_failures(net, log_n):
    """2^16 rows take the warp-per-row kernel, 2^20 and 2^24 the thread-per-row one."""
    n = 1 << log_n
    mats, w, has_c = _synthetic(np.random.default_rng(log_n), n)
    assert int(mats[0][0][6]) - int(mats[0][0][5]) == 1 << 20 and not has_c[3] and has_c[[0, 5, n - 1]].all()
    assert _check_dev(net, mats, w, n) == (0, n)
    run = np.arange(n // 2, n // 2 + 300)
    c_pos = np.cumsum(has_c) - 1                                       # row -> index of its C term
    for planted in (np.array([0]), np.array([n - 1]), run, np.concatenate([[0, 5], run, [n - 1]]), np.array([5, n - 1])):
        planted = planted[has_c[planted]]                              # an empty row has no C term to corrupt
        first = int(planted[0])
        p, c, v = mats[2]
        v = v.copy()
        v[c_pos[planted]] += np.uint64(1)
        assert _check_dev(net, mats[:2] + [(p, c, v)], w, n) == (planted.size, first), (log_n, first)


def test_r1cs_check_with_no_terms_and_argument_errors(net):
    w = np.array([1, 2, 3], dtype=np.uint64)
    for n in (1 << 16, 1 << 20):
        empty = (np.zeros(n + 1, dtype=np.uint32), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint64))
        assert _check_dev(net, [empty] * 3, w, n) == (0, n)
    lib, h = net._lib, net._h
    nf, ff = ctypes.c_uint64(7), ctypes.c_uint64(7)
    assert lib.b200zk_r1cs_check_dev(h, 0, *([None] * 9), 0, None, ctypes.byref(nf), ctypes.byref(ff)) == 0
    assert (nf.value, ff.value) == (0, 0)
    assert lib.b200zk_r1cs_check_dev(h, 0, *([None] * 9), 5, None, ctypes.byref(nf), ctypes.byref(ff)) == ERR_ARG
    import torch
    p = torch.zeros(6, dtype=torch.int32, device="cuda")
    wd = torch.zeros((1, 4), dtype=torch.int64, device="cuda")
    ptrs = [ctypes.c_void_p(p.data_ptr()), None, None] * 3
    assert lib.b200zk_r1cs_check_dev(h, 0, *ptrs, 5, ctypes.c_void_p(wd.data_ptr()), ctypes.byref(nf), ctypes.byref(ff)) == 0
    assert (nf.value, ff.value) == (0, 5)
    assert lib.b200zk_r1cs_check_dev(h, 0, *ptrs, 5, ctypes.c_void_p(wd.data_ptr()), None, ctypes.byref(ff)) == ERR_ARG
    assert lib.b200zk_r1cs_check_dev(h, 0, *ptrs, 5, None, ctypes.byref(nf), ctypes.byref(ff)) == ERR_ARG
    assert lib.b200zk_r1cs_check_dev(h, 3, *ptrs, 5, ctypes.c_void_p(wd.data_ptr()), ctypes.byref(nf), ctypes.byref(ff)) == ERR_ARG
    bad = list(ptrs)
    bad[6] = None                                                      # C's row pointers
    assert lib.b200zk_r1cs_check_dev(h, 0, *bad, 5, ctypes.c_void_p(wd.data_ptr()), ctypes.byref(nf), ctypes.byref(ff)) == ERR_ARG
    with pytest.raises(B200zkError):
        snarkjs.r1cs_check(net, [(None, None, None)] * 3, wd, 5)
