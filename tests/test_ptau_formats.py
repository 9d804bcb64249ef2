"""Setup from a Powers-of-Tau file, host side (no GPU): the zkey writer, the header and coefficient sections `zkey new`
derives from an r1cs, the ptau reader, and the pure-Python `zkey new` that the GPU path is checked against."""
import hashlib
import lzma
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")
TINY = dict(tau=0x1234567890ABCDEF, alpha=1111111111111111111, beta=2222222222222222223)


def _r2(vals):
    """canonical ints -> value * R^2 mod r as (n, 4) u64 limbs (the zkey coefficient words)."""
    from oracle import bn254 as o
    return np.array([[(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] for x in
                     (int(v) * o.MONT_R * o.MONT_R % o.R for v in vals)], dtype=np.uint64).reshape(-1, 4)


def _canonical(limbs):
    return [int.from_bytes(r.tobytes(), "little") for r in np.asarray(limbs, dtype=np.uint64).reshape(-1, 4)]


def _golden_zkey(d):
    """the complex-circuit golden arrays as a formats.ZKey (coefficients in snarkjs order via zkey_coefficients)."""
    from distributed_groth16_b200 import formats
    from oracle import layout
    n_vars, n_public, m, nc = (int(x) for x in d["dims"])
    r2 = lambda k: _r2(layout.arr_to_fr(d[k + "_vals"]))            # the golden holds Montgomery values
    mi, ci, si, vi = formats.zkey_coefficients(n_public, nc, (d["a_rows"], d["a_cols"], r2("a")), (d["b_rows"], d["b_cols"], r2("b")))
    return formats.ZKey(n_vars=n_vars, n_public=n_public, domain_size=m, alpha_g1=d["vk_g1"][0], beta_g1=d["vk_g1"][1],
                        beta_g2=d["vk_g2"][0], gamma_g2=d["vk_g2"][2], delta_g1=d["vk_g1"][2], delta_g2=d["vk_g2"][1],
                        ic=d["ic"], a_query=d["a_query"], b_g1_query=d["b_g1_query"], b_g2_query=d["b_g2_query"],
                        l_query=d["l_query"], h_query=d["h_query"], coef_matrix=mi, coef_row=ci, coef_col=si, coef_val_r2=vi)


def test_write_zkey_reproduces_the_reference_complex_circuit_zkey():
    from distributed_groth16_b200 import formats
    x = np.load(os.path.join(G, "reference_artefacts.npz"))
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    buf = formats.write_zkey(_golden_zkey(d), section10=x["zkey_sec10"].tobytes())
    assert hashlib.sha256(buf).hexdigest() == str(x["zkey_sha256"])
    assert [sid for sid, _, _ in _table(buf)] == [int(s) for s in x["zkey_order"]]
    default = formats.write_zkey(_golden_zkey(d))                      # zero csHash, zero contributions
    assert _section(default, 10) == bytes(68) and formats.read_zkey(default).n_vars == int(d["dims"][0])


def _table(buf):
    _v, n = struct.unpack_from("<II", buf, 4)
    off, out = 12, []
    for _ in range(n):
        sid, ln = struct.unpack_from("<IQ", buf, off)
        out.append((sid, off + 12, ln))
        off += 12 + ln
    return out


def _section(buf, sid):
    return next(buf[o_:o_ + ln] for s, o_, ln in _table(buf) if s == sid)


def test_zkey_new_header_and_coefficients_from_the_complex_circuit_r1cs():
    """Sections 1, 4 and the non-point fields of 2, derived from the r1cs the reference's complex-circuit zkey was made
    from (snarkjs zkey new), equal that zkey's bytes."""
    import artefact_writer as aw
    from distributed_groth16_b200 import formats
    x = np.load(os.path.join(G, "reference_artefacts.npz"))
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    ref = aw.zkey_sections(d)                       # byte-identical to the reference file (test_formats)
    r1 = formats.read_r1cs(lzma.decompress(x["complex_r1cs_xz"].tobytes()))
    n_public = r1.n_pub_out + r1.n_pub_in
    k = formats.zkey_cir_power(r1.n_constraints, n_public)
    coefs = formats.zkey_coefficients(n_public, r1.n_constraints, (r1.rows[0], r1.cols[0], _r2(_canonical(r1.vals[0]))),
                                      (r1.rows[1], r1.cols[1], _r2(_canonical(r1.vals[1]))))
    z = lambda n, w: np.zeros((n, w), dtype=np.uint64)
    n = r1.n_wires
    zk = formats.ZKey(n_vars=n, n_public=n_public, domain_size=1 << k, alpha_g1=z(1, 8), beta_g1=z(1, 8), beta_g2=z(1, 16),
                      gamma_g2=z(1, 16), delta_g1=z(1, 8), delta_g2=z(1, 16), ic=z(n_public + 1, 8), a_query=z(n, 8),
                      b_g1_query=z(n, 8), b_g2_query=z(n, 16), l_query=z(n - n_public - 1, 8), h_query=z(1 << k, 8),
                      coef_matrix=coefs[0], coef_row=coefs[1], coef_col=coefs[2], coef_val_r2=coefs[3])
    buf = formats.write_zkey(zk)
    assert _section(buf, 1) == ref[1]
    assert _section(buf, 4) == ref[4]
    assert _section(buf, 2)[:84] == ref[2][:84]                    # n8q q n8r r n_vars n_public domain_size


@pytest.fixture(scope="module")
def tiny_ptau():
    import ptau_writer as pw
    return pw.sections_oracle(TINY["tau"], TINY["alpha"], TINY["beta"], power=2)


def test_ptau_reader_accepts_the_writer_and_rejects_malformed_files(tiny_ptau, tmp_path):
    import ptau_writer as pw
    from distributed_groth16_b200 import formats
    from oracle import bn254 as o, layout
    with formats.read_ptau(pw.write_ptau(str(tmp_path / "ok.ptau"), tiny_ptau)) as pt:
        assert (pt.power, pt.ceremony_power) == (2, 2)
        assert layout.arr_to_g1(pt.alpha_g1)[0] == o.G1.mul(o.G1_GEN, TINY["alpha"])
        assert layout.arr_to_g2(pt.beta_g2)[0] == o.G2.mul(o.G2_GEN, TINY["beta"])
        lag = layout.arr_to_g1(pt.lagrange(12, 2))
        lag_s = o.intt([pow(TINY["tau"], i, o.R) for i in range(4)])
        assert lag == [o.G1.mul(o.G1_GEN, s) for s in lag_s]
        assert pt.lagrange(12, 3).shape == (8, 8) and pt.lagrange(13, 2).shape == (4, 16)
        with pytest.raises(formats.FormatError, match="too big"):
            pt.lagrange(14, 3)                                   # a circuit of domain 2^3 needs a power-3 ceremony
        with pytest.raises(formats.FormatError, match="too big"):
            pt.lagrange(12, 4)

    def bad(secs, match, magic=b"ptau"):
        p = pw.write_ptau(str(tmp_path / "bad.ptau"), secs, magic)
        with pytest.raises(formats.FormatError, match=match):
            formats.read_ptau(p).close()

    bad(tiny_ptau, "magic", magic=b"zkey")
    s1 = tiny_ptau[1]
    bad({**tiny_ptau, 1: struct.pack("<I", 48) + s1[4:]}, "BN254")
    bad({**tiny_ptau, 1: s1[:4] + (o.R).to_bytes(32, "little") + s1[36:]}, "BN254")
    for sid in (12, 13, 14, 15):
        bad({k: v for k, v in tiny_ptau.items() if k != sid}, "not prepared")
        bad({**tiny_ptau, sid: tiny_ptau[sid][:-64]}, "too short")
    bad({**tiny_ptau, 1: s1[:36] + struct.pack("<II", 3, 3)}, "too short")        # stated power above the data
    with open(str(tmp_path / "trunc.ptau"), "wb") as f:
        f.write(pw.ptau_bytes(tiny_ptau)[:-100])
    with pytest.raises(formats.FormatError, match="past the end"):
        formats.read_ptau(str(tmp_path / "trunc.ptau"))


def test_oracle_zkey_new_on_the_tiny_circuit_proves_and_verifies(tiny_ptau):
    """circom2_multiplier2 (c = a * b, c public): the pure-Python zkey new on a power-2 ptau gives a key whose oracle proof
    verifies under the oracle pairing for c and fails for c + 1."""
    import ptau_writer as pw
    import zkey_oracle
    from oracle import bn254 as o
    r1cs = open(os.path.join(G, "circom2_multiplier2.r1cs"), "rb").read()
    zk = zkey_oracle.zkey_new(r1cs, pw.ptau_bytes(tiny_ptau))
    pk, ma, mb, nc = o.read_zkey(zk)
    assert (pk.n_vars, pk.n_public, pk.domain_size, nc) == (4, 1, 4, 1)
    a, b = 3, 11
    z = [1, a * b, a, b]
    qa, qb, qc = o.qap(ma, mb, pk.n_public + 1, nc, z)
    A, B, C = o.groth16_prove(pk, z, o.h_circom(qa, qb, qc), 12345, 67890)
    assert o.groth16_verify(pk.alpha_g1, pk.beta_g2, pk.gamma_g2, pk.delta_g2, pk.ic, [a * b], A, B, C)
    assert not o.groth16_verify(pk.alpha_g1, pk.beta_g2, pk.gamma_g2, pk.delta_g2, pk.ic, [a * b + 1], A, B, C)
