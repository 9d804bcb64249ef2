"""Bellman MPC-params files (snarkjs `zkey export bellman` / `zkey bellman contribute` / `zkey import bellman`), host side
(no GPU): formats.parse_bellman and bellman_size on files the pure-Python restatement (bellman_oracle) makes from the
tiny circuit's key, the circuit hash of an exported prefix, and the refusals of malformed files."""
import hashlib
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")
TINY = dict(tau=0x1234567890ABCDEF, alpha=1111111111111111111, beta=2222222222222222223)
X1, S1 = 0x5EC12E7_0000_1111_2222_3333_4444_5555_6666_7777, 0xABCDEF0123456789


def _tiny_key(power=3):
    import ptau_writer as pw
    import zkey_oracle
    r1cs = open(os.path.join(G, "circom2_multiplier2.r1cs"), "rb").read()
    secs = pw.sections_oracle(TINY["tau"], TINY["alpha"], TINY["beta"], power)
    return zkey_oracle.zkey_new(r1cs, pw.ptau_bytes(secs)), secs


def test_oracle_export_hashes_to_the_cs_hash_and_parses():
    import bellman_oracle as bo
    import cshash_oracle as co
    from distributed_groth16_b200 import formats
    from oracle import bn254 as o
    zk, secs = _tiny_key()
    s = co.zkey_sections(zk)
    n_vars, n_public, n = struct.unpack_from("<III", s[2], 72)
    buf = bo.export(zk)
    b = formats.parse_bellman(buf)
    assert b.counts == dict(ic=n_public + 1, h=n - 1, l=n_vars - n_public - 1, a=n_vars, b1=n_vars, b2=n_vars)
    assert len(buf) == formats.bellman_size(n_public + 1, n - 1, n_vars - n_public - 1, n_vars) == b.records_offset
    assert hashlib.blake2b(buf[:b.params_end], digest_size=64).digest() == co.cs_hash(zk, co.h_from_tau(secs[2], n))
    assert b.cs_hash == bytes(64) and b.contributions == []
    # the H points are tau^i (tau^n - 1) G1 (delta = 1)
    t = TINY["tau"]
    off, ln = b.spans["h"]
    assert ln == 64 * (n - 1)
    for i in range(n - 1):
        assert buf[off + 64 * i:off + 64 * i + 64] == co.u_g1(o.G1.mul(o.G1_GEN, pow(t, i, o.R) * (pow(t, n, o.R) - 1)))
    assert b.spans["alpha_g1"] == (0, 64) and b.spans["delta_g2"] == (448, 128) and b.spans["ic"][0] == 580


def test_records_parse_into_contributions():
    import bellman_oracle as bo
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase2
    from oracle import bn254 as o
    zk, _ = _tiny_key()
    buf = bo.export(zk)
    resp, h = bo.contribute(buf, X1, o.G1.mul(o.G1_GEN, S1))
    b = formats.parse_bellman(resp)
    assert len(resp) == formats.bellman_size(b.counts["ic"], b.counts["h"], b.counts["l"], b.counts["a"], 1)
    (c,) = b.contributions
    assert c.type == 0 and c.name is None
    rec = resp[b.records_offset:]
    assert phase2.hash_pub_key(c) == rec and phase2.contribution_hash(c) == h
    assert phase2.u_g1(c.delta_after) == resp[b.spans["delta_g1"][0]:b.spans["delta_g1"][0] + 64]
    # everything but delta, H, L and the count is the challenge's
    for part in ("alpha_g1", "beta_g1", "beta_g2", "gamma_g2", "ic", "a", "b1", "b2"):
        off, ln = b.spans[part]
        assert resp[off:off + ln] == buf[off:off + ln], part
    assert resp[b.params_end:b.params_end + 64] == buf[b.params_end:b.params_end + 64]


def test_malformed_files_raise_format_error():
    import bellman_oracle as bo
    from distributed_groth16_b200 import formats
    from oracle import bn254 as o
    zk, _ = _tiny_key()
    resp, _ = bo.contribute(bo.export(zk), X1, o.G1.mul(o.G1_GEN, S1))
    b = formats.parse_bellman(resp)
    off_h = b.spans["h"][0] - 4
    more = resp[:off_h] + struct.pack(">I", b.counts["h"] + 1) + resp[off_h + 4:]
    fewer = resp[:off_h] + struct.pack(">I", b.counts["h"] - 1) + resp[off_h + 4:]
    huge = resp[:off_h] + struct.pack(">I", 1 << 30) + resp[off_h + 4:]
    rc = b.params_end + 64
    records = resp[:rc] + struct.pack(">I", 2) + resp[rc + 4:]
    flag = bytearray(resp)
    flag[b.records_offset] |= 0x80
    big = bytearray(resp)
    big[b.records_offset + 64:b.records_offset + 96] = (o.P).to_bytes(32, "big")
    cases = {"truncated": resp[:-1], "truncated in the header": resp[:300], "trailing bytes": resp + b"\0",
             "H count + 1": more, "H count - 1": fewer, "H count past the end": huge, "record count": records,
             "record flag byte": bytes(flag), "record coordinate >= q": bytes(big), "empty": b""}
    for what, buf in cases.items():
        with pytest.raises(formats.FormatError):
            formats.parse_bellman(buf)
        assert what
    with pytest.raises(formats.FormatError, match="record 0 g1_s"):
        formats.parse_bellman(bytes(big))


def test_bellman_size():
    from distributed_groth16_b200 import formats
    assert formats.bellman_size(0, 0, 0, 0) == 576 + 24 + 68
    assert formats.bellman_size(2, 3, 4, 5, 6) == 576 + 24 + 64 * (2 + 3 + 4 + 10) + 128 * 5 + 68 + 384 * 6
