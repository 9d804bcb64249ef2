"""The circuit hash (csHash) of snarkjs `zkey new`, host side (no GPU): the pure-Python restatement (cshash_oracle)
reproduces the hash snarkjs wrote into the reference's complex-circuit zkey, and its two ways of making the H points
(from section 9 by the Lagrange identity, from the ceremony's tau powers by subtraction) agree."""
import os
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")
TINY = dict(tau=0x1234567890ABCDEF, alpha=1111111111111111111, beta=2222222222222222223)


def test_oracle_reproduces_the_cs_hash_snarkjs_wrote_into_the_reference_zkey():
    """The reference's complex-circuit zkey has no contributions (delta = 1), so its csHash follows from its own
    sections, with H from section 9 by the identity.  About a minute on 8 cores."""
    import artefact_writer as aw
    import cshash_oracle as co
    from oracle import layout
    d = np.load(os.path.join(G, "complex_circuit.zkey.pk.npz"))
    want = np.load(os.path.join(G, "reference_artefacts.npz"))["zkey_sec10"].tobytes()
    assert want[64:] == struct.pack("<I", 0)                  # no contributions
    h = co.h_from_lagrange(layout.arr_to_g1(d["h_query"]))
    assert len(h) == int(d["dims"][2]) - 1 == (1 << 14) - 1
    assert co.cs_hash(aw.write_zkey(d), h) == want[:64]


def test_h_from_section_9_equals_h_from_the_tau_powers_on_the_tiny_circuit():
    """circom2_multiplier2 on power-2 and power-3 ceremonies (domain 4): the identity on the oracle zkey's section 9 gives
    tau^(n+i) G1 - tau^i G1, i < n - 1, point for point -- also at power 2, where the top Lagrange level of the ptau
    writer drops tau^(2n - 1), which only H_(n-1) would need."""
    import ptau_writer as pw
    import zkey_oracle
    import cshash_oracle as co
    from oracle import bn254 as o, layout
    r1cs = open(os.path.join(G, "circom2_multiplier2.r1cs"), "rb").read()
    for power in (2, 3):
        secs = pw.sections_oracle(TINY["tau"], TINY["alpha"], TINY["beta"], power)
        zk = zkey_oracle.zkey_new(r1cs, pw.ptau_bytes(secs))
        n = struct.unpack_from("<I", co.zkey_sections(zk)[2], 80)[0]
        assert n == 4
        h9 = layout.arr_to_g1(np.frombuffer(co.zkey_sections(zk)[9], dtype="<u8").reshape(-1, 8))
        by_identity = co.h_from_lagrange(h9, workers=2)
        by_tau = co.h_from_tau(secs[2], n)
        t = TINY["tau"]
        assert by_identity == by_tau == [o.G1.mul(o.G1_GEN, (pow(t, n + i, o.R) - pow(t, i, o.R)) % o.R)
                                         for i in range(n - 1)]
        assert co.cs_hash(zk, by_identity) == co.cs_hash(zk, by_tau)


def test_h_point_count_is_the_length_prefix():
    from distributed_groth16_b200.groth16 import cshash
    assert [cshash.h_point_count(1 << k) for k in (1, 14, 15, 22)] == [1, (1 << 14) - 1, (1 << 15) - 1, (1 << 22) - 1]
