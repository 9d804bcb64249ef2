"""Phase-2 ceremony, host side (no GPU): section 10 of a zkey (formats.read_mpc_params / mpc_params_bytes), the ChaCha
stream that hash-to-G2 and the beacon draw from, and the uncompressed point encoding the transcript hashes."""
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
G = os.path.join(HERE, "golden")


def _zkey_with(sec10: bytes) -> bytes:
    return b"zkey" + struct.pack("<II", 1, 1) + struct.pack("<IQ", 10, len(sec10)) + sec10


def _records():
    from distributed_groth16_b200 import formats
    rng = np.random.default_rng(5)
    pts = lambda w: rng.integers(0, 1 << 63, size=w, dtype=np.uint64)
    c1 = formats.Contribution(delta_after=pts(8), g1_s=pts(8), g1_sx=pts(8), g2_spx=pts(16), transcript=bytes(range(64)),
                              type=0, name="first contributor")
    c2 = formats.Contribution(delta_after=pts(8), g1_s=np.zeros(8, np.uint64), g1_sx=pts(8), g2_spx=pts(16),
                              transcript=bytes(64), type=0)
    c3 = formats.Contribution(delta_after=pts(8), g1_s=pts(8), g1_sx=pts(8), g2_spx=pts(16), transcript=b"\xab" * 64,
                              type=1, name="Final Beacon β", num_iterations_exp=10,
                              beacon_hash=bytes.fromhex("0102030405060708090a0b0c0d0e0f101112131415161718191a1b1c1d1e1f"))
    return formats.MPCParams(cs_hash=bytes(range(100, 164)), contributions=[c1, c2, c3])


def test_reference_section_10_reads_and_writes_back():
    from distributed_groth16_b200 import formats
    sec = np.load(os.path.join(G, "reference_artefacts.npz"))["zkey_sec10"].tobytes()
    mpc = formats.read_mpc_params(_zkey_with(sec))
    assert mpc.cs_hash == sec[:64] and len(mpc.cs_hash) == 64 and any(mpc.cs_hash)
    assert mpc.contributions == []
    assert formats.mpc_params_bytes(mpc) == sec


def test_records_with_a_name_and_beacon_parameters_round_trip():
    from distributed_groth16_b200 import formats
    mpc = _records()
    sec = formats.mpc_params_bytes(mpc)
    back = formats.read_mpc_params(_zkey_with(sec))
    assert back.cs_hash == mpc.cs_hash and len(back.contributions) == 3
    for a, b in zip(mpc.contributions, back.contributions):
        for f in ("delta_after", "g1_s", "g1_sx", "g2_spx"):
            assert (np.asarray(getattr(a, f)) == getattr(b, f)).all(), f
        assert (a.transcript, a.type, a.name, a.num_iterations_exp, a.beacon_hash) == \
               (b.transcript, b.type, b.name, b.num_iterations_exp, b.beacon_hash)
    assert formats.mpc_params_bytes(back) == sec
    # the parameter stream as written: name (key 1), then numIterationsExp (2) and beaconHash (3)
    c3 = back.contributions[2]
    name = c3.name.encode("utf-8")
    assert sec.endswith(struct.pack("<II", 1, 2 + len(name) + 4 + 31) + bytes([1, len(name)]) + name +
                        bytes([2, 10, 3, 31]) + c3.beacon_hash)


def test_malformed_section_10_is_rejected():
    from distributed_groth16_b200 import formats
    sec = formats.mpc_params_bytes(_records())
    first_params = 68 + 392                      # offset of the first record's parameter stream
    cases = {
        "truncated csHash": sec[:40],
        "truncated record": sec[:68 + 200],
        "truncated parameters": sec[:first_params + 5],
        "count past the section": sec[:64] + struct.pack("<I", 1000) + sec[68:],
        "unknown key": sec[:first_params] + b"\x07" + sec[first_params + 1:],
        "name past its parameters": sec[:first_params] + b"\x01\x7f" + sec[first_params + 2:],
    }
    # an over-long name: 65 bytes in a stream that is otherwise well-formed
    long_rec = sec[:64] + struct.pack("<I", 1) + sec[68:68 + 384] + struct.pack("<II", 0, 67) + b"\x01\x41" + b"n" * 65
    cases["name over 64 bytes"] = long_rec
    for what, bad in cases.items():
        with pytest.raises(formats.FormatError):
            formats.read_mpc_params(_zkey_with(bad))
            pytest.fail(what)
    with pytest.raises(formats.FormatError):
        formats.read_mpc_params(b"zkey" + struct.pack("<II", 1, 0))            # no section 10
    mpc = _records()
    mpc.contributions[0].name = "x" * 65
    with pytest.raises(formats.FormatError):
        formats.mpc_params_bytes(mpc)


def test_chacha_matches_rfc7539_chacha20():
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms
    from distributed_groth16_b200.groth16.phase2 import ChaCha
    for seed in ([0] * 8, [0x01234567, 0x89ABCDEF, 0xDEADBEEF, 0, 1, 2, 0xFFFFFFFF, 0x80000000]):
        ks = Cipher(algorithms.ChaCha20(struct.pack("<8I", *seed), bytes(16)), mode=None).encryptor().update(bytes(64 * 5))
        rng = ChaCha(seed)
        assert [rng.next_u32() for _ in range(80)] == list(struct.unpack("<80I", ks))
    h = bytes(range(32, 96))
    ks = Cipher(algorithms.ChaCha20(struct.pack("<8I", *struct.unpack(">8I", h[:32])), bytes(16)),
                mode=None).encryptor().update(bytes(64))
    rng = ChaCha.from_hash(h)
    w = struct.unpack("<16I", ks)
    assert rng.next_u64() == (w[0] << 32) | w[1] and rng.next_bool() == bool(w[2] & 1)


def test_field_from_rng_masks_and_rejects():
    from distributed_groth16_b200.groth16.phase2 import ChaCha, field_from_rng
    from distributed_groth16_b200.formats import FQ_MODULUS, FR_MODULUS
    ref, rng = ChaCha([7] * 8), ChaCha([7] * 8)
    for mod in (FR_MODULUS, FQ_MODULUS) * 4:
        while True:
            v = sum(ref.next_u64() << (64 * i) for i in range(4)) & ((1 << 254) - 1)
            if v < mod:
                break
        assert field_from_rng(rng, mod) == v


def test_uncompressed_encoding_of_the_generators_and_infinity():
    from oracle import bn254 as o, layout
    from distributed_groth16_b200.groth16.phase2 import u_g1, u_g2
    assert u_g1(layout.g1_to_arr([(1, 2)])) == bytes(31) + b"\x01" + bytes(31) + b"\x02"
    assert u_g1(np.zeros(8, np.uint64)) == b"\x40" + bytes(63)
    assert u_g2(np.zeros(16, np.uint64)) == b"\x40" + bytes(127)
    x0 = 0x1800DEEF121F1E76426A00665E5C4479674322D4F75EDADD46DEBD5CD992F6ED
    x1 = 0x198E9393920D483A7260BFB731FB5D25F1AA493335A9E71297E485B7AEF312C2
    y0 = 0x12C85EA5DB8C6DEB4AAB71808DCB408FE3D1E7690C43D37B4CE6CC0166FA7DAA
    y1 = 0x090689D0585FF075EC9E99AD690C3395BC4B313370B38EF355ACDADCD122975B
    assert o.G2_GEN == ((x0, x1), (y0, y1))
    want = bytes.fromhex(
        "198e9393920d483a7260bfb731fb5d25f1aa493335a9e71297e485b7aef312c2"
        "1800deef121f1e76426a00665e5c4479674322d4f75edadd46debd5cd992f6ed"
        "090689d0585ff075ec9e99ad690c3395bc4b313370b38ef355acdadcd122975b"
        "12c85ea5db8c6deb4aab71808dcb408fe3d1e7690c43d37b4ce6cc0166fa7daa")
    assert u_g2(layout.g2_to_arr([o.G2_GEN])) == want


def test_g2_cofactor_clears_the_twist():
    """The twist's order is r (2q - r): hash-to-G2 multiplies by 2q - r, and the result lies in the order-r subgroup."""
    from oracle import bn254 as o
    from distributed_groth16_b200.groth16.phase2 import G2_COFACTOR, ChaCha
    import phase2_oracle
    assert G2_COFACTOR == 2 * o.P - o.R
    pt = phase2_oracle.from_rng(ChaCha([3] * 8), g2=True)
    assert pt is not None and o.G2.is_on_curve(pt)
    assert o.G2.from_jac(o.G2.jac_mul(o.G2.to_jac(pt), o.R)) is None
