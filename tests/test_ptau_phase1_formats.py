"""Phase-1 ceremony files on the host: section-7 records, the streaming writer, `new` and the first challenge hash against
tests/phase1_oracle.py, the oracle's own Blake2b, and the RNG position _from_rng leaves behind."""
import hashlib
import struct

import numpy as np
import pytest

from distributed_groth16_b200 import formats
from distributed_groth16_b200.groth16 import phase2


def _pt(rng, w):
    return rng.integers(0, 1 << 63, w, dtype=np.uint64)


def _record(rng, **kw):
    key = {k: {"g1_s": _pt(rng, 8), "g1_sx": _pt(rng, 8), "g2_spx": _pt(rng, 16)} for k in ("tau", "alpha", "beta")}
    return formats.PTauContribution(tau_g1=_pt(rng, 8), tau_g2=_pt(rng, 16), alpha_g1=_pt(rng, 8), beta_g1=_pt(rng, 8),
                                    beta_g2=_pt(rng, 16), key=key, partial_hash=rng.bytes(216), next_challenge=rng.bytes(64),
                                    **kw)


def _same(a, b):
    for f in ("tau_g1", "tau_g2", "alpha_g1", "beta_g1", "beta_g2"):
        assert (getattr(a, f) == getattr(b, f)).all(), f
    for k in ("tau", "alpha", "beta"):
        for f in ("g1_s", "g1_sx", "g2_spx"):
            assert (a.key[k][f] == b.key[k][f]).all(), (k, f)
    for f in ("partial_hash", "next_challenge", "type", "name", "num_iterations_exp", "beacon_hash"):
        assert getattr(a, f) == getattr(b, f), f


def test_section7_round_trip():
    rng = np.random.default_rng(1)
    recs = [_record(rng), _record(rng, name="alice"), _record(rng, type=1, name="ßeacon", num_iterations_exp=10,
                                                              beacon_hash=bytes(range(32))),
            _record(rng, type=1, num_iterations_exp=63, beacon_hash=b"")]
    sec = formats.ptau_contributions_bytes(recs)
    assert struct.unpack_from("<I", sec)[0] == 4
    back = formats.parse_ptau_contributions(sec)
    assert len(back) == 4
    for a, b in zip(recs, back):
        _same(a, b)
    assert formats.ptau_contributions_bytes(back) == sec
    assert formats.parse_ptau_contributions(formats.ptau_contributions_bytes([])) == []
    # layout: the first record's tauG1 right after the count, its partialHash after the 152 point limbs
    assert sec[4:68] == recs[0].tau_g1.astype("<u8").tobytes()
    assert sec[4 + 1216:4 + 1432] == recs[0].partial_hash
    assert struct.unpack_from("<II", sec, 4 + 1496) == (0, 0)


def test_section7_rejects():
    rng = np.random.default_rng(2)
    good = formats.ptau_contributions_bytes([_record(rng, name="x")])
    cases = {
        "short count": b"\x01\x00",
        "count past the section": struct.pack("<I", 2) + good[4:],
        "short record": good[:4] + good[4:1000],
        "parameters past the record": good[:-1],
        "unknown key": good[:4 + 1500] + struct.pack("<I", 2) + bytes([9, 0]),
        "over-long name": good[:4 + 1500] + struct.pack("<I", 67) + bytes([1, 65]) + b"a" * 65,
        "name not UTF-8": good[:4 + 1500] + struct.pack("<I", 3) + bytes([1, 1, 0xFF]),
    }
    for what, sec in cases.items():
        with pytest.raises(formats.FormatError):
            formats.parse_ptau_contributions(sec)
            pytest.fail(what)
    with pytest.raises(formats.FormatError):
        formats.ptau_contributions_bytes([_record(rng, name="n" * 65)])
    with pytest.raises(formats.FormatError):
        formats.ptau_contributions_bytes([_record(rng, type=1)])


def test_writer_section_table_and_lengths(tmp_path):
    power = 3
    p = str(tmp_path / "w.ptau")
    lens = formats.PTau.tau_section_bytes(power)
    with formats.PTauWriter(p, power) as w:
        for sid in (2, 3, 4, 5, 6):
            data = bytes([sid]) * lens[sid]
            w.write(sid, data[:7])
            w.write(sid, data[7:])
        with pytest.raises(ValueError):
            w.write(6, b"x")                                   # past the section's length
        sec7 = formats.ptau_contributions_bytes([])
        w.write_contributions(sec7)
        w.close()
    buf = open(p, "rb").read()
    assert buf[:4] == b"ptau" and struct.unpack_from("<II", buf, 4) == (1, 7)
    off, table = 12, []
    while off < len(buf):
        sid, ln = struct.unpack_from("<IQ", buf, off)
        table.append((sid, ln))
        if sid == 1:
            assert buf[off + 12:off + 12 + ln] == struct.pack("<I", 32) + formats.FQ_MODULUS.to_bytes(32, "little") + \
                struct.pack("<II", power, power)
        elif sid <= 6:
            assert buf[off + 12:off + 12 + ln] == bytes([sid]) * ln
        off += 12 + ln
    assert table == [(1, 44)] + [(sid, lens[sid]) for sid in (2, 3, 4, 5, 6)] + [(7, 4)]
    with formats.PTau(p, prepared=False) as pt:
        assert (pt.power, pt.ceremony_power) == (power, power)


def test_writer_refuses_out_of_order_and_short(tmp_path):
    p = str(tmp_path / "bad.ptau")
    w = formats.PTauWriter(p, 2)
    with pytest.raises(ValueError):
        w.write(3, b"x")                                       # section 2 first
    w.write(2, b"x" * 64)
    with pytest.raises(ValueError):
        w.write(3, b"x")                                       # section 2 is not complete
    with pytest.raises(ValueError):
        w.write_contributions(b"\x00" * 4)
    with pytest.raises(ValueError):
        w.close()
    with pytest.raises(ValueError):
        formats.PTauWriter(p, 0)
    with pytest.raises(ValueError):
        formats.PTauWriter(p, 28)


def test_ptau_preamble_bytes():
    """Section 1 of both writers comes from ptau_preamble: magic, version, section count, (n8, q, power, power)."""
    assert formats.ptau_preamble(11, 5) == b"ptau" + struct.pack("<II", 1, 11) + struct.pack("<IQ", 1, 44) + \
        struct.pack("<I", 32) + formats.FQ_MODULUS.to_bytes(32, "little") + struct.pack("<II", 5, 5)


@pytest.mark.parametrize("power", [1, 2, 3])
def test_new_equals_the_oracle(tmp_path, power):
    import phase1_oracle
    from distributed_groth16_b200.groth16 import phase1
    p = str(tmp_path / "new.ptau")
    phase1.new(p, power)
    assert open(p, "rb").read() == phase1_oracle.new(power)


@pytest.mark.parametrize("power", [1, 2, 5])
def test_first_challenge_hash_equals_the_oracle(power):
    import phase1_oracle
    from distributed_groth16_b200.groth16 import phase1
    assert phase1.first_challenge_hash(power) == phase1_oracle.first_challenge_hash(power)


def test_oracle_blake2b_against_hashlib():
    import phase1_oracle
    rng = np.random.default_rng(3)
    for n in (0, 1, 127, 128, 129, 256, 300):
        data = rng.bytes(n)
        h = phase1_oracle.Blake2b()
        h.update(data[:n // 3])
        h = phase1_oracle.Blake2b.from_state(h.state())
        h.update(data[n // 3:])
        assert h.digest() == hashlib.blake2b(data, digest_size=64).digest(), n


def test_host_compressed_encoding_against_the_oracle():
    import phase1_oracle
    from oracle import bn254 as o, layout
    from distributed_groth16_b200.groth16 import phase1
    for k in (1, 2, 3, 12345, o.R - 1):
        p1, p2 = o.G1.mul(o.G1_GEN, k), o.G2.mul(o.G2_GEN, k)
        assert phase1.c_g1(layout.g1_to_arr([p1])[0]) == phase1_oracle.c_g1(p1)
        assert phase1.c_g2(layout.g2_to_arr([p2])[0]) == phase1_oracle.c_g2(p2)
    assert phase1.c_g1(np.zeros(8, dtype=np.uint64)) == phase1_oracle.c_g1(None)
    assert phase1.c_g2(np.zeros(16, dtype=np.uint64)) == phase1_oracle.c_g2(None)


def test_from_rng_leaves_the_chacha_where_one_at_a_time_does(monkeypatch):
    """phase2._from_rng decodes 16 candidates per device call; afterwards the RNG must stand right after the accepted
    candidate, as in a one-candidate-at-a-time restatement (phase2_oracle.from_rng).  The device decompression is
    replaced by the oracle's here, so the check runs without a GPU."""
    import torch
    import phase2_oracle
    from oracle import bn254 as o, layout

    class FakeNet:
        _h = None

        def _dev(self):
            return torch.device("cpu")

    class FakeLib:
        @staticmethod
        def b200zk_points_decompress_dev(h, sid, g2, data_ptr, n, check, out_ptr, bad):
            w = 64 if g2 else 32
            raw = ctypes_string(data_ptr.value, n * w)
            pts = []
            for i in range(n):
                try:
                    pts.append((o.g2_decompress if g2 else o.g1_decompress)(raw[w * i:w * i + w]))
                except ValueError:
                    pts.append(None)
            arr = (layout.g2_to_arr if g2 else layout.g1_to_arr)(pts)
            import ctypes
            ctypes.memmove(out_ptr.value, arr.ctypes.data, arr.nbytes)
            return 0

    def ctypes_string(ptr, n):
        import ctypes
        return ctypes.string_at(ptr, n)

    net = FakeNet()
    net._lib = FakeLib()
    monkeypatch.setattr(phase2, "_scale_one", lambda net, p, k, g2=False: p)
    for seed in range(6):
        a = phase2.ChaCha([seed, 1, 2, 3, 4, 5, 6, 7])
        b = phase2.ChaCha([seed, 1, 2, 3, 4, 5, 6, 7])
        for _ in range(3):
            got = phase2._from_rng(net, a, g2=False)
            want = phase2_oracle.from_rng(b, g2=False)
            assert (got == layout.g1_to_arr([want])[0]).all()
        assert [a.next_u32() for _ in range(40)] == [b.next_u32() for _ in range(40)]
