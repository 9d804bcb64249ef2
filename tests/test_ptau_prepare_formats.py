"""The unprepared Powers-of-Tau reader (formats.PTau(prepared=False)) and the streaming writer of prepared files
(formats.PreparedPTauWriter): accept / reject cases and the section table and lengths, with no device work."""
import os
import struct
import sys

import numpy as np
import pytest

from distributed_groth16_b200 import formats

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import artefact_writer as aw  # noqa: E402
import ptau_writer as pw  # noqa: E402


def _s1(power, ceremony_power=None, n8=32, q=aw.Q):
    return struct.pack("<I", n8) + q.to_bytes(n8, "little") + struct.pack("<II", power, power if ceremony_power is None else ceremony_power)


def _secs(power, s7=struct.pack("<I", 0)):
    """Sections 1-7 of a ceremony of this power with distinct filler bytes (the reader and writer never look inside)."""
    secs = {1: _s1(power)}
    for sid, ln in formats.PTau.tau_section_bytes(power).items():
        secs[sid] = bytes([sid]) * ln
    secs[7] = s7
    return secs


def _write(tmp_path, secs, magic=b"ptau", name="u.ptau"):
    return pw.write_ptau(str(tmp_path / name), secs, magic)


@pytest.mark.parametrize("power", [0, 1, 5])
def test_unprepared_reader_accepts_sections_1_to_7(tmp_path, power):
    path = _write(tmp_path, _secs(power))
    with formats.PTau(path, prepared=False) as pt:
        assert pt.power == power
        assert pt.points(2, 0, 1, 8).tobytes() == bytes([2]) * 64
    with pytest.raises(formats.FormatError, match="not prepared"):
        formats.read_ptau(path)


def test_unprepared_reader_accepts_a_prepared_file(tmp_path):
    secs = _secs(2)
    for sid, ln in formats.PTau.lagrange_section_bytes(2).items():
        secs[sid] = bytes(ln)
    path = _write(tmp_path, secs)
    with formats.PTau(path, prepared=False) as pt:
        assert pt.power == 2
    formats.read_ptau(path).close()


@pytest.mark.parametrize("case", ["magic", "n8", "q", "power"] + ["missing%d" % s for s in range(2, 8)] +
                         ["short%d" % s for s in range(2, 7)])
def test_unprepared_reader_rejects(tmp_path, case):
    secs, magic = _secs(3), b"ptau"
    if case == "magic":
        magic = b"zkey"
    elif case == "n8":
        secs[1] = _s1(3, n8=48, q=aw.Q)
    elif case == "q":
        secs[1] = _s1(3, q=aw.R)
    elif case == "power":
        secs[1] = _s1(28)
    elif case.startswith("missing"):
        del secs[int(case[7:])]
    else:
        sid = int(case[5:])
        secs[sid] = secs[sid][:-1]
    path = _write(tmp_path, secs, magic)
    with pytest.raises(formats.FormatError):
        formats.PTau(path, prepared=False)


def _table(buf):
    assert buf[:4] == b"ptau"
    version, nsec = struct.unpack_from("<II", buf, 4)
    off, out = 12, []
    for _ in range(nsec):
        sid, ln = struct.unpack_from("<IQ", buf, off)
        out.append((sid, off + 12, ln))
        off += 12 + ln
    assert off == len(buf)
    return version, out


@pytest.mark.parametrize("power", [0, 1, 3, 6])
def test_writer_section_table_and_lengths(tmp_path, power):
    """11 sections in the order 1, 2-7, 12-15; section 1 restated with ceremonyPower = power; 2-7 byte for byte (including
    a non-empty section 7); each Lagrange level at point 2^k - 1 of its section."""
    secs = _secs(power, s7=struct.pack("<I", 1) + b"contribution record" * 7)
    secs[1] = _s1(power, ceremony_power=power + 4)
    src = _write(tmp_path, secs)
    dst = str(tmp_path / "p.ptau")
    with formats.PTau(src, prepared=False) as pt:
        w = formats.PreparedPTauWriter(dst, pt)
        order = w.levels()
        assert order == [(12, k) for k in range(power + 2)] + [(s, k) for s in (13, 14, 15) for k in range(power + 1)]
        for sid, k in order:
            width = 16 if sid == 13 else 8
            lv = np.full(((1 << k), width), sid * 1000 + k, dtype=np.uint64)
            w.write_level(sid, k, lv)
        w.close()
    buf = open(dst, "rb").read()
    version, table = _table(buf)
    assert version == 1
    assert [sid for sid, _, _ in table] == list(pw.ORDER)
    spans = {sid: (off, ln) for sid, off, ln in table}
    assert buf[spans[1][0]:spans[1][0] + spans[1][1]] == _s1(power)
    for sid in range(2, 8):
        off, ln = spans[sid]
        assert buf[off:off + ln] == secs[sid], sid
    lag = formats.PTau.lagrange_section_bytes(power)
    for sid in (12, 13, 14, 15):
        assert spans[sid][1] == lag[sid]
        width = 16 if sid == 13 else 8
        arr = np.frombuffer(buf, dtype="<u8", count=lag[sid] // 8, offset=spans[sid][0]).reshape(-1, width)
        for k in range(power + (2 if sid == 12 else 1)):
            assert (arr[(1 << k) - 1:(2 << k) - 1] == sid * 1000 + k).all(), (sid, k)
    with formats.read_ptau(dst) as pt:                     # the product reader takes it
        assert pt.power == power and pt.ceremony_power == power


def test_writer_checks_order_length_and_completeness(tmp_path):
    src = _write(tmp_path, _secs(1))
    with formats.PTau(src, prepared=False) as pt:
        w = formats.PreparedPTauWriter(str(tmp_path / "p.ptau"), pt)
        with pytest.raises(ValueError, match="out of order"):
            w.write_level(13, 0, bytes(128))
        with pytest.raises(ValueError, match="bytes"):
            w.write_level(12, 0, bytes(128))
        w.write_level(12, 0, bytes(64))
        with pytest.raises(ValueError, match="incomplete"):
            w.close()
