"""The host half of the native prover (csrc/snarkjs_files.h, built with g++ through tests/host/snarkjs_files_host_test.cpp)
against the Python readers and writers: on well-formed and malformed zkeys and wtns files it accepts exactly what
formats.read_zkey / read_wtns accept, with the same header fields and the same FormatError message, and its JSON equals
formats.write_proof_json / write_public_json.

Where the native reader is stricter, by design: a zkey whose section 1 protocol is not Groth16 (1) is refused by name
(read_zkey never reads section 1), and a file shorter than a section claims is refused (read_zkey only notices when it
reads the missing bytes, so a cut inside section 10, which it never reads, passes there).  The coefficient records are
checked on the device in the library; here the harness applies the same predicate (coef_record_ok) to every record."""
import os
import struct
import subprocess

import numpy as np
import pytest

from distributed_groth16_b200 import formats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q, R = formats.FQ_MODULUS, formats.FR_MODULUS
RS = b"\x1e"


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    exe = tmp_path_factory.mktemp("sjf") / "snarkjs_files_host_test"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-Wall", "-Werror", "-o", str(exe),
                           os.path.join(ROOT, "tests", "host", "snarkjs_files_host_test.cpp")])
    d = tmp_path_factory.mktemp("sjf_in")

    def run(mode, blobs):
        paths = []
        for i, b in enumerate(blobs):
            p = d / ("%s_%d.bin" % (mode, i))
            p.write_bytes(b)
            paths.append(str(p))
        out = subprocess.run([str(exe), mode] + paths, capture_output=True, check=True).stdout
        parts = out.split(RS)
        assert parts[-1] == b"" and len(parts) == len(blobs) + 1
        return [x.decode() for x in parts[:-1]]
    return run


# ---- zkeys ----------------------------------------------------------------------------------------------------------------
def _zkey(n_vars=10, n_public=2, domain=16, nc=5, seed=1) -> formats.ZKey:
    rng = np.random.default_rng(seed)
    pts = lambda n, w: rng.integers(0, 2**63, (n, w), dtype=np.uint64)
    rows = np.concatenate([rng.integers(0, nc, 12), np.arange(nc, nc + n_public + 1)]).astype(np.uint32)
    k = rows.size
    return formats.ZKey(n_vars=n_vars, n_public=n_public, domain_size=domain, alpha_g1=pts(1, 8)[0], beta_g1=pts(1, 8)[0],
                        beta_g2=pts(1, 16)[0], gamma_g2=pts(1, 16)[0], delta_g1=pts(1, 8)[0], delta_g2=pts(1, 16)[0],
                        ic=pts(n_public + 1, 8), a_query=pts(n_vars, 8), b_g1_query=pts(n_vars, 8), b_g2_query=pts(n_vars, 16),
                        l_query=pts(n_vars - n_public - 1, 8), h_query=pts(domain, 8),
                        coef_matrix=rng.integers(0, 2, k).astype(np.uint32), coef_row=rows,
                        coef_col=rng.integers(0, n_vars, k).astype(np.uint32), coef_val_r2=pts(k, 4))


def _split(buf: bytes):
    """-> (preamble, [(sid, payload)]) of a snarkjs container"""
    nsec = struct.unpack_from("<I", buf, 8)[0]
    off, secs = 12, []
    for _ in range(nsec):
        sid, ln = struct.unpack_from("<IQ", buf, off)
        secs.append((sid, buf[off + 12:off + 12 + ln]))
        off += 12 + ln
    return buf[:12], secs


def _join(pre: bytes, secs) -> bytes:
    return pre[:8] + struct.pack("<I", len(secs)) + b"".join(struct.pack("<IQ", sid, len(p)) + p for sid, p in secs)


def _edit(buf: bytes, sid: int, fn) -> bytes:
    pre, secs = _split(buf)
    return _join(pre, [(s, fn(p) if s == sid else p) for s, p in secs])


def _drop(buf: bytes, sid: int) -> bytes:
    pre, secs = _split(buf)
    return _join(pre, [(s, p) for s, p in secs if s != sid])


def _hdr(buf: bytes, off: int, data: bytes) -> bytes:
    return _edit(buf, 2, lambda p: p[:off] + data + p[off + len(data):])


def _records(buf: bytes, k: int, field: int, value: int) -> bytes:
    """record k's field (0 = m, 1 = c, 2 = s) set to value"""
    return _edit(buf, 4, lambda p: p[:4 + 44 * k + 4 * field] + struct.pack("<I", value) + p[4 + 44 * k + 4 * field + 4:])


def _corpus():
    base = formats.write_zkey(_zkey())
    zk = _zkey()
    c = {"valid": base, "valid n_public=0": formats.write_zkey(_zkey(n_public=0, seed=2)),
         "valid all public": formats.write_zkey(_zkey(n_vars=6, n_public=5, seed=3)),
         "valid no records": formats.write_zkey(formats.ZKey(**{**_zkey().__dict__, "coef_matrix": np.zeros(0, np.uint32),
                                                                "coef_row": np.zeros(0, np.uint32), "coef_col": np.zeros(0, np.uint32),
                                                                "coef_val_r2": np.zeros((0, 4), np.uint64)})),
         "bad magic": b"zkez" + base[4:], "bad magic quote": b"z'k\x00" + base[4:],
         "not BN254 q": _hdr(base, 4, (Q + 2).to_bytes(32, "little")),
         "not BN254 r": _hdr(base, 40, (R - 2).to_bytes(32, "little")),
         "not BN254 n8q": _hdr(base, 0, struct.pack("<I", 48)),
         "n_vars = 0": _hdr(base, 72, struct.pack("<I", 0)),
         "n_public + 1 > n_vars": _hdr(base, 76, struct.pack("<I", 10)),
         "n_public = 2^32 - 1": _hdr(base, 76, struct.pack("<I", 0xFFFFFFFF)),
         "domain 12": _hdr(base, 80, struct.pack("<I", 12)),
         "domain 0": _hdr(base, 80, struct.pack("<I", 0)),
         "coefficient section too short": _edit(base, 4, lambda p: struct.pack("<I", struct.unpack_from("<I", p)[0] + 1) + p[4:]),
         "record m = 2": _records(base, 3, 0, 2),
         "record s = n_vars": _records(base, 5, 2, zk.n_vars),
         "record c = domain": _records(base, 0, 1, zk.domain_size),
         "three bad records": _records(_records(_records(base, 9, 2, 77), 4, 0, 5), 11, 1, 1 << 20),
         "protocol 2": _edit(base, 1, lambda p: struct.pack("<I", 2)),
         }
    for sid in range(2, 10):
        c["missing section %d" % sid] = _drop(base, sid)
    for sid in (3, 5, 6, 7, 8, 9):
        c["section %d short" % sid] = _edit(base, sid, lambda p: p[:-8])
    pre, secs = _split(base)
    off = 12
    for sid, p in secs:
        off += 12
        if len(p) > 1:
            c["cut inside section %d" % sid] = base[:off + len(p) // 2]
        off += len(p)
    return c


def _python_zkey(buf):
    try:
        zk = formats.read_zkey(buf)
    except formats.FormatError as e:
        return "ERR " + str(e)
    except Exception as e:                     # noqa: BLE001 -- truncated files fail inside struct / numpy
        return "EXC " + type(e).__name__
    return "OK %d %d %d %d" % (zk.n_vars, zk.n_public, zk.domain_size, zk.coef_row.size)


def test_zkey_headers_and_refusals_match_read_zkey(harness):
    corpus = _corpus()
    got = dict(zip(corpus, harness("zkey", list(corpus.values()))))
    rec_msg = "zkey coefficient section: matrix index > 1, signal index >= n_vars or constraint index >= domain size"
    for name, buf in corpus.items():
        py, c = _python_zkey(buf), got[name]
        if name == "protocol 2":
            assert py.startswith("OK") and c.startswith("ERR zkey protocol 2 is not Groth16 (1)"), (py, c)
        elif name.startswith("cut inside section"):
            assert c.startswith("ERR zkey section") and "runs past the end of the file" in c, (name, c)
            assert py.startswith("EXC") or name == "cut inside section 10", (name, py)
        elif py == "ERR " + rec_msg:
            ok, n_vars, n_public, dom, ncoef, nbad, first = c.split(" ")
            assert ok == "OK" and int(nbad) > 0, (name, c)
            sec4 = dict(_split(buf)[1])[4]
            rec = np.frombuffer(sec4, dtype=np.dtype([("m", "<u4"), ("c", "<u4"), ("s", "<u4"), ("v", "<u8", (4,))]),
                                count=int(ncoef), offset=4)
            badm = (rec["m"] > 1) | (rec["s"] >= int(n_vars)) | (rec["c"] >= int(dom))
            assert (int(nbad), int(first)) == (int(badm.sum()), int(np.flatnonzero(badm)[0])), (name, c)
        elif py.startswith("OK"):
            assert c.startswith(py + " 0 "), (name, py, c)
        else:
            assert py.startswith("ERR"), (name, py)
            assert c == py, (name, py, c)
    assert got["three bad records"].split(" ")[5:] == ["3", "4"]


# ---- wtns -----------------------------------------------------------------------------------------------------------------
def _wtns(values, n8=32, prime=R, count=None, data_cut=0) -> bytes:
    s1 = struct.pack("<I", n8) + prime.to_bytes(n8, "little") + struct.pack("<I", len(values) if count is None else count)
    s2 = b"".join(int(v).to_bytes(32, "little") for v in values)
    s2 = s2[:len(s2) - data_cut]
    return b"wtns" + struct.pack("<II", 2, 2) + struct.pack("<IQ", 1, len(s1)) + s1 + struct.pack("<IQ", 2, len(s2)) + s2


def test_wtns_headers_and_refusals_match_read_wtns(harness):
    vals = [1, 5, R - 1, 0, 123456789]
    base = _wtns(vals)
    corpus = {"valid": base, "empty witness": _wtns([]), "bad magic": b"wtnz" + base[4:], "n8 = 48": _wtns(vals, n8=48),
              "prime q": _wtns(vals, prime=Q), "data section too short": _wtns(vals, data_cut=1),
              "count above the data": _wtns(vals, count=6), "count below the data": _wtns(vals, count=4),
              "cut inside the data": base[:-40], "cut inside section 1": base[:30],
              "missing section 2": base[:12 + 12 + 40].replace(struct.pack("<II", 2, 2), struct.pack("<II", 2, 1), 1)}
    got = dict(zip(corpus, harness("wtns", list(corpus.values()))))
    for name, buf in corpus.items():
        try:
            py = "OK %d" % formats.read_wtns(buf).shape[0]
        except formats.FormatError as e:
            py = "ERR " + str(e)
        except Exception as e:                 # noqa: BLE001
            py = "EXC " + type(e).__name__
        if py.startswith("EXC"):
            assert got[name].startswith("ERR wtns"), (name, py, got[name])
        else:
            assert got[name] == py, (name, py, got[name])


# ---- JSON ---------------------------------------------------------------------------------------------------------------
def _be(v):
    return int(v).to_bytes(32, "big")


def _enc_g1(p):
    return b"\x40" + bytes(63) if p is None else _be(p[0]) + _be(p[1])


def _enc_g2(p):
    return b"\x40" + bytes(127) if p is None else _be(p[0][1]) + _be(p[0][0]) + _be(p[1][1]) + _be(p[1][0])


def test_json_writer_equals_the_python_writer(harness):
    rng = np.random.default_rng(7)
    rand = lambda: int.from_bytes(rng.bytes(32), "little") % Q
    specials = [0, 1, Q - 1]
    proofs = []
    for k in range(40):
        pick = lambda: specials[rng.integers(0, 3)] if rng.random() < 0.3 else rand()
        a = None if k % 7 == 1 else (pick(), pick())
        b = None if k % 7 == 2 else ((pick(), pick()), (pick(), pick()))
        c = None if k % 7 == 3 else (pick(), pick())
        proofs.append(formats.SnarkjsProof(a, b, c))
    proofs.append(formats.SnarkjsProof(None, None, None))
    proofs.append(formats.SnarkjsProof((Q - 1, Q - 1), ((Q - 1, Q - 1), (Q - 1, Q - 1)), (Q - 1, Q - 1)))
    got = harness("proof", [_enc_g1(p.pi_a) + _enc_g1(p.pi_c) + _enc_g2(p.pi_b) for p in proofs])
    for p, g in zip(proofs, got):
        assert g == formats.write_proof_json(p)
    assert max(len(g) for g in got) + 1 == 810                 # B200ZK_PROOF_JSON_MAX

    publics = [[], [0], [1], [R - 1], [10 ** 76, 2 * 10 ** 76 - 1, 10 ** 76 - 1, 10 ** 57, 10 ** 19, 10 ** 19 - 1], [0, 1, R - 1] + [int.from_bytes(rng.bytes(32), "little") % R for _ in range(30)],
               [10 ** k for k in range(77)], [R - 1] * 5]
    got = harness("public", [b"".join(int(v).to_bytes(32, "little") for v in vals) for vals in publics])
    for vals, g in zip(publics, got):
        assert g == formats.write_public_json(vals)
        assert len(g) + 1 <= 3 + 82 * len(vals)                   # B200ZK_PUBLIC_JSON_MAX(n_public)
    assert len(got[0]) + 1 == 3 and len(got[-1]) + 1 == 3 + 82 * 5   # reached with no signal and with 77-digit signals
