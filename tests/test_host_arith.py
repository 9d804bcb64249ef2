"""b200zk_test_arith's op bodies (csrc/selftest.cu: fp.cuh, codec.cuh, pairing.cuh, glv.cuh, ec.cuh) compiled for the host with
g++ and run over the whole operand corpus of tests/arith_oracle.py, record for record against the big-integer answers.
The same bodies run on the device in tests/test_gpu_arith_exact.py; this run needs no GPU and validates the corpus and the
references first.  Device-only ops (the root of unity, quad_ops) are left to the GPU test."""
import os
import subprocess

import numpy as np
import pytest

import arith_oracle as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = tmp_path_factory.mktemp("arith_exe") / "arith_host_test"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-o", str(path), os.path.join(ROOT, "tests", "host", "arith_host_test.cpp")])
    return path


def test_record_sizes_match_the_device_table(exe):
    """Every op code and record size of tests/arith_oracle.py is the one selftest.cu's arith_words gives, device-only ops
    (the root of unity, quad_ops) included, and selftest.cu knows no op the oracle lacks."""
    r = subprocess.run([str(exe), "--table"], capture_output=True, text=True, check=True)
    table = {int(op): (int(i), int(o)) for op, i, o in (line.split() for line in r.stdout.splitlines())}
    assert table == {op.code: (op.n_in, op.n_out) for op in A.OPS.values()}


@pytest.fixture(scope="module")
def host_out(tmp_path_factory, exe):
    tmp = tmp_path_factory.mktemp("arith")
    names = [n for n, op in A.OPS.items() if not op.device_only]
    C = A.corpus()
    blob = [np.array([len(names)], dtype="<u8").tobytes()]
    for n in names:
        op = A.OPS[n]
        recs = C[n]
        blob.append(np.array([op.code, len(recs), op.n_in], dtype="<u8").tobytes())
        blob.append(np.array([r for _, r in recs], dtype="<u8").tobytes())
    (tmp / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([str(exe), str(tmp / "in.bin"), str(tmp / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    flat = np.fromfile(tmp / "out.bin", dtype="<u8")
    out, pos = {}, 0
    for n in names:
        op = A.OPS[n]
        cnt = len(C[n]) * op.n_out
        out[n] = flat[pos:pos + cnt].reshape(-1, op.n_out)
        pos += cnt
    assert pos == flat.size
    return out


@pytest.mark.parametrize("name", [n for n, op in A.OPS.items() if not op.device_only])
def test_host_arith_exact(host_out, name):
    bad = A.mismatches(name, host_out[name])
    assert not bad, "%d of %d records wrong, first:\n%s" % (len(bad), len(host_out[name]), "\n".join(bad[:3]))
