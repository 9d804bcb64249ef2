"""Blake2b-512 with an exported state: csrc/blake2b.cuh compiled for the host (tests/host/blake2b_host_test.cpp), and the
library's b200zk_blake2b512_* entries (no GPU needed) against hashlib."""
import hashlib
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_blake2b_header_on_host(tmp_path):
    exe = tmp_path / "blake2b_host_test"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tests", "host", "blake2b_host_test.cpp")])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout + out.stderr


def _lib_blake2b():
    from distributed_groth16_b200 import build
    build.build()
    from distributed_groth16_b200.groth16.phase1 import Blake2b512
    return Blake2b512


def test_library_entries_equal_hashlib_small():
    Blake2b512 = _lib_blake2b()
    rng = np.random.default_rng(11)
    for n in range(0, 301):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        h = Blake2b512()
        h.update(data)
        assert h.digest() == hashlib.blake2b(data, digest_size=64).digest(), n


def test_library_entries_equal_hashlib_large_random_splits():
    Blake2b512 = _lib_blake2b()
    rng = np.random.default_rng(12)
    for mb in (1, 3, 10):
        data = rng.integers(0, 256, mb << 20, dtype=np.uint8)
        cuts = np.sort(rng.integers(0, data.size + 1, 37))
        h = Blake2b512()
        lo = 0
        for hi in list(cuts) + [data.size]:
            h.update(data[lo:hi])
            lo = hi
        assert h.digest() == hashlib.blake2b(data.tobytes(), digest_size=64).digest(), mb


def test_export_import_resumes_to_the_same_digest():
    Blake2b512 = _lib_blake2b()
    rng = np.random.default_rng(13)
    data = rng.integers(0, 256, 5000, dtype=np.uint8).tobytes()
    for cut in (0, 1, 127, 128, 129, 256, 4999, 5000):
        h = Blake2b512()
        h.update(data[:cut])
        st = h.state()
        assert len(st) == 216
        r = Blake2b512(st)
        r.update(data[cut:])
        assert r.digest() == hashlib.blake2b(data, digest_size=64).digest(), cut
        # after exactly 128 k bytes the last block stays buffered (c = 128, t = 128 (k - 1))
        if cut and cut % 128 == 0:
            assert int.from_bytes(st[208:212], "little") == 128
            assert int.from_bytes(st[192:200], "little") == cut - 128
            assert st[:128] == data[cut - 128:cut]


def test_invalid_state_is_refused():
    Blake2b512 = _lib_blake2b()
    import pytest
    with pytest.raises(ValueError):
        Blake2b512(bytes(215))
    h = Blake2b512(bytes(216))                # outlen 0: no update / final can produce it
    with pytest.raises(ValueError):
        h.update(b"x")
    with pytest.raises(ValueError):
        h.digest()
