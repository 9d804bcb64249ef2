"""csrc/glv.cuh (the GLV scalar split of the G1 / G2 MSM and of points_scale) compiled for the host: for every k the split
must satisfy k1 + lambda k2 = k (mod r) and |k1|, |k2| < 2^127 -- the MSM's GLV windows (Wh c >= 128) and the width-5 NAF
of points_scale are sized for that bound -- and equal the Python restatement in tests/dlog_oracle.py bit for bit.

Inputs: the edges 0, 1, r - 1, lambda, r - lambda and j r / N, then 2^20 + 10^6 uniform scalars; the largest |k1| and |k2|
seen over all of them (about 2^126.1) are reported and held to the bound."""
import os
import subprocess

import numpy as np

from oracle import bn254 as o

import dlog_oracle as dl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _scalars():
    lam = dl.LAMBDA
    edges = [0, 1, 2, o.R - 1, o.R - 2, lam, o.R - lam, lam - 1, lam + 1, (o.R - 1) // 2, (o.R + 1) // 2, (1 << 253) - 1, 1 << 253]
    edges += [j * o.R // 4096 for j in range(4096)] + [(j * o.R // 4096 + 1) % o.R for j in range(4096)]
    rng = np.random.default_rng(2026)
    n = (1 << 20) + 10 ** 6
    raw = rng.integers(0, 1 << 63, size=(n, 4), dtype=np.int64).astype(np.uint64) << np.uint64(1)
    raw |= rng.integers(0, 2, size=(n, 4), dtype=np.int64).astype(np.uint64)
    raw[:, 3] &= np.uint64((1 << 62) - 1)                       # < 2^254 < 2r
    rnd = [int.from_bytes(row.tobytes(), "little") % o.R for row in raw]
    return edges + rnd


def test_glv_split_on_the_host(tmp_path):
    ks = _scalars()
    n = len(ks)
    blob = np.array([n], dtype="<u8").tobytes() + b"".join(k.to_bytes(32, "little") for k in ks)
    (tmp_path / "in.bin").write_bytes(blob)
    exe = tmp_path / "glv_host_test"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.check_call([cxx, "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tests", "host", "glv_host_test.cpp")])
    r = subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    out = np.fromfile(tmp_path / "out.bin", dtype="<u4").reshape(n, 10)
    k1abs = out[:, 0:4].astype(np.uint64)
    k2abs = out[:, 4:8].astype(np.uint64)
    # both halves < 2^127: the top bit of limb 3 is clear
    assert not (out[:, 3] >> 31).any() and not (out[:, 7] >> 31).any()
    big = lambda a: [int(a[i, 0]) | int(a[i, 1]) << 32 | int(a[i, 2]) << 64 | int(a[i, 3]) << 96 for i in range(a.shape[0])]
    a1, a2 = big(k1abs), big(k2abs)
    bad = []
    best1 = best2 = (0, 0)
    for i, k in enumerate(ks):
        k1 = -a1[i] if out[i, 8] else a1[i]
        k2 = -a2[i] if out[i, 9] else a2[i]
        if (k1 + dl.LAMBDA * k2 - k) % o.R or (k1, k2) != dl.glv_decompose(k) or (k1 == 0 and out[i, 8]) or (k2 == 0 and out[i, 9]):
            bad.append(k)
        best1 = max(best1, (a1[i], k))
        best2 = max(best2, (a2[i], k))
    assert not bad, "split wrong for %d scalars, first %#x" % (len(bad), bad[0])
    # the extremes found by the search: still below 2^127, and the mirror agrees with the device code there too
    assert best1[0] < 1 << 127 and best2[0] < 1 << 127
    assert best1[0] >= 1 << 125 and best2[0] >= 1 << 125                 # the search did reach the large halves
    for _, k in (best1, best2):
        k1, k2 = dl.glv_decompose(k)
        assert (k1 + dl.LAMBDA * k2 - k) % o.R == 0 and max(abs(k1), abs(k2)) < 1 << 127
