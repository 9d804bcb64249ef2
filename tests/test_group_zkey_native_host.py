"""`b200zk-prove --devices` without a GPU: argument parsing and file mapping come before any CUDA call, so every usage error
exits 2 with the usage line and a missing file exits 1 naming it, and neither writes an output file."""
import os
import subprocess

import pytest


@pytest.fixture(scope="module")
def exe():
    from distributed_groth16_b200 import build
    build.build()
    return build.PROVE_EXE


@pytest.mark.parametrize("args", [
    ["--device", "0", "--devices", "0,1"],
    ["--devices", "0", "--device", "0"],
    ["--devices", ""],
    ["--devices", ","],
    ["--devices", "0,"],
    ["--devices", ",0"],
    ["--devices", "0,,1"],
    ["--devices", "a,b"],
    ["--devices", "0;1"],
    ["--devices", "-1,0"],
    ["--devices", "0,1,2"],
    ["--devices", "0,1,2,3,4,5"],
    ["--devices", "0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0"],
    ["--devices"],
])
def test_usage_errors_exit_2(exe, tmp_path, args):
    paths = [str(tmp_path / f) for f in ("k.zkey", "w.wtns", "p.json", "u.json")]
    r = subprocess.run([exe] + args + paths, capture_output=True, text=True)
    assert r.returncode == 2, (args, r.returncode, r.stderr)
    assert r.stderr.startswith("usage: b200zk-prove [--device N | --devices"), r.stderr
    assert os.listdir(tmp_path) == []


@pytest.mark.parametrize("devices", ["0", "0,0", "0,1,2,3", "7,6,5,4,3,2,1,0"])
def test_missing_zkey_exits_1_and_names_it(exe, tmp_path, devices):
    (tmp_path / "w.wtns").write_bytes(b"wtns")
    missing = str(tmp_path / "missing.zkey")
    r = subprocess.run([exe, "--devices", devices, missing, str(tmp_path / "w.wtns"), str(tmp_path / "p.json"), str(tmp_path / "u.json")],
                       capture_output=True, text=True)
    assert r.returncode == 1, r.stderr
    assert missing in r.stderr and "No such file" in r.stderr, r.stderr
    assert sorted(os.listdir(tmp_path)) == ["w.wtns"]
