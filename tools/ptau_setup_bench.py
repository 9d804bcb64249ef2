"""Times the setup from a Powers-of-Tau file (snarkjs `zkey new` on the GPU): zkey_from_r1cs end to end (ceremony levels
read from the memory-mapped file, transposes, the points_spmv products, the zkey writer) and the points_spmv kernels
alone (per-kernel CUDA events of the library's profiler, in a separate run), on

  * the reference's sha256 circuit (tests/golden/sha256_circuit.npz), 2^15 domain;
  * a seeded synthetic circuit of 2^20 - 2 constraints with sha256's column skew: per constraint 3.54 A, 2.33 B and 1.44 C
    non-zeros, 17 % of A in the constant wire's column, every other column short; 62 % / 43 % / 99 % of the A / B / C
    coefficients short (v or r - v below 2^64).

The ceremony is synthetic (tests/ptau_writer.py, power = the circuit's); the r1cs is passed parsed, so r1cs parsing is not
in the time.  Prints one JSON line (also written to --out DIR/ptau_setup_bench_<library>.json).
usage: python tools/ptau_setup_bench.py [--reps 3] [--skip-2p20] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

TOXIC = (0x1234567890ABCDEF1234567890ABCDEF, 11111111111111111111, 22222222222222222223)
R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def sha256_r1cs():
    from distributed_groth16_b200 import formats
    s = np.load(os.path.join(ROOT, "tests", "golden", "sha256_circuit.npz"))
    n_wires, n_pub, nc = (int(v) for v in s["dims"])
    return formats.R1CS(n_wires, n_pub, 0, 0, nc, [s[k + "_rows"] for k in "abc"], [s[k + "_cols"] for k in "abc"],
                        [s[k + "_vals"] for k in "abc"])


def synthetic_r1cs(log_m=20, seed=1):
    from distributed_groth16_b200 import formats
    rng = np.random.default_rng(seed)
    nc = (1 << log_m) - 2
    n_vars = nc
    r_limbs = np.array([(R >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)

    def matrix(per_row, col0, short):
        nnz = int(per_row * nc)
        rows = np.sort(rng.integers(0, nc, size=nnz)).astype(np.uint32)
        cols = rng.integers(1, n_vars, size=nnz).astype(np.uint32)
        cols[rng.random(nnz) < col0] = 0
        vals = rng.integers(0, 1 << 63, size=(nnz, 4), dtype=np.uint64)
        vals[:, 3] %= r_limbs[3]                                        # full: below r
        s = rng.random(nnz) < short
        vals[s, 1:] = 0
        neg = s & (rng.random(nnz) < 0.5)                              # r - v for half of the short ones
        lo = vals[neg, 0] >> np.uint64(2)
        vals[neg] = r_limbs
        vals[neg, 0] = r_limbs[0] - lo                                  # r_limbs[0] > 2^61 > lo: no borrow
        return rows, cols, vals

    m = [matrix(3.54, 0.1676, 0.62), matrix(2.33, 0.0012, 0.43), matrix(1.44, 0.0, 0.99)]
    return formats.R1CS(n_vars, 1, 0, n_vars - 2, nc, [x[0] for x in m], [x[1] for x in m], [x[2] for x in m])


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = (x.strip() for x in q.split(","))
        return dict(gpu=name, power_limit=pl, sm_clock_max=clk)
    except Exception as e:            # the numbers are reported without a card name rather than not at all
        return dict(gpu="unknown (%s)" % e)


def run_case(net, name, r1, power, reps, tmp):
    import ptau_writer as pw
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import circom
    nnz = {k: int(len(r1.rows[i])) for i, k in enumerate("abc")}
    t0 = time.perf_counter()
    secs = pw.sections_gpu(net, *TOXIC, power)
    path = pw.write_ptau(os.path.join(tmp, name + ".ptau"), {k: v for k, v in secs.items() if k not in (2, 3)})
    del secs
    t_ptau = time.perf_counter() - t0
    times = []
    with formats.read_ptau(path) as pt:
        circom.zkey_from_r1cs(net, r1, pt)                             # warm-up: module load, NTT plans, MSM workspaces
        for _ in range(reps):
            net.sync(0)
            t0 = time.perf_counter()
            zk = circom.zkey_from_r1cs(net, r1, pt)
            times.append(time.perf_counter() - t0)
        net.profile(True)
        net.profile_reset()
        circom.zkey_from_r1cs(net, r1, pt)
        net.sync(0)
        prof = net.profile_report()
        net.profile(False)
    os.remove(path)
    spmv = {k: v for k, v in prof.items() if k.startswith("points_") or k.startswith("msm_") or k == "xyzz_to_affine"}
    return dict(n_constraints=int(r1.n_constraints), n_vars=int(r1.n_wires), nnz=nnz, ptau_power=power,
                zkey_bytes=len(zk), zkey_new_s=dict(min=min(times), median=float(np.median(times)), reps=reps),
                spmv_kernels_ms=round(sum(v["ms"] for v in spmv.values()), 3), spmv_kernels=spmv,
                synthetic_ptau_write_s=round(t_ptau, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-2p20", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from distributed_groth16_b200 import Net, _native
    net = Net(0)
    net.use_torch_stream(0)
    res = dict(lib=os.path.basename(_native.LIB_PATH), **gpu_info(), cases={})
    with tempfile.TemporaryDirectory() as tmp:
        res["cases"]["sha256"] = run_case(net, "sha256", sha256_r1cs(), 15, a.reps, tmp)
        if not a.skip_2p20:
            res["cases"]["synthetic_2p20"] = run_case(net, "synthetic", synthetic_r1cs(), 20, a.reps, tmp)
    res.update(gpu_info_after=gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ptau_setup_bench_%s.json" % res["lib"].replace(".so", "")), "w") as f:
            f.write(line + "\n")
    net.close()


if __name__ == "__main__":
    main()
