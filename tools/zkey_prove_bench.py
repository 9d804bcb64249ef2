"""snarkjs `groth16 prove` from a .zkey and a .wtns, native path against Python path, per size:

  cmd_s         b200zk-prove as a process (context, load without tables, one proof, both JSON files), wall time
  load_*_s      ZKeyProver(...) with the automatic table policy / without tables, wall time
  csr_gpu_ms    the load's CSR kernels (coefficient check, histogram, scan, scatter), summed CUDA-event times
  csr_numpy_ms  numpy coo_to_csr of both matrices of the same coefficient section (circom.load_zkey's host step)
  prove_s       one proof from a loaded handle (automatic tables), median of --reps
  python_s      circom.groth16_prove (read_zkey, coo_to_csr, key upload with tables, proof, JSON), one call

The keys' points come from Net.generate_g1 / generate_g2, so every point's discrete log is known (tests/dlog_oracle.py
base_logs, the KeySpec keys of the tests); the circuit is nc = m - 4 constraints with Poisson(2) terms per row over n_vars = m / 2
variables, 3 public inputs, and a random witness.  The zkey is written by formats.write_zkey, the same layout as
tests/artefact_writer.write_zkey, whose one Python step per coefficient record would take minutes at 2^22 (16.8 M records).
Every path must give the same proof.json for the same (r, s).

  python tools/zkey_prove_bench.py --log-m 16,18,20,22 --reps 5 --out /tmp/zkey_prove_bench.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [l.strip() for l in q.stdout.strip().splitlines()]


def below_r(rng, n):
    v = rng.integers(0, 1 << 64, (n, 4), dtype=np.uint64)
    v[:, 3] %= np.uint64(R >> 192)
    return v


def files(net, log_m, seed):
    """-> (zkey bytes, wtns bytes)"""
    import struct
    from distributed_groth16_b200 import formats
    m = 1 << log_m
    n_public, n_vars = 3, m // 2
    nc = m - n_public - 1
    rng = np.random.default_rng(seed)
    coo = []
    for _ in range(2):
        rows = np.repeat(np.arange(nc, dtype=np.uint32), rng.poisson(2.0, nc))
        coo.append((rows, rng.integers(0, n_vars, rows.size, dtype=np.uint32), below_r(rng, rows.size)))
    mi, ci, si, vi = formats.zkey_coefficients(n_public, nc, coo[0], coo[1])
    g1 = lambda s, n: net.generate_g1(seed + s, n).cpu().numpy().view(np.uint64)
    g2 = lambda s, n: net.generate_g2(seed + s, n).cpu().numpy().view(np.uint64)
    vk1, vk2 = g1(6, 3), g2(7, 3)
    zk = formats.ZKey(n_vars=n_vars, n_public=n_public, domain_size=m, alpha_g1=vk1[0], beta_g1=vk1[1], beta_g2=vk2[0],
                      gamma_g2=vk2[2], delta_g1=vk1[2], delta_g2=vk2[1], ic=g1(8, n_public + 1), a_query=g1(1, n_vars),
                      b_g1_query=g1(2, n_vars), b_g2_query=g2(3, n_vars), l_query=g1(4, n_vars - n_public - 1), h_query=g1(5, m),
                      coef_matrix=mi, coef_row=ci, coef_col=si, coef_val_r2=vi)
    w = below_r(rng, n_vars)
    w[0] = [1, 0, 0, 0]
    s1 = struct.pack("<I", 32) + R.to_bytes(32, "little") + struct.pack("<I", n_vars)
    s2 = w.astype("<u8").tobytes()
    wtns = b"wtns" + struct.pack("<II", 2, 2) + struct.pack("<IQ", 1, len(s1)) + s1 + struct.pack("<IQ", 2, len(s2)) + s2
    return formats.write_zkey(zk), wtns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-m", default="16,18,20,22")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from distributed_groth16_b200 import Net, build, formats
    from distributed_groth16_b200.groth16 import circom
    from distributed_groth16_b200.groth16.native_prover import NO_TABLES, ZKeyProver
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the H100")
    build.build()
    net = Net(0)
    zero = np.zeros(4, dtype=np.uint64)
    results = dict(card=card(), sizes=[])
    tmp = tempfile.mkdtemp(prefix="zkey_prove_bench_")
    for log_m in (int(x) for x in args.log_m.split(",")):
        zkey, wtns = files(net, log_m, 0x5EED0 + log_m)
        zp, wp = os.path.join(tmp, "k.zkey"), os.path.join(tmp, "w.wtns")
        open(zp, "wb").write(zkey)
        open(wp, "wb").write(wtns)
        row = dict(log_m=log_m, zkey_mb=round(len(zkey) / 2**20, 1))

        # numpy's CSR of the same section, as circom.load_zkey runs it
        zk = formats.read_zkey(zkey)
        a_coo, b_coo = circom.zkey_matrices_coo(zk)
        t0 = time.perf_counter()
        for c in (a_coo, b_coo):
            formats.coo_to_csr(c[0], c[1], c[2], zk.num_constraints)
        row["csr_numpy_ms"] = round((time.perf_counter() - t0) * 1e3, 2)
        del zk, a_coo, b_coo

        # warm-up of every shape, then loads
        with ZKeyProver(net, zkey, NO_TABLES) as h:
            h.prove(wtns, zero, zero)
        net.profile(True)                       # kernel times in a load of their own: events slow the host
        net.profile_reset()
        ZKeyProver(net, zkey, NO_TABLES).free()
        prof = net.profile_report()
        net.profile(False)
        row["csr_gpu_ms"] = round(sum(prof[k]["ms"] for k in ("zkey_coef_check", "zkey_coef_hist", "msm_scan", "zkey_coef_scatter")
                                      if k in prof), 3)
        for name, tw in (("load_tables_s", 0), ("load_no_tables_s", NO_TABLES)):
            t0 = time.perf_counter()
            h = ZKeyProver(net, zkey, tw)
            row[name] = round(time.perf_counter() - t0, 4)
            if tw == 0:
                texts = h.prove(wtns, zero, zero)[:2]
                ts = []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    h.prove(wtns)
                    ts.append(time.perf_counter() - t0)
                row["prove_s"] = round(statistics.median(ts), 4)
            h.free()
        t0 = time.perf_counter()
        py = circom.groth16_prove(net, zkey, wtns, zero, zero)
        row["python_s"] = round(time.perf_counter() - t0, 4)
        assert py == texts, "native and Python texts differ at 2^%d" % log_m
        ts = []
        for _ in range(2):
            t0 = time.perf_counter()
            r = subprocess.run([build.PROVE_EXE, zp, wp, os.path.join(tmp, "proof.json"), os.path.join(tmp, "public.json")],
                               capture_output=True, text=True)
            ts.append(time.perf_counter() - t0)
            assert r.returncode == 0, r.stderr
        row["cmd_s"] = round(min(ts), 4)
        assert open(os.path.join(tmp, "public.json")).read() == texts[1]
        results["sizes"].append(row)
        print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=results["card"])))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(results, open(args.out, "w"), indent=1)
    net.close()


if __name__ == "__main__":
    main()
