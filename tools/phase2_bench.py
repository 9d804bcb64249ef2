"""Times the phase-2 contribution (snarkjs `zkey contribute` on the GPU):

  * the one-scalar-many-points kernel, b200zk_points_scale_dev (G1: GLV + width-5 NAF, block-batched inversions), against
    the per-point ladder it replaces, b200zk_points_matmul_dev(n_chunks = n, l = 1, rows = 1), on 2^20 and 2^22 generated
    G1 points and one random scalar: CUDA events around each launch, warm-up first, the two kernels alternated in the
    same run, outputs asserted equal;
  * phase2.contribute end to end on a synthetic key with a 2^20 domain (L = 2^20 - 2 and H = 2^20 generated points,
    the other sections tiny), split into parsing, the record (proof of knowledge, transcript, hash-to-G2, delta),
    host <-> device transfers of L and H, the kernel, and serialisation.

Field products per point (operation counts kept here; a squaring counted as a product): an XYZZ doubling is 9, a mixed
addition 10, a general XYZZ addition 14, the affine normalisation 4 plus the inverse.  points_scale: 127 doublings,
~43 mixed additions (width-5 NAF of two 127-bit halves), 7 general additions and 7 normalisations for the table and
one for the result, each with ~16 products of the block-wide prefix / suffix and 1/64 of an inversion: ~1900.  matmul:
256 doublings, ~128 general additions, one inversion (~500 product-equivalents of the binary extended Euclid): ~4600.  The rate is reported as products / s against the 32-bit multiply-add ceiling of DESIGN
section 4 (32 lanes/clk/SM x 132 SMs x 1980 MHz / 128 multiply-adds per product ~ 65 G products/s).
Prints one JSON line (also written to --out DIR/phase2_bench.json).
usage: python tools/phase2_bench.py [--reps 10] [--sizes 20,22] [--out DIR]"""
import argparse
import json
import os
import struct
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617
PRODUCTS = dict(points_scale=127 * 9 + 43 * 10 + 7 * 14 + 8 * (4 + 16) + 8 * 500 / 64, points_matmul=256 * 9 + 128 * 14 + 4 + 500)
CEILING = 65e9


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = (x.strip() for x in q.split(","))
        return dict(gpu=name, power_limit=pl, sm_clock_max=clk)
    except Exception as e:            # the numbers are reported without a card name rather than not at all
        return dict(gpu="unknown (%s)" % e)


def kernels(net, log_n, reps):
    import torch
    from distributed_groth16_b200._native import c_vp
    from distributed_groth16_b200.groth16 import phase2
    n = 1 << log_n
    pts = net.generate_g1(0x5CA1E + log_n, n)
    k = int.from_bytes(os.urandom(32), "little") % R
    km = torch.from_numpy(np.array([((k << 256) % R >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)],
                                   dtype=np.uint64).view(np.int64)).to(pts.device).reshape(1, 4)
    out_s, out_m = torch.empty_like(pts), torch.empty_like(pts)
    run = dict(points_scale=lambda: phase2.points_scale(net, pts, k, out=out_s),
               points_matmul=lambda: net.check(net._lib.b200zk_points_matmul_dev(net._h, 0, 0, c_vp(pts.data_ptr()), n, 1,
                                                                                  c_vp(km.data_ptr()), 1, c_vp(out_m.data_ptr()))))
    for f in run.values():                                   # warm-up: module load, first launches
        f()
    net.sync(0)
    assert torch.equal(out_s, out_m), "points_scale and points_matmul disagree"
    ms = {name: [] for name in run}
    st = torch.cuda.current_stream()
    for _ in range(reps):
        for name, f in run.items():                          # alternated in the same run
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            f()
            b.record(st)
            b.synchronize()
            ms[name].append(a.elapsed_time(b))
    res = dict(n=n)
    for name, v in ms.items():
        med = float(np.median(v))
        rate = PRODUCTS[name] * n / (med * 1e-3)
        res[name] = dict(ms_median=round(med, 3), ms_min=round(min(v), 3), points_per_s=round(n / (med * 1e-3)),
                         products_per_s=round(rate), share_of_ceiling=round(rate / CEILING, 3))
    res["speedup"] = round(res["points_matmul"]["ms_median"] / res["points_scale"]["ms_median"], 2)
    return res


def synthetic_zkey(net, log_m):
    """A zkey whose L (2^log_m - 2 points) and H (2^log_m points) are generated G1 points; the other sections are a valid
    tiny header and empty query sections, which contribute() copies untouched."""
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import phase2
    m = 1 << log_m
    g1 = phase2._scale_one(net, np.array([((1 << 256) % formats.FQ_MODULUS >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] +
                                         [((2 << 256) % formats.FQ_MODULUS >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)],
                                         dtype=np.uint64), 1)
    g2 = net.generate_g2(7, 1).cpu().numpy().view(np.uint64)[0]
    l = net.generate_g1(11, m - 2).cpu().numpy().view(np.uint64)
    h = net.generate_g1(12, m).cpu().numpy().view(np.uint64)
    hdr = struct.pack("<I", 32) + formats.FQ_MODULUS.to_bytes(32, "little") + struct.pack("<I", 32) + \
        formats.FR_MODULUS.to_bytes(32, "little") + struct.pack("<III", m, 1, m)
    hdr += b"".join(np.asarray(p, dtype="<u8").tobytes() for p in (g1, g1, g2, g2, g1, g2))
    secs = {1: struct.pack("<I", 1), 2: hdr, 3: bytes(128), 4: struct.pack("<I", 0), 5: b"", 6: b"", 7: b"",
            8: l.tobytes(), 9: h.tobytes(), 10: bytes(64) + struct.pack("<I", 0)}
    order = (1, 2, 4, 3, 9, 8, 5, 6, 7, 10)
    z = b"zkey" + struct.pack("<II", 1, len(order)) + b"".join(struct.pack("<IQ", s, len(secs[s])) + secs[s] for s in order)
    return z, g1


def contribute_e2e(net, log_m, reps):
    from distributed_groth16_b200.groth16 import phase2
    z, g1 = synthetic_zkey(net, log_m)
    g1_s = phase2._scale_one(net, g1, 0x123456789)
    x = int.from_bytes(os.urandom(32), "little") % R or 1
    phase2.contribute(net, z, x, g1_s)                                      # warm-up
    runs = []
    for _ in range(reps):
        t = {}
        net.sync(0)
        t0 = time.perf_counter()
        phase2.contribute(net, z, x, g1_s, timings=t)
        t["total_s"] = time.perf_counter() - t0
        runs.append(t)
    med = {k: round(float(np.median([r[k] for r in runs])), 4) for k in runs[0]}
    return dict(domain=1 << log_m, l_points=(1 << log_m) - 2, h_points=1 << log_m, zkey_mb=round(len(z) / 2 ** 20, 1),
                reps=reps, median_s=med)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sizes", default="20,22")
    ap.add_argument("--e2e-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from distributed_groth16_b200 import Net
    net = Net(0)
    net.use_torch_stream(0)
    res = dict(**gpu_info(), kernels={}, products_per_point=PRODUCTS, ceiling_products_per_s=CEILING)
    for lg in (int(s) for s in a.sizes.split(",")):
        res["kernels"]["2^%d" % lg] = kernels(net, lg, a.reps)
    res["contribute_2^20"] = contribute_e2e(net, 20, a.e2e_reps)
    res.update(gpu_info_after=gpu_info())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "phase2_bench.json"), "w") as f:
            f.write(line + "\n")
    net.close()


if __name__ == "__main__":
    main()
