"""Times snarkjs `powersoftau prepare phase2` on the GPU (groth16/ptau.prepare_phase2) on synthetic ceremonies:

  * the tau sections 1-7 of a power-P ceremony are made on the device with the building blocks tests/ptau_writer.py's
    sections_gpu uses (powers of tau, fixed-base multiplication of the generators), without its Lagrange levels, and
    written to a temporary directory that is deleted afterwards;
  * prepare_phase2 end to end (file I/O included), with its split into transform, host <-> device transfers and writes;
  * the transform alone (b200zk_points_intt_dev, in place) per section and level: CUDA events around each call, after a
    warm-up on every section's group;
  * the twiddle-multiplication rate, from shapes: a level of 2^k points has k passes of 2^(k-1) butterflies, of which
    2^(k-1) - 2^(k-1-s) in pass s have a twiddle other than w^0, i.e. (k - 1) 2^(k-1) + 1 full scalar multiplications
    (the issue's estimate (k/2) 2^k counts the w^0 ones too); beside it the rate of b200zk_points_scale_dev on 2^20 G1
    points measured in the same run, the repository's yardstick for one scalar multiplication per point.
Prints one JSON line (also written to --out DIR/ptau_prepare_bench.json).
usage: python tools/ptau_prepare_bench.py [--powers 20,22] [--out DIR] [--tmp DIR]"""
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

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617
TAU, ALPHA, BETA = 0x1234567890ABCDEF1234567890ABCDEF, 11111111111111111111, 22222222222222222223


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk, clk_max = (x.strip() for x in q.split(","))
        return dict(gpu=name, power_limit=pl, sm_clock=clk, sm_clock_max=clk_max)
    except Exception as e:            # the numbers are reported without a card name rather than not at all
        return dict(gpu="unknown (%s)" % e)


def multiplications(k: int) -> int:
    return (k - 1) * (1 << (k - 1)) + 1 if k else 0


def write_unprepared(net, path, power):
    import struct
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16.setup import _fixed_base, _powers
    n1, n = (2 << power) - 1, 1 << power
    pts = lambda sc, g2=False: _fixed_base(net, sc.contiguous(), g2).cpu().numpy().tobytes()
    s1 = struct.pack("<I", 32) + formats.FQ_MODULUS.to_bytes(32, "little") + struct.pack("<II", power, power)
    secs = [(1, s1), (2, pts(_powers(net, TAU, 1, n1))), (3, pts(_powers(net, TAU, 1, n), True)),
            (4, pts(_powers(net, TAU, ALPHA, n))), (5, pts(_powers(net, TAU, BETA, n))), (6, pts(_powers(net, TAU, BETA, 1), True)),
            (7, struct.pack("<I", 0))]
    with open(path, "wb") as f:
        f.write(b"ptau" + struct.pack("<II", 1, len(secs)))
        for sid, body in secs:
            f.write(struct.pack("<IQ", sid, len(body)) + body)


def scale_rate(net, reps=5):
    import torch
    from distributed_groth16_b200.groth16 import phase2
    n = 1 << 20
    pts = net.generate_g1(0x5CA1E + 20, n)
    out = torch.empty_like(pts)
    k = int.from_bytes(os.urandom(32), "little") % R
    phase2.points_scale(net, pts, k, out=out)
    net.sync(0)
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        phase2.points_scale(net, pts, k, out=out)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    med = float(np.median(ms))
    return dict(n=n, ms_median=round(med, 3), mults_per_s=round(n / (med * 1e-3)))


def transform_levels(net, path):
    """CUDA-event time of every level of every section, in place on the tau points."""
    import torch
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16 import ptau
    out = {}
    with formats.PTau(path, prepared=False) as pt:
        for sid, (src, g2, extra) in ptau._SECTIONS.items():
            ptau.points_intt(net, net.to_device(ptau._tau_level(pt, sid, 4)), g2)       # warm-up
            net.sync(0)
            per = {}
            for k in range(pt.power + extra + 1):
                d = net.to_device(ptau._tau_level(pt, sid, k))
                net.sync(0)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                ptau.points_intt(net, d, g2, out=d)
                b.record()
                b.synchronize()
                per[k] = round(a.elapsed_time(b), 3)
                del d
            mults = sum(multiplications(k) for k in per)
            total = sum(per.values())
            out[sid] = dict(g2=g2, ms_per_level=per, ms_total=round(total, 1), mults=mults,
                            mults_per_s=round(mults / (total * 1e-3)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--powers", default="20,22")
    ap.add_argument("--out", default=None)
    ap.add_argument("--tmp", default=None)
    a = ap.parse_args()
    from distributed_groth16_b200 import Net
    from distributed_groth16_b200.groth16 import ptau
    net = Net(0)
    net.use_torch_stream(0)
    res = dict(info=gpu_info(), points_scale_g1=scale_rate(net), ceremonies={})
    for p in (int(x) for x in a.powers.split(",")):
        with tempfile.TemporaryDirectory(dir=a.tmp) as tmp:
            src, dst = os.path.join(tmp, "u.ptau"), os.path.join(tmp, "p.ptau")
            write_unprepared(net, src, p)
            levels = transform_levels(net, src)
            t = {}
            t0 = time.perf_counter()
            ptau.prepare_phase2(net, src, dst, timings=t)
            wall = time.perf_counter() - t0
            res["ceremonies"][p] = dict(end_to_end_s=round(wall, 2), split_s={k: round(v, 2) for k, v in t.items()},
                                        output_bytes=os.path.getsize(dst), sections=levels)
    res["info_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ptau_prepare_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
