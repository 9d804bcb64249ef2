"""Times the phase-1 ceremony on the GPU (groth16/phase1.py) end to end:

  * per power: `new`, `contribute`, `beacon` (e = 10) and `verify` on files in a temporary directory that is deleted
    afterwards; contribute / beacon split into kernel (b200zk_points_mul_powers_dev), encode (b200zk_points_encode_dev),
    host Blake2b, host <-> device transfers, file reads / writes and the key (fromRng, hash-to-G2, pairings excluded);
  * in the same process, the kernel's rate on 2^20 G1 and 2^18 G2 points (CUDA events, median of 5) next to
    b200zk_points_scale_dev on 2^20 G1 points and the point iNTT's twiddle products (b200zk_points_intt_dev, one 2^20 G1
    level and one 2^18 G2 level: (k - 1) 2^(k-1) + 1 scalar multiplications each);
  * the card name and power limit from nvidia-smi, before and after.
Prints one JSON line (also written to --out DIR/ptau_phase1_bench.json).
usage: python tools/ptau_phase1_bench.py [--powers 20,22] [--out DIR] [--tmp DIR]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from ptau_prepare_bench import gpu_info, multiplications  # noqa: E402

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617
BEACON = bytes(range(32))


def _median_ms(fn, reps=5):
    import torch
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def kernel_rates(net):
    import torch
    from distributed_groth16_b200.groth16 import phase1, phase2, ptau
    out = {}
    first, ratio = (int.from_bytes(os.urandom(32), "little") % R for _ in range(2))
    for g2, log_n in ((False, 20), (True, 18)):
        n = 1 << log_n
        pts = net.generate_g2(0x1B + log_n, n) if g2 else net.generate_g1(0x1B + log_n, n)
        res = torch.empty_like(pts)
        ms = _median_ms(lambda: phase1.points_mul_powers(net, pts, first, ratio, g2, out=res))
        ms_i = _median_ms(lambda: ptau.points_intt(net, pts, g2, out=res))
        m = multiplications(log_n)
        out["g2" if g2 else "g1"] = dict(n=n, mul_powers_ms=round(ms, 3), mul_powers_per_s=round(n / (ms * 1e-3)),
                                         intt_ms=round(ms_i, 3), intt_mults=m, intt_mults_per_s=round(m / (ms_i * 1e-3)))
        if not g2:
            k = first
            ms_s = _median_ms(lambda: phase2.points_scale(net, pts, k, out=res))
            out["g1"].update(points_scale_ms=round(ms_s, 3), points_scale_per_s=round(n / (ms_s * 1e-3)))
        del pts, res
    return out


def ceremony(net, power, tmp):
    from distributed_groth16_b200.groth16 import phase1, phase2
    p0, p1, p2 = (os.path.join(tmp, "p%d.ptau" % k) for k in range(3))
    res = {}
    t0 = time.perf_counter()
    phase1.new(p0, power)
    res["new_s"] = round(time.perf_counter() - t0, 2)
    t = {}
    t0 = time.perf_counter()
    phase1.contribute(net, p0, p1, phase2.ChaCha.from_hash(os.urandom(32)), timings=t)
    res["contribute_s"] = round(time.perf_counter() - t0, 2)
    res["contribute_split_s"] = {k: round(v, 2) for k, v in t.items()}
    os.unlink(p0)
    t = {}
    t0 = time.perf_counter()
    phase1.beacon(net, p1, p2, BEACON, 10, timings=t)
    res["beacon_s"] = round(time.perf_counter() - t0, 2)
    res["beacon_split_s"] = {k: round(v, 2) for k, v in t.items()}
    t0 = time.perf_counter()
    rep = phase1.verify(net, p2)
    res["verify_s"] = round(time.perf_counter() - t0, 2)
    res["verify_ok"] = rep.ok
    res["file_bytes"] = os.path.getsize(p2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--powers", default="20,22")
    ap.add_argument("--out", default=None)
    ap.add_argument("--tmp", default=None)
    a = ap.parse_args()
    from distributed_groth16_b200 import Net
    net = Net(0)
    net.use_torch_stream(0)
    res = dict(info=gpu_info(), kernels=kernel_rates(net), ceremonies={})
    for p in (int(x) for x in a.powers.split(",")):
        with tempfile.TemporaryDirectory(dir=a.tmp) as tmp:
            res["ceremonies"][p] = ceremony(net, p, tmp)
    res["info_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ptau_phase1_bench.json"), "w") as f:
            f.write(line + "\n")
    net.close()


if __name__ == "__main__":
    main()
