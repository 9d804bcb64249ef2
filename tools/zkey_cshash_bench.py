"""Times the circuit hash (csHash) of snarkjs `zkey new` on the GPU (groth16/cshash.py):

  * per domain 2^k: cshash.cs_hash over a synthetic key of n_vars = 2^k - 9 (random points, a few at infinity) and
    2^(k+1) - 1 random tau^i G1 points held in host memory (no file reads), split into the sub kernel
    (b200zk_points_sub_dev), the encode kernel (b200zk_points_encode_dev), host <-> device copies and host Blake2b, with
    the bytes hashed;
  * in the same process, the sub kernel alone (CUDA events, median of 5) on 2^22 G1 and 2^20 G2 points;
  * the card name and power limit from nvidia-smi, before and after.
Prints one JSON line (also written to --out DIR/zkey_cshash_bench.json).
usage: python tools/zkey_cshash_bench.py [--logs 20,22] [--out DIR]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from ptau_phase1_bench import _median_ms  # noqa: E402
from ptau_prepare_bench import gpu_info  # noqa: E402


class _TauG1:
    """Section 2 of a ceremony (tau^i G1) from host memory: what cshash.cs_hash reads of a formats.PTau."""

    def __init__(self, pts):
        self.pts = pts

    def has_section(self, sid):
        return sid == 2

    def section_span(self, sid):
        return 0, self.pts.shape[0] * 64

    def points(self, sid, first, count, width):
        return self.pts[first:first + count].copy()


def sub_rates(net):
    import torch
    from distributed_groth16_b200.groth16 import phase1
    out = {}
    for g2, log_n in ((False, 22), (True, 20)):
        n = 1 << log_n
        gen = net.generate_g2 if g2 else net.generate_g1
        a, b = gen(0x51 + log_n, n), gen(0x52 + log_n, n)
        res = torch.empty_like(a)
        ms = _median_ms(lambda: phase1.points_sub(net, a, b, g2, out=res))
        out["g2" if g2 else "g1"] = dict(n=n, ms=round(ms, 3), points_per_s=round(n / (ms * 1e-3)))
        del a, b, res
    return out


def cs_hash_run(net, log_n):
    import numpy as np
    from distributed_groth16_b200.groth16 import cshash
    from distributed_groth16_b200.groth16.phase1 import G1_GEN, G2_GEN
    n, n_public = 1 << log_n, 2
    n_vars = n - 9
    tau = _TauG1(net.generate_g1(0x70 + log_n, 2 * n - 1).cpu().numpy().view(np.uint64))
    a = net.generate_g1(0x71 + log_n, n_vars)
    a[[0, 5, n_vars - 1]] = 0
    q = dict(domain_size=n, alpha_g1=G1_GEN, beta_g1=G1_GEN, beta_g2=G2_GEN, gamma_g2=G2_GEN, delta_g1=G1_GEN,
             delta_g2=G2_GEN, ic=net.generate_g1(0x72 + log_n, n_public + 1),
             l_query=net.generate_g1(0x73 + log_n, n_vars - n_public - 1), a_query=a,
             b_g1_query=net.generate_g1(0x74 + log_n, n_vars), b_g2_query=net.generate_g2(0x75 + log_n, n_vars))
    hashed = 6 * 64 + 4 * 6 + 64 * (n_public + 1 + cshash.h_point_count(n) + (n_vars - n_public - 1) + 2 * n_vars) + 128 * n_vars
    cshash.cs_hash(net, q, tau, chunk=1 << 16)                   # warm-up: module load, allocator
    net.sync(0)
    t = {}
    t0 = time.perf_counter()
    digest = cshash.cs_hash(net, q, tau, timings=t)
    total = time.perf_counter() - t0
    return dict(domain=n, n_vars=n_vars, hashed_bytes=hashed, total_s=round(total, 3),
                split_s={k: round(v, 3) for k, v in t.items()},
                host_blake2b_mb_per_s=round(hashed / t["hash_s"] / 1e6, 1), digest=digest[:8].hex())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", default="20,22")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from distributed_groth16_b200 import Net
    net = Net(0)
    net.use_torch_stream(0)
    res = dict(info=gpu_info(), sub=sub_rates(net), cs_hash={})
    for k in (int(x) for x in a.logs.split(",")):
        res["cs_hash"][k] = cs_hash_run(net, k)
    res["info_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "zkey_cshash_bench.json"), "w") as f:
            f.write(line + "\n")
    net.close()


if __name__ == "__main__":
    main()
