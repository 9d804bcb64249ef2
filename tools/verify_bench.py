"""Times one Groth16 verification on the GPU (k_groth16_verify, csrc/verify.cu) against the number of public inputs.

The kernel runs four Miller loops and one final exponentiation; the IC sum IC_0 + sum_i x_i IC_{i+1} runs on one thread
as a 256-bit double-and-add per input, so its cost grows linearly with n_public.  For each n the key and the proof have
known discrete logs (every point is e G by b200zk_fixed_base_mul_dev) and the proof is valid, so the call is checked to
accept.  CUDA events on the library's stream around one b200zk_groth16_verify call (host-to-device copies of the key and
the inputs, the kernel, the one-word result); one warm-up call, then the median of --reps calls.
Prints one JSON line (also written to --out DIR/verify_bench.json).
usage: python tools/verify_bench.py [--n 1,1000,4096] [--reps 5] [--out DIR]"""
import argparse
import ctypes
import json
import os
import random
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def mont(vals):
    b = b"".join((v % R * (1 << 256) % R).to_bytes(32, "little") for v in vals)
    return np.frombuffer(b, dtype=np.uint64).reshape(-1, 4).copy()


def points(net, exps, g2):
    import torch
    from distributed_groth16_b200._native import c_vp
    sc = net.to_device(mont(exps))
    out = torch.empty((len(exps), 16 if g2 else 8), dtype=torch.int64, device=sc.device)
    net.check(net._lib.b200zk_fixed_base_mul_dev(net._h, int(g2), c_vp(sc.data_ptr()), len(exps), c_vp(out.data_ptr())))
    return np.ascontiguousarray(out.cpu().numpy().view(np.uint64))


def time_verify(net, n, reps, rng):
    import torch
    from distributed_groth16_b200.context import _ptr
    rnd = lambda: rng.randrange(1, R)
    al, be, ga, de, a, b = (rnd() for _ in range(6))
    ic, x = [rnd() for _ in range(n + 1)], [rnd() for _ in range(n)]
    s = (ic[0] + sum(xi * l for xi, l in zip(x, ic[1:]))) % R
    c = (a * b - al * be - ga * s) * pow(de, -1, R) % R
    g1 = points(net, [al, a, c] + ic, False)
    g2 = points(net, [be, ga, de, b], True)
    xm = mont(x) if n else np.zeros((1, 4), dtype=np.uint64)
    icp = np.ascontiguousarray(g1[3:])
    ok = ctypes.c_int(0)

    def call():
        net.check(net._lib.b200zk_groth16_verify(net._h, _ptr(g1[0]), _ptr(g2[0]), _ptr(g2[1]), _ptr(g2[2]), _ptr(icp), n,
                                                 _ptr(xm) if n else None, _ptr(g1[1]), _ptr(g2[3]), _ptr(g1[2]),
                                                 ctypes.byref(ok)))
    call()
    assert ok.value == 1, "the valid proof at n_public = %d was rejected" % n
    st = torch.cuda.current_stream()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        call()
        e1.record(st)
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
        assert ok.value == 1
    return dict(n_public=n, ms_median=round(float(np.median(ms)), 3), ms_min=round(min(ms), 3), reps=reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", default="1,1000,4096")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from phase2_bench import gpu_info
    from distributed_groth16_b200 import Net
    net = Net(0)
    net.use_torch_stream(0)
    rng = random.Random(0xBE7C)
    res = dict(**gpu_info(), verify=[time_verify(net, int(n), a.reps, rng) for n in a.n.split(",")])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "verify_bench.json"), "w") as f:
            f.write(line + "\n")
    net.close()


if __name__ == "__main__":
    main()
