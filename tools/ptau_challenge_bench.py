"""Times a phase-1 ceremony round by challenge and response on the GPU (groth16/phase1.py):

  * per power: `export challenge`, `challenge contribute`, `import response` and `verify` of the imported file, on files
    in a temporary directory that is deleted afterwards, each split into kernel (b200zk_points_mul_powers_dev), decode
    (b200zk_points_decode_dev), encode (b200zk_points_encode_dev), host Blake2b, host <-> device transfers, file reads /
    writes and the key;
  * in the same process, the decode kernel alone (CUDA events, median of 5, including the read-back of its two counters)
    on 2^20 G1 and 2^18 G2 points, compressed and uncompressed (G2 compressed with and without the subgroup check);
  * the card name and power limit from nvidia-smi, before and after.
Prints one JSON line (also written to --out DIR/ptau_challenge_bench.json).
usage: python tools/ptau_challenge_bench.py [--powers 20,22] [--out DIR] [--tmp DIR]"""
import argparse
import ctypes
import json
import os
import sys
import tempfile
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from ptau_phase1_bench import _median_ms  # noqa: E402
from ptau_prepare_bench import gpu_info  # noqa: E402


def decode_rates(net):
    import torch
    from distributed_groth16_b200._native import c_vp
    from distributed_groth16_b200.groth16 import phase1
    out = {}
    for g2, log_n in ((False, 20), (True, 18)):
        n = 1 << log_n
        pts = net.generate_g2(0x2C + log_n, n) if g2 else net.generate_g1(0x2C + log_n, n)
        res = torch.empty_like(pts)
        for compressed in (False, True):
            enc = phase1.points_encode(net, pts, g2, compressed)
            for check in ((0, 1) if g2 and compressed else (0,)):
                bad, first = ctypes.c_size_t(), ctypes.c_size_t()
                call = lambda: net.check(net._lib.b200zk_points_decode_dev(
                    net._h, 0, int(g2), c_vp(enc.data_ptr()), n, int(compressed), check, c_vp(res.data_ptr()),
                    ctypes.byref(bad), ctypes.byref(first)))
                ms = _median_ms(call)
                assert torch.equal(res, pts)
                key = "%s_%s%s" % ("g2" if g2 else "g1", "c" if compressed else "u", "_subgroup" if check else "")
                out[key] = dict(n=n, ms=round(ms, 3), points_per_s=round(n / (ms * 1e-3)))
        del pts, res, enc
    return out


def _timed(fn):
    t = {}
    t0 = time.perf_counter()
    r = fn(t)
    return r, round(time.perf_counter() - t0, 2), {k: round(v, 2) for k, v in t.items()}


def ceremony(net, power, tmp):
    from distributed_groth16_b200.groth16 import phase1, phase2
    p0, p1, ch, rs = (os.path.join(tmp, f) for f in ("p0.ptau", "p1.ptau", "challenge", "response"))
    phase1.new(p0, power)
    res = {}
    _, res["export_s"], res["export_split_s"] = _timed(lambda t: phase1.export_challenge(net, p0, ch, timings=t))
    res["challenge_bytes"] = os.path.getsize(ch)
    rng = phase2.ChaCha.from_hash(os.urandom(32))
    _, res["challenge_contribute_s"], res["challenge_contribute_split_s"] = _timed(
        lambda t: phase1.challenge_contribute(net, ch, rs, rng, timings=t))
    res["response_bytes"] = os.path.getsize(rs)
    os.unlink(ch)
    _, res["import_s"], res["import_split_s"] = _timed(lambda t: phase1.import_response(net, p0, rs, p1, timings=t))
    os.unlink(p0)
    t0 = time.perf_counter()
    res["verify_ok"] = phase1.verify(net, p1).ok
    res["verify_s"] = round(time.perf_counter() - t0, 2)
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
    res = dict(info=gpu_info(), decode=decode_rates(net), ceremonies={})
    for p in (int(x) for x in a.powers.split(",")):
        with tempfile.TemporaryDirectory(dir=a.tmp) as tmp:
            res["ceremonies"][p] = ceremony(net, p, tmp)
    res["info_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ptau_challenge_bench.json"), "w") as f:
            f.write(line + "\n")
    net.close()


if __name__ == "__main__":
    main()
