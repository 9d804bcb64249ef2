"""Times a phase-2 bellman round on the GPU (groth16/bellman.py): `zkey export bellman`, `zkey bellman contribute` and
`zkey import bellman` on a synthetic key per domain 2^k (random points, n_vars = 2^k - 9), each split into the point NTT /
iNTT, points_mul_powers, decode, scale and encode kernels, host <-> device transfers and host work, every stage between
two device synchronisations; the round is checked (export(import(response)) == response).  Also the card name and power
limit from nvidia-smi, before and after.  Prints one JSON line (also written to --out DIR/zkey_bellman_bench.json).
usage: python tools/zkey_bellman_bench.py [--logs 20,22] [--out DIR]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from ptau_prepare_bench import gpu_info  # noqa: E402


def synthetic_key(net, log_n: int) -> bytes:
    import numpy as np
    from distributed_groth16_b200 import formats
    from distributed_groth16_b200.groth16.phase1 import G1_GEN, G2_GEN
    n, n_public = 1 << log_n, 2
    n_vars = n - 9
    host = lambda t: t.cpu().numpy().view(np.uint64)
    zk = formats.ZKey(n_vars=n_vars, n_public=n_public, domain_size=n, alpha_g1=G1_GEN, beta_g1=G1_GEN, beta_g2=G2_GEN,
                      gamma_g2=G2_GEN, delta_g1=G1_GEN, delta_g2=G2_GEN, ic=host(net.generate_g1(0x80 + log_n, n_public + 1)),
                      a_query=host(net.generate_g1(0x81 + log_n, n_vars)), b_g1_query=host(net.generate_g1(0x82 + log_n, n_vars)),
                      b_g2_query=host(net.generate_g2(0x83 + log_n, n_vars)),
                      l_query=host(net.generate_g1(0x84 + log_n, n_vars - n_public - 1)),
                      h_query=host(net.generate_g1(0x85 + log_n, n)), coef_matrix=np.zeros(0, np.uint32),
                      coef_row=np.zeros(0, np.uint32), coef_col=np.zeros(0, np.uint32), coef_val_r2=np.zeros((0, 4), np.uint64))
    return formats.write_zkey(zk)


def round_run(net, log_n: int) -> dict:
    from distributed_groth16_b200.groth16 import bellman
    from distributed_groth16_b200.groth16.phase1 import G1_GEN
    z = synthetic_key(net, log_n)
    out = dict(domain=1 << log_n, zkey_bytes=len(z))
    steps = (("export", lambda: bellman.export(net, z, timings=t)),
             ("contribute", lambda: bellman.contribute(net, res["export"], 0x1234567890ABCDEF, G1_GEN, timings=t)[0]),
             ("import", lambda: bellman.import_response(net, z, res["contribute"], name="bench", timings=t)))
    res = {}
    for name, fn in steps:
        t = {}
        net.sync(0)
        t0 = time.perf_counter()
        res[name] = fn()
        net.sync(0)
        out[name] = dict(total_s=round(time.perf_counter() - t0, 3), split_s={k: round(v, 3) for k, v in t.items()})
    out["params_bytes"] = len(res["export"])
    out["round_trip_ok"] = bellman.export(net, res["import"]) == res["contribute"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", default="20,22")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from distributed_groth16_b200 import Net
    net = Net(0)
    net.use_torch_stream(0)
    res = dict(info=gpu_info(), rounds={})
    round_run(net, 10)                                            # warm-up: module load, allocator
    for k in (int(x) for x in a.logs.split(",")):
        res["rounds"][k] = round_run(net, k)
    res["info_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "zkey_bellman_bench.json"), "w") as f:
            f.write(line + "\n")
    net.close()


if __name__ == "__main__":
    main()
