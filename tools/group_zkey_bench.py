"""One Groth16 proof from the witness on device 0 to the 128 bytes on the host, three ways, alternated in one process:

  (a) group:   GroupProvingKey.create_proof_r1cs (the QAP sharded over the group, each GPU in its column layout)
  (b) compose: one-GPU qap(), a, b, c and z copied to the host, GroupProvingKey.create_proof (what (a) replaces)
  (c) single:  circom.prove_from_matrices on one GPU

for P = 1 and, on a box with >= 2 GPUs, every GPU.  The three must give the same bytes.  Also times the one-GPU
b200zk_qap_dev of this tree against a library built from an earlier tree (--before-lib), alternated, with CUDA events.

The circuit is synthetic: nc = m - 3 constraints with Poisson(2) terms per row over n_vars = m / 2 variables, 3 inputs, a
random witness, and a key of generated points (the MSM and NTT work of a proof depends only on the sizes).

  python tools/group_zkey_bench.py --log-m 20,22 --reps 5 --out /tmp/group_zkey_bench.json \
      [--before-lib build/parent/libb200zk.so]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R_TOP = 21888242871839275222246405745257275088548364400416034343698204186575808495617 >> 192


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [l.strip() for l in q.stdout.strip().splitlines()]


def instance(net, log_m, seed):
    import torch
    from distributed_groth16_b200._constants import FR_ONE_MONT
    m = 1 << log_m
    nc, ni, n_vars = m - 3, 3, m // 2
    rng = np.random.default_rng(seed)
    csr = []
    for _ in range(2):
        cnt = rng.poisson(2.0, nc)
        rows = np.repeat(np.arange(nc, dtype=np.uint32), cnt)
        cols = rng.integers(0, n_vars, rows.size, dtype=np.uint32)
        vals = rng.integers(0, 1 << 64, (rows.size, 4), dtype=np.uint64)
        vals[:, 3] %= np.uint64(R_TOP)                          # below r, in Montgomery form as they stand
        csr.append((rows, cols, vals))
    z = net.generate_fr(seed, n_vars)
    z[0] = torch.tensor(np.array(FR_ONE_MONT, dtype=np.uint64).view(np.int64), device=z.device)
    pts = dict(a=net.generate_g1(seed + 1, n_vars), b1=net.generate_g1(seed + 2, n_vars), b2=net.generate_g2(seed + 3, n_vars),
               l=net.generate_g1(seed + 4, n_vars - ni), h=net.generate_g1(seed + 5, m))
    vk1, vk2 = net.generate_g1(seed + 6, 3).cpu().numpy().view(np.uint64), net.generate_g2(seed + 7, 2).cpu().numpy().view(np.uint64)
    return dict(m=m, nc=nc, ni=ni, n_vars=n_vars, coo=csr, z=z, pts=pts, vk1=vk1, vk2=vk2)


def timed(fn, sync):
    sync()
    t0 = time.perf_counter()
    out = fn()
    sync()
    return out, (time.perf_counter() - t0) * 1e3


def bench_proofs(net, I, devices_list, reps):
    import torch
    from distributed_groth16_b200.group import Group, GroupConstraintMatrices, GroupProvingKey
    from distributed_groth16_b200.groth16 import circom
    from distributed_groth16_b200.groth16.proving_key import ProvingKey
    from distributed_groth16_b200.groth16.qap import ConstraintMatrices, qap
    sync = torch.cuda.synchronize
    log_m = I["m"].bit_length() - 1
    host = {k: v.cpu().numpy().view(np.uint64) for k, v in I["pts"].items()}
    vk = np.concatenate([I["vk1"].reshape(-1), I["vk2"].reshape(-1)])
    pk = ProvingKey.from_device(net, I["pts"]["a"], I["pts"]["b1"], I["pts"]["b2"], I["pts"]["l"], I["pts"]["h"], I["ni"], vk)
    mats = ConstraintMatrices(net, I["ni"], I["nc"], I["coo"][0], I["coo"][1], values_montgomery_depth=0)
    z = I["z"]
    rows = []
    for devices in devices_list:
        g = Group(devices)
        gpk = GroupProvingKey(g, host["a"], host["b1"], host["b2"], host["l"], host["h"], I["ni"], I["vk1"][0], I["vk1"][1], I["vk1"][2],
                              I["vk2"][0], I["vk2"][1])
        gm = GroupConstraintMatrices(g, I["ni"], I["nc"], I["coo"][0], I["coo"][1], 0, log_m, I["n_vars"])

        def compose():
            q = qap(mats, z, net)
            a, b, c, zh = (t.cpu().numpy().view(np.uint64) for t in (q.a, q.b, q.c, z))
            return gpk.create_proof(zh, a, b, c)
        paths = {"a_group": lambda: gpk.create_proof_r1cs(gm, z), "b_compose": compose,
                 "c_single": lambda: circom.prove_from_matrices(pk, mats, z)}
        outs = {k: fn() for k, fn in paths.items()}                 # warm-up: module loads, workspaces, plans
        assert len(set(outs.values())) == 1, "the three paths disagree"
        ms = {k: [] for k in paths}
        for _ in range(reps):
            for k, fn in paths.items():
                out, t = timed(fn, sync)
                assert out == outs[k]
                ms[k].append(t)
        rows.append(dict(log_m=log_m, P=len(devices), devices=devices, table_bytes_single=pk.table_bytes, table_bytes_group=gpk.table_bytes,
                         **{k + "_ms": dict(median=statistics.median(v), min=min(v), all=v) for k, v in ms.items()}))
        print(json.dumps(rows[-1]), flush=True)
        gm.free()
        gpk.free()
        g.close()
    pk.free()
    return rows


def bench_qap(net, I, before_lib, reps, iters):
    """b200zk_qap_dev of this tree and of before_lib on the same device buffers, alternated; CUDA events over `iters` calls"""
    import torch
    from distributed_groth16_b200._native import c_vp
    from distributed_groth16_b200.groth16.qap import ConstraintMatrices
    mats = ConstraintMatrices(net, I["ni"], I["nc"], I["coo"][0], I["coo"][1], values_montgomery_depth=0)
    log_m = I["m"].bit_length() - 1
    outs = [torch.empty((I["m"], 4), dtype=torch.int64, device=I["z"].device) for _ in range(3)]
    (ap, ac, av), (bp, bc, bv) = mats.csr
    args = [c_vp(t.data_ptr()) for t in (ap, ac, av, bp, bc, bv)]
    libs = {"after": (net._lib, net._h)}
    if before_lib:
        old = ctypes.CDLL(os.path.abspath(before_lib))
        old.b200zk_ctx_create.argtypes = [ctypes.c_int, ctypes.POINTER(c_vp)]
        old.b200zk_ctx_set_stream.argtypes = [c_vp, ctypes.c_int, c_vp]
        old.b200zk_qap_dev.argtypes = [c_vp, ctypes.c_int] + [c_vp] * 6 + [ctypes.c_size_t, ctypes.c_size_t, c_vp, ctypes.c_uint] + [c_vp] * 3
        h = c_vp()
        assert old.b200zk_ctx_create(net.device, ctypes.byref(h)) == 0
        assert old.b200zk_ctx_set_stream(h, 0, c_vp(torch.cuda.current_stream().cuda_stream)) == 0
        libs["before"] = (old, h)
    results = {}
    for name, (lib, h) in libs.items():
        assert lib.b200zk_qap_dev(h, 0, *args, I["nc"], I["ni"], c_vp(I["z"].data_ptr()), log_m, *(c_vp(t.data_ptr()) for t in outs)) == 0
        torch.cuda.synchronize()
        results[name] = [t.clone() for t in outs]
    if "before" in results:
        assert all(torch.equal(x, y) for x, y in zip(results["before"], results["after"])), "qap_dev before / after differ"
    ms = {k: [] for k in libs}
    for rep in range(reps):
        for name, (lib, h) in sorted(libs.items(), reverse=bool(rep % 2)):        # ABBA: neither runs first every time
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                lib.b200zk_qap_dev(h, 0, *args, I["nc"], I["ni"], c_vp(I["z"].data_ptr()), log_m, *(c_vp(t.data_ptr()) for t in outs))
            e1.record()
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1) / iters)
    row = dict(log_m=log_m, **{"qap_dev_%s_ms" % k: dict(median=statistics.median(v), min=min(v), all=v) for k, v in ms.items()})
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-m", default="20,22")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--qap-iters", type=int, default=20)
    ap.add_argument("--before-lib", default=None, help="libb200zk.so built from an earlier tree, for the qap_dev comparison")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("group_zkey_bench: no CUDA device; nothing is measured without one")
    from distributed_groth16_b200 import Net
    net = Net(0)
    net.use_torch_stream(0)
    n = torch.cuda.device_count()
    devices_list = [[0]]
    w = 1
    while w * 2 <= min(n, 8):
        w *= 2
    if w >= 2:
        devices_list.append(list(range(w)))
    res = dict(card=card(), n_gpus=n, proofs=[], qap_dev=[])
    for log_m in (int(x) for x in args.log_m.split(",")):
        I = instance(net, log_m, 0x6B0000 + log_m)
        res["qap_dev"].append(bench_qap(net, I, args.before_lib, args.reps, args.qap_iters))
        res["proofs"] += bench_proofs(net, I, devices_list, args.reps)
        del I
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(dict(card=res["card"])))


if __name__ == "__main__":
    main()
