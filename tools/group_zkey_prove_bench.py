"""snarkjs `groth16 prove` from a .zkey and a .wtns on a group: the native group path (GroupZKeyProver, b200zk_group_zkey_*)
against the Python group path (group.load_zkey, circom.groth16_prove_group), per size and group:

  load_py_{tables,no_tables}_s      group.load_zkey (read_zkey, coo_to_csr, the host reorder per GPU, key upload), wall time
  load_native_{tables,no_tables}_s  GroupZKeyProver(...) (the sort on GPU 0, slices to each GPU, key upload), wall time
  prove_native_s                    one proof from a resident handle (automatic tables), JSON texts included
  prove_py_s                        circom.groth16_prove_group, which reads and uploads the key on every call
  cmd_devices_s / cmd_device_s      `b200zk-prove --devices ...` / `b200zk-prove --device 0` as a process, wall time

Each figure is the median of --reps rounds; within a round the two paths alternate.  Groups: P = 1 (`Group([0])`) and
P = 8 emulated on one GPU (`Group([0] * 8)`: every rank's work runs on GPU 0, so those rows measure host work and the sort, not
multi-GPU speed), plus every GPU of the box when it has 2 or more.  Keys and witnesses are tools/zkey_prove_bench.py's (known
discrete logs, nc = m - 4 Poisson(2) rows).  Every path must give the same texts for (r, s) = (0, 0).

  python tools/group_zkey_prove_bench.py --log-m 20,22 --reps 3 --out /tmp/group_zkey_prove_bench.json
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from zkey_prove_bench import card, files  # noqa: E402


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-m", default="20,22")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from distributed_groth16_b200 import Net, build
    from distributed_groth16_b200 import group as grp
    from distributed_groth16_b200.groth16 import circom
    from distributed_groth16_b200.groth16.native_prover import NO_TABLES, GroupZKeyProver
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: this benchmark measures the H100")
    build.build()
    net = Net(0)
    zero = np.zeros(4, dtype=np.uint64)
    n_dev = torch.cuda.device_count()
    worlds = [("P=1", [0]), ("P=8 emulated on one GPU", [0] * 8)]
    if n_dev >= 2:
        p = 1 << (min(n_dev, 8).bit_length() - 1)
        worlds.append(("P=%d real peers" % p, list(range(p))))
    results = dict(card=card(), n_gpus=n_dev, rows=[])
    tmp = tempfile.mkdtemp(prefix="group_zkey_prove_bench_")
    for log_m in (int(x) for x in args.log_m.split(",")):
        zkey, wtns = files(net, log_m, 0x5EED0 + log_m)
        zp, wp = os.path.join(tmp, "k.zkey"), os.path.join(tmp, "w.wtns")
        open(zp, "wb").write(zkey)
        open(wp, "wb").write(wtns)
        for wname, devices in worlds:
            g = grp.Group(devices)
            row = dict(log_m=log_m, world=wname)
            t = {k: [] for k in ("load_py_tables_s", "load_native_tables_s", "load_py_no_tables_s", "load_native_no_tables_s",
                                 "prove_native_s", "prove_py_s", "cmd_devices_s", "cmd_device_s")}
            with GroupZKeyProver(g, zkey, NO_TABLES) as h:      # warm-up of every shape
                want = h.prove(wtns, zero, zero)[:2]
            for _ in range(args.reps):
                for tables in (True, False):
                    sfx = "tables" if tables else "no_tables"
                    os.environ["B200ZK_PK_TABLES"] = "1" if tables else "0"      # read by group.load_zkey's key upload
                    dt, (gpk, mats, _) = timed(lambda: grp.load_zkey(g, zkey))
                    t["load_py_%s_s" % sfx].append(dt)
                    mats.free()
                    gpk.free()
                    os.environ.pop("B200ZK_PK_TABLES")
                    dt, h = timed(lambda: GroupZKeyProver(g, zkey, 0 if tables else NO_TABLES))
                    t["load_native_%s_s" % sfx].append(dt)
                    if tables:
                        dt, got = timed(lambda: h.prove(wtns, zero, zero))
                        assert got[:2] == want, (log_m, wname)
                        t["prove_native_s"].append(dt)
                    h.free()
                dt, py = timed(lambda: circom.groth16_prove_group(g, zkey, wtns, zero, zero))
                assert py == want, (log_m, wname)
                t["prove_py_s"].append(dt)
                for key, flag in (("cmd_devices_s", ["--devices", ",".join(map(str, devices))]), ("cmd_device_s", ["--device", "0"])):
                    dt, r = timed(lambda: subprocess.run([build.PROVE_EXE] + flag + [zp, wp, os.path.join(tmp, "p.json"),
                                                                                      os.path.join(tmp, "u.json")],
                                                         capture_output=True, text=True))
                    assert r.returncode == 0, r.stderr
                    assert open(os.path.join(tmp, "u.json")).read() == want[1]
                    t[key].append(dt)
            g.close()
            row.update({k: round(statistics.median(v), 4) for k, v in t.items()})
            results["rows"].append(row)
            print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()
    print(json.dumps(dict(card=results["card"], n_gpus=n_dev)))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(results, open(args.out, "w"), indent=1)
    net.close()


if __name__ == "__main__":
    main()
