"""The Groth16 prover (csrc/prove.cu) against exact answers from 2^16 to 2^24 constraints.

Every point of the proving keys here is generated with a known discrete log (tests/dlog_oracle.py), so each proof
element is e G for an exponent made of integer dot products (tests/prove_dlog_oracle.py, itself checked against the CPU
twin in tests/test_prove_dlog_oracle.py).  No curve MSM is needed for the expectation at any size.  Covered here:
  - h_circom_dev bit for bit against the CPU twin at 2^16, 2^20, 2^22 and 2^24;
  - m = n_vars = 2^16 .. 2^24 over the fixed-base tables and over the generic MSM (2^24: the tables exceed the budget and
    every query runs the generic MSM, four window groups on split streams), random and sha256-like witnesses (0 / 1
    almost everywhere: giant buckets), every randomiser family, proofs whose elements are the point at infinity, and
    the host-staged entry point;
  - key shapes: n_vars in {1, 40, m, 3m + 7}, n_inputs in {1, 2, 17, n_vars}, query rows at infinity (index 0, half the
    b-queries, all of l_query), and the exact table bytes of the mixed case where short queries get no table;
    n_inputs = n_vars also at 2^20 and 2^22, over the tables and the generic MSM;
  - the table budget and window variables, and the W * n >= 2^31 guard of the table build;
  - the two-level NTT twiddle tables (B200ZK_NTT_BIGTAB=0, read once per process) in a fresh process;
  - one Net reused across sizes and live keys, and a proof running while other host threads use slots 1 and 2.
A failure names the size, the configuration, the witness family and the (r, s) case.

Measured on one H100 80GB HBM3 at a 700 W power limit: 433 s for the file, most of it in the 2^24 leg (CPU h and the
exact dot products)."""
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

from oracle import bn254 as o, layout

import dlog_oracle as dl
import prove_dlog_oracle as po

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
R = o.R
LADDER = [16, 20, 22, 24]
RS_RANDOM = (0x2F1E3D4C5B6A79881726354453627180 % R, 0x0A1B2C3D4E5F60718293A4B5C6D7E8F9 * 7 % R)


# ---- helpers ----------------------------------------------------------------------------------------------------------
def _host(t):
    return t.cpu().numpy().view(np.uint64)


_QAP = {}


def qap_inputs(net, cref, m):
    """a, b, c on the device (seeded per m) and the CPU twin's h, kept for the whole module"""
    if m not in _QAP:
        a, b, c = (net.generate_fr(0x6A000000 + 8 * m + k, m) for k in range(3))
        _QAP[m] = (a, b, c, po.expected_h(cref, _host(a), _host(b), _host(c)))
    return _QAP[m]


def make_key(net, spec, tables=True):
    """ProvingKey.from_device on generated points; tables=False uploads with B200ZK_PK_TABLES=0 (no table build)"""
    import torch
    from distributed_groth16_b200.groth16 import ProvingKey
    pts = spec.device_points(net)
    old = os.environ.pop("B200ZK_PK_TABLES", None)
    if not tables:
        os.environ["B200ZK_PK_TABLES"] = "0"
    try:
        pk = ProvingKey.from_device(net, pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], spec.n_inputs, po.vk_array(pts))
    finally:
        os.environ.pop("B200ZK_PK_TABLES", None)
        if old is not None:
            os.environ["B200ZK_PK_TABLES"] = old
    del pts
    torch.cuda.empty_cache()
    if not tables:
        assert pk.table_bytes == 0
    return pk


def require_tables(pk, what):
    """a leg that needs the tables fails (never skips) when they could not be built, and says how much HBM was free"""
    import torch
    if pk.table_bytes == 0:
        free, total = torch.cuda.mem_get_info()
        pytest.fail("%s: no fixed-base tables were built (free HBM %.1f GB of %.1f GB)" % (what, free / 2**30, total / 2**30))


def expected_table_bytes(net, spec, c=0):
    """pk_precompute_dev's bytes: one table per query of >= 64 points, window c or the automatic one"""
    n1, naux = spec.n_vars - 1, spec.n_vars - spec.n_inputs
    total = 0
    for cnt, psz in ((n1, 64), (n1, 64), (n1, 128), (naux, 64), (spec.m, 64)):
        if cnt >= 64:
            total += net.msm_table_windows(c or net.msm_table_auto_window(cnt)) * cnt * psz
    return total


def witness(net, n, kind, seed):
    """(device tensor, host limbs) with z[0] = 1"""
    import torch
    if kind == "random":
        z = net.generate_fr(seed, n)
        z[0] = torch.from_numpy(po.ONE.view(np.int64)).to(z.device)
        return z, _host(z)
    zh = po.sha256_like_witness(n, seed)
    return net.to_device(zh), zh


def fr(v):
    return layout.fr_to_arr([v])[0]


def check_proof(pk, e, z, abc, r, s, what, mirror=False, staged=False):
    from distributed_groth16_b200.groth16 import prove
    a, b, c = abc[:3]
    if staged:
        got = prove.create_proof(pk, _host(z), _host(a), _host(b), _host(c), fr(r), fr(s), mirror_reference_bg1=mirror)
    else:
        got = prove.create_proof_dev(pk, z, a, b, c, fr(r), fr(s), mirror_reference_bg1=mirror)
    want = po.proof_bytes(e, r, s)
    if got != want:
        parts = [n for n, lo, hi in (("A", 0, 32), ("B", 32, 96), ("C", 96, 128)) if got[lo:hi] != want[lo:hi]]
        pytest.fail("proof mismatch: %s, r=%#x s=%#x, elements %s differ (tables %d bytes)" % (what, r, s, parts, pk.table_bytes))


def rs_cases(e, full):
    cases = {"r=s=0": (0, 0), "r,s random": RS_RANDOM}
    if full:
        cases.update({"r only": (RS_RANDOM[0], 0), "s only": (0, RS_RANDOM[1]), "r=s=ord-1": (R - 1, R - 1)})
        cases.update({"designed " + k: v for k, v in po.designed_cases(e).items()})
    return cases


@pytest.fixture(scope="module")
def net():
    """This module's own GPU party, closed when the module ends.  The 2^22 and 2^24 legs grow the slot workspaces to tens
    of GB; on the session's Net they would stay allocated for the rest of the run, and the key tables of later tests and
    other processes are sized by the HBM left free.  The switch subprocess runs first, before this Net exists."""
    import torch
    from distributed_groth16_b200 import Net
    n = Net(0)
    n.use_torch_stream(0)
    yield n
    torch.cuda.synchronize()
    _QAP.clear()
    n.close()
    torch.cuda.empty_cache()


# ---- 1. the two-level NTT twiddle tables (read once per process) ------------------------------------------------------------
def prove_legs(net, cref, legs, name, all_inputs=False):
    """per (log_m, path) a key with n_inputs = 2, or n_inputs = n_vars when `all_inputs`, proved at (0, 0) and random (r, s)"""
    import torch
    for log_m, path in legs:
        m = 1 << log_m
        abc = qap_inputs(net, cref, m)
        z, zh = witness(net, m, "random", 0x66000000 + log_m)
        ni = m if all_inputs else 2
        key = po.KeySpec(m, m, ni, 0x67000000 + 64 * log_m + (ni == m))
        e = po.exponents(key, zh, abc[3])
        pk = make_key(net, key, tables=path == "tables")
        if path == "tables":
            require_tables(pk, "%s m=2^%d" % (name, log_m))
        for cname, (r, s) in rs_cases(e, full=False).items():
            check_proof(pk, e, z, abc, r, s, "%s m=2^%d %s n_inputs=%d rs=%s" % (name, log_m, path, ni, cname))
        pk.free()
        torch.cuda.empty_cache()


def run_prove_switch(spec):
    """Body of one switch subprocess"""
    import torch
    from distributed_groth16_b200 import Net
    from oracle import cref
    cref.build()
    net = Net(0)
    net.use_torch_stream(0)
    prove_legs(net, cref, spec["legs"], spec["name"])
    torch.cuda.synchronize()
    net.close()


PROVE_SWITCHES = [
    ({"B200ZK_NTT_BIGTAB": "0"}, {"legs": [(20, "tables")]}),
]

SCRIPT = r"""
import json, sys
sys.path.insert(0, %r)
sys.path.insert(0, %r)
import test_gpu_prove_exact as t
t.run_prove_switch(json.loads(%r))
print("prove switch checks ok")
"""


@pytest.mark.parametrize("env,spec", PROVE_SWITCHES, ids=["%s=%s" % next(iter(e.items())) for e, _ in PROVE_SWITCHES])
def test_prove_switches(env, spec):
    import gc
    import torch
    spec = dict(spec, name="%s=%s" % next(iter(env.items())))
    _QAP.clear()                   # the subprocess sizes its tables by the HBM free when it starts: hand back what this one caches
    gc.collect()
    torch.cuda.empty_cache()
    e = dict(os.environ)
    for k in ("B200ZK_PK_TABLE_WINDOW", "B200ZK_PK_TABLE_MAX_GB", "B200ZK_PK_TABLES"):
        e.pop(k, None)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", SCRIPT % (ROOT, HERE, json.dumps(spec))], env=e, capture_output=True, text=True,
                       timeout=1200, cwd=ROOT)
    assert r.returncode == 0 and "prove switch checks ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


# ---- 2. h at scale ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_m", LADDER)
def test_h_ladder(net, cref, log_m):
    m = 1 << log_m
    a, b, c, h = qap_inputs(net, cref, m)
    got = _host(net.h_circom_dev(a, b, c))
    bad = np.nonzero((got != h).any(axis=1))[0]
    assert bad.size == 0, "h_circom_dev m=2^%d: %d rows differ, first %s" % (log_m, bad.size, bad[:8])


# ---- 3. key shapes ------------------------------------------------------------------------------------------------------
def _inf_patterns(nv, nl):
    half = list(range(0, nv, 2))
    return {"no infinity": {}, "index 0 at infinity": {"a": [0], "b1": [0], "b2": [0]},
            "half of b at infinity": {"b1": half, "b2": half[::-1]}, "l_query all infinity": {"l": list(range(nl))}}


@pytest.mark.parametrize("nv_kind", ["1", "40", "m", "3m+7"])
@pytest.mark.parametrize("log_m", [12, 16])
def test_key_shapes(net, cref, log_m, nv_kind):
    m = 1 << log_m
    nv = {"1": 1, "40": 40, "m": m, "3m+7": 3 * m + 7}[nv_kind]
    abc = qap_inputs(net, cref, m)
    z, zh = witness(net, nv, "random", 0x63000000 + nv)
    for ii, ni in enumerate(sorted({1, 2, 17, nv})):
        if ni > nv:
            continue
        pats = list(_inf_patterns(nv, nv - ni).items())
        # n_inputs = 2 runs every row pattern; the other n_inputs one pattern each, in turn
        for pname, inf in (pats if ni == 2 else [pats[ii % len(pats)]]):
            spec = po.KeySpec(m, nv, ni, 0x64000000 + 1000 * log_m + 10 * ii + len(inf), inf)
            e = po.exponents(spec, zh, abc[3])
            for tables in (True, False):
                pk = make_key(net, spec, tables)
                if tables:
                    assert pk.table_bytes == expected_table_bytes(net, spec), (nv, ni)
                for cname, (r, s) in rs_cases(e, full=False).items():
                    check_proof(pk, e, z, abc, r, s, "m=2^%d n_vars=%d n_inputs=%d %s tables=%s rs=%s"
                                % (log_m, nv, ni, pname, tables, cname))
                pk.free()


# ---- 4. table budget and window (read on every precompute) ----------------------------------------------------------------
def test_table_budget_and_window(net, cref, monkeypatch):
    m = 1 << 20
    spec = po.KeySpec(m, m, 2, 0x65000000)
    abc = qap_inputs(net, cref, m)
    z, zh = witness(net, m, "random", 0x65000001)
    e = po.exponents(spec, zh, abc[3])
    pk = make_key(net, spec)
    require_tables(pk, "m=2^20 automatic tables")
    monkeypatch.setenv("B200ZK_PK_TABLE_MAX_GB", "0")
    assert pk.precompute(0) == 0
    check_proof(pk, e, z, abc, *RS_RANDOM, "m=2^20 B200ZK_PK_TABLE_MAX_GB=0")
    monkeypatch.delenv("B200ZK_PK_TABLE_MAX_GB")
    for c in (7, 16, 22):
        monkeypatch.setenv("B200ZK_PK_TABLE_WINDOW", str(c))
        got = pk.precompute(0)
        require_tables(pk, "m=2^20 B200ZK_PK_TABLE_WINDOW=%d" % c)
        assert got == expected_table_bytes(net, spec, c)
        check_proof(pk, e, z, abc, *RS_RANDOM, "m=2^20 B200ZK_PK_TABLE_WINDOW=%d" % c)
    monkeypatch.delenv("B200ZK_PK_TABLE_WINDOW")
    pk.free()


# ---- 5. one Net reused across sizes and keys --------------------------------------------------------------------------------
def test_reuse_across_sizes_and_live_keys(net, cref):
    """2^22, then 2^16, then two live 2^22 keys interleaved: the slot workspaces and the small / io buffers go from large to
    small and back.  Then a key built without tables, proved, given tables, proved again."""
    import torch
    legs = []
    for tag, log_m, seed, tables in (("K22a", 22, 0x68000000, True), ("K16", 16, 0x68000100, True),
                                     ("K22b", 22, 0x68000200, False)):
        m = 1 << log_m
        spec = po.KeySpec(m, m, 2, seed)
        abc = qap_inputs(net, cref, m)
        z, zh = witness(net, m, "random", seed + 1)
        legs.append((tag, make_key(net, spec, tables), po.exponents(spec, zh, abc[3]), z, abc))
    require_tables(legs[0][1], "K22a")
    order = [0, 1, 2, 0, 2, 0, 1]
    for k, i in enumerate(order):
        tag, pk, e, z, abc = legs[i]
        check_proof(pk, e, z, abc, *RS_RANDOM, "reuse step %d key %s" % (k, tag))
    for _, pk, *_ in legs:
        pk.free()
    del legs
    torch.cuda.empty_cache()
    m = 1 << 16
    spec = po.KeySpec(m, m, 3, 0x68000300)
    abc = qap_inputs(net, cref, m)
    z, zh = witness(net, m, "sha256-like", 0x68000301)
    e = po.exponents(spec, zh, abc[3])
    pk = make_key(net, spec, tables=False)
    check_proof(pk, e, z, abc, *RS_RANDOM, "key without tables")
    pk.precompute(0)
    require_tables(pk, "precompute(0) after an upload without tables")
    check_proof(pk, e, z, abc, *RS_RANDOM, "same key after precompute(0)")
    pk.free()


# ---- 6. concurrency ------------------------------------------------------------------------------------------------------
def test_prove_while_other_threads_use_slots_1_and_2(net, cref):
    """The prover takes slots 1 and 2 for its own MSMs; two host threads loop host-staged MSMs on those slots meanwhile."""
    from distributed_groth16_b200.groth16 import prove
    m = 1 << 20
    spec = po.KeySpec(m, m, 2, 0x69000000)
    abc = qap_inputs(net, cref, m)
    z, zh = witness(net, m, "random", 0x69000001)
    e = po.exponents(spec, zh, abc[3])
    want = po.proof_bytes(e, *RS_RANDOM)
    pk = make_key(net, spec)
    jobs = []
    for sid in (1, 2):
        seed, n = 0x69000010 + sid, 20000 + 777 * sid
        bases, scalars = cref.g1_generate(seed, n), cref.fr_generate(seed, n)
        jobs.append((sid, bases, scalars, dl.expected_msm(seed, scalars)))
    errors, done = [], threading.Event()
    start = threading.Barrier(3)

    def prover():
        try:
            start.wait()
            for rep in range(4):
                got = prove.create_proof_dev(pk, z, *abc[:3], fr(RS_RANDOM[0]), fr(RS_RANDOM[1]))
                assert got == want, ("proof", rep)
        except BaseException as ex:      # noqa: BLE001 -- reported by the main thread
            errors.append(repr(ex))
        finally:
            done.set()

    def msm_loop(sid, bases, scalars, exp):
        try:
            start.wait()
            rep = 0
            while not done.is_set() or rep < 2:
                out, inf = net.msm(bases, scalars, sid=sid)
                assert inf == exp[1] and (out == exp[0]).all(), ("msm", sid, rep)
                rep += 1
        except BaseException as ex:      # noqa: BLE001
            errors.append(repr(ex))

    threads = [threading.Thread(target=prover)] + [threading.Thread(target=msm_loop, args=j) for j in jobs]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in threads), "a worker thread hung"
    assert not errors, errors
    pk.free()


# ---- 7. every variable public -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_m,path", [(20, "tables"), (22, "tables"), (22, "generic")])
def test_all_inputs_public(net, cref, log_m, path):
    """n_inputs = n_vars: the l_query MSM is empty (n = 0).  Runs before the size ladder: its 2^24 leg grows this module's slot
    workspaces until 60% of the free HBM no longer holds the 2^22 tables."""
    prove_legs(net, cref, [(log_m, path)], "n_inputs=n_vars", all_inputs=True)


# ---- 8. size ladder -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_m", LADDER)
def test_size_ladder(net, cref, log_m, monkeypatch):
    import torch
    m = 1 << log_m
    spec = po.KeySpec(m, m, 2, 0x61000000 + 16 * log_m)
    abc = qap_inputs(net, cref, m)
    h = abc[3]
    pk = make_key(net, spec)
    if log_m <= 22:
        require_tables(pk, "m=2^%d automatic tables" % log_m)
        assert pk.table_bytes == expected_table_bytes(net, spec)
    else:
        assert pk.table_bytes == 0, "2^24: the tables (84 GB) must exceed the budget (DESIGN.md section 3)"
    wits = {k: witness(net, m, k, 0x62000000 + log_m + 64 * i) for i, k in enumerate(("random", "sha256-like"))}
    exps = {k: po.exponents(spec, zh, h) for k, (_, zh) in wits.items()}
    cfg = "tables" if pk.table_bytes else "generic"
    for wk, (z, _) in wits.items():
        for cname, (r, s) in rs_cases(exps[wk], full=log_m == 20 and wk == "random").items():
            check_proof(pk, exps[wk], z, abc, r, s, "m=2^%d %s witness=%s rs=%s" % (log_m, cfg, wk, cname))
    z, e = wits["random"][0], exps["random"]
    if log_m == 20:
        check_proof(pk, e, z, abc, 0, RS_RANDOM[1], "m=2^20 %s mirror_bg1 r=0" % cfg, mirror=True)
    if log_m in (20, 24):
        check_proof(pk, e, z, abc, *RS_RANDOM, "m=2^%d %s host-staged create_proof" % (log_m, cfg), staged=True)
    # the generic MSM on the same key
    assert pk.precompute(None) == 0
    for wk, (zz, _) in wits.items():
        check_proof(pk, exps[wk], zz, abc, *RS_RANDOM, "m=2^%d generic witness=%s" % (log_m, wk))
    if log_m in (20, 22):
        pk.precompute(0)
        require_tables(pk, "m=2^%d forced table build" % log_m)
        check_proof(pk, e, z, abc, *RS_RANDOM, "m=2^%d rebuilt tables" % log_m)
    if log_m == 24:
        # c = 2: W * n = 128 * 2^24 = 2^31 for h_query: refused before any allocation, whatever the budget
        monkeypatch.setenv("B200ZK_PK_TABLE_WINDOW", "2")
        monkeypatch.setenv("B200ZK_PK_TABLE_MAX_GB", "1000")
        assert pk.precompute(0) == 0
        monkeypatch.delenv("B200ZK_PK_TABLE_WINDOW")
        monkeypatch.delenv("B200ZK_PK_TABLE_MAX_GB")
        check_proof(pk, e, z, abc, *RS_RANDOM, "m=2^24 after the W*n guard")
    pk.free()
    del wits
    torch.cuda.empty_cache()

