"""Stream order of the device-pointer entry points: every `*_dev` call is ordered on the caller's torch stream.

The other GPU tests hand the library inputs that are already finished, so a missing stream edge cannot show there.  Here
each case races the library against its caller:
  - late write: the input first holds a poison (another complete, valid input of the same shape) and the real input is
    copied in on the current torch stream behind `torch.cuda._sleep`, so an entry point that does not wait for the caller's
    stream reads the whole poison;
  - early read: the output, filled with a poison, is cloned by a torch op on the current stream right after the call returns,
    before any synchronisation;
  - detection power: an event recorded after the late write must still be pending when an asynchronous entry point returns
    (otherwise something synchronised the device and the case proved nothing).  Each case first runs once on finished inputs,
    which warms every plan, table and workspace, gives the reference and times the op; the delay is the larger of 50 ms and
    20 times that time.
Only value data is poisoned (points, field elements, witnesses, never CSR structure), so a missing edge gives a wrong
answer, never an out-of-range access.  Each case runs once.

Also here: two host-staged MSMs in a row on one slot (the staging buffer must not be overwritten while the first MSM's
kernels still read it), re-binding slot 0 from one torch stream to another (the new stream must wait for the old one's
work through the slot), the prover's slots 1 and 2 behind a caller's work on slot 1, and a control case whose stream edge
is missing on purpose and which must see the poison.

Measured on one H100 80GB HBM3 at a 700 W power limit: 45 s for the file.
"""
import ctypes
import time

import numpy as np
import pytest

from oracle import bn254 as o, layout

import dlog_oracle as dl
import prove_dlog_oracle as po

pytestmark = pytest.mark.gpu

c_vp = ctypes.c_void_p
ONE_M = np.array([12436184717236109307, 3962172157175319849, 7381016538464732718, 1011752739694698287], dtype=np.uint64)
MIN_DELAY_MS = 50.0
DELAY_OVER_OP = 20.0


# ---- harness -------------------------------------------------------------------------------------------------------
_RATE = {}


def _cycles_per_ms():
    """torch.cuda._sleep's rate on this device, measured once with CUDA events"""
    import torch
    if "r" not in _RATE:
        torch.cuda._sleep(1000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        cycles = 20_000_000
        e0.record()
        torch.cuda._sleep(cycles)
        e1.record()
        torch.cuda.synchronize()
        _RATE["r"] = cycles / e0.elapsed_time(e1)
    return _RATE["r"]


def _delay_cycles(op_ms):
    ms = max(MIN_DELAY_MS, DELAY_OVER_OP * op_ms)
    assert ms < 5000, "op of %.1f ms is too slow to race" % op_ms
    return int(ms * _cycles_per_ms())


def _late_write(pairs, cycles):
    """on the current torch stream: a sleep, then dst.copy_(real) for every (dst, real); returns an event recorded after them"""
    import torch
    torch.cuda._sleep(cycles)
    for dst, real in pairs:
        dst.copy_(real)
    ev = torch.cuda.Event()
    ev.record()
    return ev


def _same(a, b):
    (ra, oa), (rb, ob) = a, b
    if isinstance(ra, tuple) or isinstance(rb, tuple):
        same_ret = len(ra) == len(rb) and all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(ra, rb))
    else:
        same_ret = np.array_equal(np.asarray(ra if ra is not None else 0), np.asarray(rb if rb is not None else 0))
    return same_ret and len(oa) == len(ob) and all(np.array_equal(x, y) for x, y in zip(oa, ob))


def race(what, inputs, outs, call, asynchronous, check=None, norm=None):
    """inputs: [(dst, real, poison)] CUDA tensors; outs: CUDA tensors the call writes; call(): issues the entry point and
    returns its host result (or None).  norm(outs) maps the host copies of outs to a canonical form (XYZZ sums: affine, since
    the bucket order may change the projective coordinates).  check(ref) asserts the reference run exactly."""
    import torch

    def _snap(ret, arrs):
        arrs = [a.cpu().numpy().copy() for a in arrs]
        return ret, norm(arrs) if norm is not None else arrs
    for dst, _, poison in inputs:
        dst.copy_(poison)
    torch.cuda.synchronize()
    want_poison = _snap(call(), outs)
    torch.cuda.synchronize()
    for dst, real, _ in inputs:
        dst.copy_(real)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ret = call()
    torch.cuda.synchronize()
    op_ms = (time.perf_counter() - t0) * 1e3
    want = _snap(ret, outs)
    assert not _same(want, want_poison), "%s: the poison gives the same answer as the input, the case cannot see a race" % what
    if check is not None:
        check(want)

    for dst, _, poison in inputs:
        dst.copy_(poison)
    for t in outs:
        t.fill_(-1)
    torch.cuda.synchronize()
    ev = _late_write([(dst, real) for dst, real, _ in inputs], _delay_cycles(op_ms))
    ret = call()
    early = [t.clone() for t in outs]
    pending = not ev.query()
    torch.cuda.synchronize()
    got = _snap(ret, early)
    if not _same(got, want):
        raise AssertionError("%s: result read on the caller's stream differs from the answer on finished inputs%s"
                             % (what, " and equals the answer for the poison" if _same(got, want_poison) else ""))
    if asynchronous:
        assert pending, ("%s: the late write had completed when the call returned (op %.2f ms), so the case proved nothing"
                         % (what, op_ms))
    return want


def _dev(net, arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).to(net._dev())


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def _xyzz_to_affine(net, xyzz, g2):
    return net.sum_points_dev(_dev(net, xyzz.view(np.uint64)), 1, g2=g2)


def _affine(net, g2):
    """norm for race(): every XYZZ output as its affine limbs followed by the infinity flag"""
    def f(arrs):
        return [np.append(*_xyzz_to_affine(net, a, g2)).astype(np.uint64) for a in arrs]
    return f


def _check_affine(want):
    """check for race() on one MSM output normalised by _affine"""
    def f(ref):
        _assert_point((ref[1][0][:-1], bool(ref[1][0][-1])), want, "reference run")
    return f


def _assert_point(got, want, what):
    (gp, ginf), (wp, winf) = got, want
    assert ginf == winf and (np.asarray(gp) == wp).all(), "%s: not the exact MSM" % what


# ---- A. late inputs and early reads, one case per device-pointer entry ------------------------------------------------
@pytest.mark.parametrize("g2,n", [(False, 3001), (True, 3001), (False, 1 << 22)], ids=["G1-3001", "G2-3001", "G1-2^22"])
def test_msm_dev(net, g2, n):
    """n = 3001 runs on the slot's stream alone; 2^22 G1 has four window groups and uses the slot's side stream"""
    import torch
    seed, pseed = 0x50A00000 + n + g2, 0x50B00000 + n + g2
    gen = net.generate_g2 if g2 else net.generate_g1
    real, poison = gen(seed, n), gen(pseed, n)
    bases = torch.empty_like(real)
    scalars = net.generate_fr(seed ^ 0x77, n)
    out = torch.empty(32 if g2 else 16, dtype=torch.int64, device=net._dev())
    fn = net._lib.b200zk_msm_g2_dev if g2 else net._lib.b200zk_msm_g1_dev
    want = dl.expected_msm(seed, _host(scalars), g2)

    def call():
        net.check(fn(net._h, 0, c_vp(bases.data_ptr()), c_vp(scalars.data_ptr()), n, c_vp(out.data_ptr())))

    race("msm_%s_dev n=%d" % ("g2" if g2 else "g1", n), [(bases, real, poison)], [out], call, True, check=_check_affine(want),
         norm=_affine(net, g2))


def test_msm_table_dev(net):
    import torch
    n, seed = 3001, 0x50C00000
    c = net.msm_table_auto_window(n)
    table = net.msm_table_build(net.generate_g1(seed, n), c)
    real, poison = net.generate_fr(seed ^ 0x77, n), net.generate_fr(seed ^ 0x78, n)
    scalars = torch.empty_like(real)
    out = torch.empty(16, dtype=torch.int64, device=net._dev())
    want = dl.expected_msm(seed, _host(real), False)

    def call():
        net.check(net._lib.b200zk_msm_table_dev(net._h, 0, 0, c_vp(table.data_ptr()), c_vp(scalars.data_ptr()), n, c,
                                                c_vp(out.data_ptr())))

    race("msm_table_dev", [(scalars, real, poison)], [out], call, True, check=_check_affine(want), norm=_affine(net, False))


@pytest.mark.parametrize("log_n", [10, 20])
@pytest.mark.parametrize("batch", [1, 4])
@pytest.mark.parametrize("kind", ["forward", "inverse", "coset"])
def test_ntt_fr_dev(net, cref, log_n, batch, kind):
    """2^10 takes two passes through the slot's ws_ntt scratch"""
    import torch
    n = 1 << log_n
    inverse, coset = kind == "inverse", kind == "coset"
    seed = 0x50D00000 + 16 * log_n + batch
    real, poison = net.generate_fr(seed, n * batch), net.generate_fr(seed ^ 0x99, n * batch)
    x = torch.empty_like(real)
    out = torch.empty_like(real)
    xh = _host(real)
    want = np.concatenate([cref.ntt(xh[b * n:(b + 1) * n], inverse=inverse, coset=coset) for b in range(batch)])

    def call():
        net.check(net._lib.b200zk_ntt_fr_dev(net._h, 0, c_vp(x.data_ptr()), c_vp(out.data_ptr()), log_n, int(inverse), int(coset),
                                             batch))

    def check(ref):
        assert (ref[1][0].view(np.uint64).reshape(-1, 4) == want).all(), "reference run differs from the CPU NTT"

    race("ntt_fr_dev %s 2^%d x%d" % (kind, log_n, batch), [(x, real, poison)], [out], call, True, check=check)


def test_ntt_fr_batched_post_dev(net, cref):
    """the column step of a 2^20 four-step NTT on rank 1 of 4: 256 transforms of 2^10, each times base^((b + b0) k)"""
    import torch
    log_t, batch, log_base, b0 = 10, 256, 20, 256
    real, poison = net.generate_fr(0x50E00000, batch << log_t), net.generate_fr(0x50E00001, batch << log_t)
    x = torch.empty_like(real)
    out = torch.empty_like(real)
    want = cref.ntt_batched_post(_host(real), log_t, batch, False, log_base, False, b0, 1, 0, 0)

    def call():
        net.check(net._lib.b200zk_ntt_fr_batched_post_dev(net._h, 0, c_vp(x.data_ptr()), c_vp(out.data_ptr()), log_t, batch, 0,
                                                          log_base, 0, b0, 1, 0, 0))

    def check(ref):
        assert (ref[1][0].view(np.uint64).reshape(-1, 4) == want).all(), "reference run differs from the CPU twin"

    race("ntt_fr_batched_post_dev", [(x, real, poison)], [out], call, True, check=check)


def _fr_triple(net, seed, n):
    import torch
    reals = [net.generate_fr(seed + k, n) for k in range(3)]
    poisons = [net.generate_fr(seed + 16 + k, n) for k in range(3)]
    dsts = [torch.empty_like(r) for r in reals]
    return reals, poisons, dsts


def test_h_circom_dev(net, cref):
    import torch
    log_m = 16
    reals, poisons, (a, b, c) = _fr_triple(net, 0x50F00000, 1 << log_m)
    out = torch.empty_like(a)
    want = cref.h_circom(*(_host(t) for t in reals))

    def call():
        net.check(net._lib.b200zk_h_circom_dev(net._h, c_vp(a.data_ptr()), c_vp(b.data_ptr()), c_vp(c.data_ptr()), log_m,
                                               c_vp(out.data_ptr())))

    def check(ref):
        assert (ref[1][0].view(np.uint64).reshape(-1, 4) == want).all(), "reference run differs from the CPU h"

    race("h_circom_dev", list(zip((a, b, c), reals, poisons)), [out], call, True, check=check)


def test_fr_convert_dev(net):
    import torch
    n = 1 << 16
    real, poison = net.generate_fr(0x51000000, n), net.generate_fr(0x51000001, n)
    x = torch.empty_like(real)
    out = torch.empty_like(real)
    want = np.asarray(layout.arr_to_fr(_host(real)[:64]), dtype=object)

    def call():
        net.check(net._lib.b200zk_fr_convert_dev(net._h, 0, c_vp(x.data_ptr()), c_vp(out.data_ptr()), n, 0, 1))

    def check(ref):                          # Montgomery -> canonical: the first rows are the integers themselves
        got = ref[1][0].view(np.uint64).reshape(-1, 4)[:64]
        assert [sum(int(w) << (64 * i) for i, w in enumerate(row)) for row in got] == list(want)

    race("fr_convert_dev", [(x, real, poison)], [out], call, True, check=check)


def test_fr_mul_sub_dev(net):
    import torch
    n = 1 << 16
    reals, poisons, (a, b, c) = _fr_triple(net, 0x51100000, n)
    out = torch.empty_like(a)
    ra, rb, rc = (layout.arr_to_fr(_host(t)[:64]) for t in reals)
    want = [(x * y - z) % o.R for x, y, z in zip(ra, rb, rc)]

    def call():
        net.check(net._lib.b200zk_fr_mul_sub_dev(net._h, 0, c_vp(a.data_ptr()), c_vp(b.data_ptr()), c_vp(c.data_ptr()),
                                                 c_vp(out.data_ptr()), n))

    def check(ref):
        assert layout.arr_to_fr(ref[1][0].view(np.uint64).reshape(-1, 4)[:64]) == want

    race("fr_mul_sub_dev", list(zip((a, b, c), reals, poisons)), [out], call, True, check=check)


def _csr(rng, n_rows, n_cols, vals):
    """CSR with 1..4 terms per row, columns in range, values from `vals` ((nnz, 4) Montgomery limbs, enough rows)"""
    cnt = rng.integers(1, 5, n_rows)
    ptr = np.zeros(n_rows + 1, dtype=np.uint32)
    ptr[1:] = np.cumsum(cnt)
    nnz = int(ptr[-1])
    idx = rng.integers(0, n_cols, nnz).astype(np.uint32)
    return ptr, idx, np.ascontiguousarray(vals[:nnz])


def _u32_dev(net, arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint32).view(np.int32)).to(net._dev())


def test_qap_dev(net, cref):
    """the witness is written late; the matrices are finished before the case starts"""
    import torch
    log_m, nc, ni, n_vars = 14, 12000, 3, 9000
    m = 1 << log_m
    rng = np.random.default_rng(0x5120)
    vals = cref.fr_generate(0x5121, 5 * nc)
    a_csr, b_csr = _csr(rng, nc, n_vars, vals), _csr(rng, nc, n_vars, vals[::-1])
    mats = [(_u32_dev(net, p), _u32_dev(net, i), _dev(net, v)) for p, i, v in (a_csr, b_csr)]
    real, poison = net.generate_fr(0x5122, n_vars), net.generate_fr(0x5123, n_vars)
    z = torch.empty_like(real)
    outs = [torch.empty((m, 4), dtype=torch.int64, device=net._dev()) for _ in range(3)]
    want = cref.qap(a_csr, b_csr, _host(real), nc, ni, m)
    torch.cuda.synchronize()
    (ap, ac, av), (bp, bc, bv) = mats

    def call():
        net.check(net._lib.b200zk_qap_dev(net._h, 0, c_vp(ap.data_ptr()), c_vp(ac.data_ptr()), c_vp(av.data_ptr()),
                                          c_vp(bp.data_ptr()), c_vp(bc.data_ptr()), c_vp(bv.data_ptr()), nc, ni, c_vp(z.data_ptr()),
                                          log_m, *(c_vp(t.data_ptr()) for t in outs)))

    def check(ref):
        for name, g, w in zip("abc", ref[1], want):
            assert (g.view(np.uint64).reshape(-1, 4) == w).all(), "reference run: vector %s differs from the CPU QAP" % name

    race("qap_dev", [(z, real, poison)], outs, call, True, check=check)


def _points(net, g2, seed, n):
    return (net.generate_g2 if g2 else net.generate_g1)(seed, n)


def _point_inputs(net, g2, seed, n, count=1):
    import torch
    reals = [_points(net, g2, seed + k, n) for k in range(count)]
    poisons = [_points(net, g2, seed + 16 + k, n) for k in range(count)]
    return list(zip([torch.empty_like(r) for r in reals], reals, poisons))


K_SCALE = (np.array([0x1234567890ABCDEF, 0x0FEDCBA987654321, 0x1111222233334444, 0x0123456789ABCDEF], dtype=np.uint64))
K_RATIO = (np.array([0x9E3779B97F4A7C15, 0x5, 0, 0], dtype=np.uint64))


@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_points_scale_dev(net, g2):
    import torch
    n = 4096
    ins = _point_inputs(net, g2, 0x51300000 + g2, n)
    pts = ins[0][0]
    out = torch.empty_like(pts)

    def call():
        net.check(net._lib.b200zk_points_scale_dev(net._h, 0, int(g2), c_vp(pts.data_ptr()), n, c_vp(K_SCALE.ctypes.data),
                                                   c_vp(out.data_ptr())))

    race("points_scale_dev %s" % ("G2" if g2 else "G1"), ins, [out], call, True)


def test_points_mul_powers_dev(net):
    """returns once out is complete (temporary device memory), so only the result is checked"""
    import torch
    n = 4096
    ins = _point_inputs(net, False, 0x51400000, n)
    pts = ins[0][0]
    out = torch.empty_like(pts)

    def call():
        net.check(net._lib.b200zk_points_mul_powers_dev(net._h, 0, 0, c_vp(pts.data_ptr()), n, c_vp(K_SCALE.ctypes.data),
                                                        c_vp(K_RATIO.ctypes.data), c_vp(out.data_ptr())))

    race("points_mul_powers_dev", ins, [out], call, False)


@pytest.mark.parametrize("inverse", [False, True], ids=["ntt", "intt"])
def test_points_ntt_dev(net, inverse):
    """returns once out is complete (temporary device memory), so only the result is checked"""
    import torch
    log_n = 12
    ins = _point_inputs(net, False, 0x51500000 + inverse, 1 << log_n)
    pts = ins[0][0]
    out = torch.empty_like(pts)
    fn = net._lib.b200zk_points_intt_dev if inverse else net._lib.b200zk_points_ntt_dev

    def call():
        net.check(fn(net._h, 0, 0, c_vp(pts.data_ptr()), log_n, c_vp(out.data_ptr())))

    race("points_%s_dev" % ("intt" if inverse else "ntt"), ins, [out], call, False)


def test_points_sub_dev(net):
    import torch
    n = 1 << 16
    ins = _point_inputs(net, False, 0x51600000, n, count=2)
    a, b = ins[0][0], ins[1][0]
    out = torch.empty_like(a)

    def call():
        net.check(net._lib.b200zk_points_sub_dev(net._h, 0, 0, c_vp(a.data_ptr()), c_vp(b.data_ptr()), n, c_vp(out.data_ptr())))

    race("points_sub_dev", ins, [out], call, True)


@pytest.mark.parametrize("fmt", [0, 1], ids=["uncompressed", "compressed"])
def test_points_encode_dev(net, fmt):
    import torch
    n = 1 << 14
    ins = _point_inputs(net, True, 0x51700000 + fmt, n)
    pts = ins[0][0]
    out = torch.empty((n, (128 if fmt == 0 else 64) // 8), dtype=torch.int64, device=net._dev())

    def call():
        net.check(net._lib.b200zk_points_encode_dev(net._h, 0, 1, c_vp(pts.data_ptr()), n, fmt, c_vp(out.data_ptr())))

    race("points_encode_dev fmt %d" % fmt, ins, [out], call, True)


def test_points_compress_dev(net):
    import torch
    n = 1 << 14
    ins = _point_inputs(net, False, 0x51800000, n)
    pts = ins[0][0]
    out = torch.empty((n, 4), dtype=torch.int64, device=net._dev())

    def call():
        net.check(net._lib.b200zk_points_compress_dev(net._h, 0, 0, c_vp(pts.data_ptr()), n, c_vp(out.data_ptr())))

    race("points_compress_dev", ins, [out], call, True)


def test_points_matmul_dev(net):
    import torch
    n_chunks, l, rows = 512, 8, 12
    ins = _point_inputs(net, False, 0x51900000, n_chunks * l)
    real_m, poison_m = net.generate_fr(0x51900100, rows * l), net.generate_fr(0x51900101, rows * l)
    ins.append((torch.empty_like(real_m), real_m, poison_m))
    pts, mat = ins[0][0], ins[1][0]
    out = torch.empty((n_chunks * rows, 8), dtype=torch.int64, device=net._dev())

    def call():
        net.check(net._lib.b200zk_points_matmul_dev(net._h, 0, 0, c_vp(pts.data_ptr()), n_chunks, l, c_vp(mat.data_ptr()), rows,
                                                    c_vp(out.data_ptr())))

    race("points_matmul_dev", ins, [out], call, True)


def test_points_spmv_dev(net, cref):
    """values and points are written late; row pointers and columns are finished first.  Reads ptr to the host, so only
    the result is checked"""
    import torch
    n_rows, n_pts = 3000, 2048
    rng = np.random.default_rng(0x51A0)
    ptr, idx, vals = _csr(rng, n_rows, n_pts, cref.fr_generate(0x51A1, 5 * n_rows))
    nnz = idx.shape[0]
    d_ptr, d_idx = _u32_dev(net, ptr), _u32_dev(net, idx)
    real_v, poison_v = _dev(net, vals), net.generate_fr(0x51A2, nnz)
    ins = _point_inputs(net, False, 0x51A00000, n_pts) + [(torch.empty_like(real_v), real_v, poison_v)]
    pts, val = ins[0][0], ins[1][0]
    out = torch.empty((n_rows, 8), dtype=torch.int64, device=net._dev())
    torch.cuda.synchronize()

    def call():
        net.check(net._lib.b200zk_points_spmv_dev(net._h, 0, 0, c_vp(d_ptr.data_ptr()), c_vp(d_idx.data_ptr()), c_vp(val.data_ptr()),
                                                  c_vp(pts.data_ptr()), n_rows, c_vp(out.data_ptr())))

    race("points_spmv_dev", ins, [out], call, False)


@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_fixed_base_mul_dev(net, g2):
    import torch
    n = 1 << 14
    real, poison = net.generate_fr(0x51B00000 + g2, n), net.generate_fr(0x51B00010 + g2, n)
    sc = torch.empty_like(real)
    out = torch.empty((n, 16 if g2 else 8), dtype=torch.int64, device=net._dev())
    k = layout.arr_to_fr(_host(real)[:2])

    def call():
        net.check(net._lib.b200zk_fixed_base_mul_dev(net._h, int(g2), c_vp(sc.data_ptr()), n, c_vp(out.data_ptr())))

    def check(ref):
        for i in range(2):
            assert (ref[1][0].view(np.uint64)[i] == dl.point_from_exponent(k[i], g2)[0]).all(), "reference run: row %d" % i

    race("fixed_base_mul_dev %s" % ("G2" if g2 else "G1"), [(sc, real, poison)], [out], call, True, check=check)


def _xyzz_partials(net, g2, seed, count):
    """`count` valid XYZZ points: the partials of small MSMs"""
    import torch
    w = 32 if g2 else 16
    out = torch.empty((count, w), dtype=torch.int64, device=net._dev())
    for k in range(count):
        net.msm_dev(_points(net, g2, seed + k, 300), net.generate_fr(seed + 100 + k, 300), out_xyzz=out[k], g2=g2)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_xyzz_sum_dev(net, g2):
    import torch
    count = 6
    real, poison = _xyzz_partials(net, g2, 0x51C00000 + 1000 * g2, count), _xyzz_partials(net, g2, 0x51C10000 + 1000 * g2, count)
    x = torch.empty_like(real)
    out = torch.empty(32 if g2 else 16, dtype=torch.int64, device=net._dev())

    def call():
        net.check(net._lib.b200zk_xyzz_sum_dev(net._h, 0, int(g2), c_vp(x.data_ptr()), count, 1, c_vp(out.data_ptr())))

    race("xyzz_sum_dev %s" % ("G2" if g2 else "G1"), [(x, real, poison)], [out], call, True, norm=_affine(net, g2))


# -- entry points that synchronise by design: the result check only --------------------------------------------------
@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_g_sum_dev(net, g2):
    import torch
    count = 5
    real, poison = _xyzz_partials(net, g2, 0x51D00000 + 1000 * g2, count), _xyzz_partials(net, g2, 0x51D10000 + 1000 * g2, count)
    x = torch.empty_like(real)
    w = 16 if g2 else 8
    fn = net._lib.b200zk_g2_sum_dev if g2 else net._lib.b200zk_g1_sum_dev

    def call():
        out = np.zeros(w, dtype=np.uint64)
        inf = ctypes.c_int(0)
        net.check(fn(net._h, 0, c_vp(x.data_ptr()), count, c_vp(out.ctypes.data), ctypes.byref(inf)))
        return out, inf.value

    race("g%d_sum_dev" % (2 if g2 else 1), [(x, real, poison)], [], call, False)


@pytest.mark.parametrize("fmt", [0, 1], ids=["uncompressed", "compressed"])
def test_points_decode_dev(net, fmt):
    import torch
    n, pb = 1 << 12, 64 if fmt == 0 else 32

    def encodings(seed):
        pts = _points(net, False, seed, n)
        enc = torch.empty((n, pb // 8), dtype=torch.int64, device=net._dev())
        net.check(net._lib.b200zk_points_encode_dev(net._h, 0, 0, c_vp(pts.data_ptr()), n, fmt, c_vp(enc.data_ptr())))
        torch.cuda.synchronize()
        return enc

    real, poison = encodings(0x51E00000 + fmt), encodings(0x51E10000 + fmt)
    data = torch.empty_like(real)
    out = torch.empty((n, 8), dtype=torch.int64, device=net._dev())

    def call():
        bad, first = ctypes.c_size_t(7), ctypes.c_size_t(7)
        net.check(net._lib.b200zk_points_decode_dev(net._h, 0, 0, c_vp(data.data_ptr()), n, fmt, 0, c_vp(out.data_ptr()),
                                                    ctypes.byref(bad), ctypes.byref(first)))
        return bad.value, first.value

    race("points_decode_dev fmt %d" % fmt, [(data, real, poison)], [out], call, False)


@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_points_decompress_dev(net, g2):
    import torch
    n = 1 << 12
    real = net.points_compress(_points(net, g2, 0x51F00000 + g2, n), g2=g2)
    poison = net.points_compress(_points(net, g2, 0x51F10000 + g2, n), g2=g2)
    data = torch.empty_like(real)
    out = torch.empty((n, 16 if g2 else 8), dtype=torch.int64, device=net._dev())

    def call():
        bad = ctypes.c_size_t(7)
        net.check(net._lib.b200zk_points_decompress_dev(net._h, 0, int(g2), c_vp(data.data_ptr()), n, int(g2), c_vp(out.data_ptr()),
                                                        ctypes.byref(bad)))
        return bad.value

    race("points_decompress_dev %s" % ("G2" if g2 else "G1"), [(data, real, poison)], [out], call, False)


# -- the prover ------------------------------------------------------------------------------------------------------
PROVE_SHAPE = (1 << 14, 12000, 3)           # m, n_vars, n_inputs


def _prove_instance(cref, seed):
    """(z, a, b, c) host arrays of PROVE_SHAPE, z[0] = 1"""
    m, n_vars, ni = PROVE_SHAPE
    z = cref.fr_generate(seed, n_vars)
    z[0] = ONE_M
    a, b, c = (cref.fr_generate(seed + k, m) for k in (1, 2, 3))
    return (z, a, b, c)


@pytest.fixture(scope="module")
def prover(net, cref):
    """a proving key of known-log points on the session context"""
    from distributed_groth16_b200.groth16.proving_key import ProvingKey
    m, n_vars, ni = PROVE_SHAPE
    spec = po.KeySpec(m, n_vars, ni, 0x5200 << 8)
    pts = spec.device_points(net)
    pk = ProvingKey.from_device(net, pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], ni, po.vk_array(pts))
    yield spec, pk
    pk.free()


def _expected_proof(cref, spec, inst):
    z, a, b, c = inst
    return po.proof_bytes(po.exponents(spec, z, po.expected_h(cref, a, b, c)), 0, 0)


def test_groth16_prove_dev(net, cref, prover):
    """z, a, b and c are written late on slot 0's stream; the prover's slots 1 and 2 must wait for them too"""
    import torch
    from distributed_groth16_b200.groth16 import prove
    spec, pk = prover
    real = [_dev(net, v) for v in _prove_instance(cref, 0x5210)]
    poison = [_dev(net, v) for v in _prove_instance(cref, 0x5220)]
    dst = [torch.empty_like(t) for t in real]
    want = _expected_proof(cref, spec, [_host(t) for t in real])

    def check(ref):
        assert ref[0] == want, "reference run: not the proof of the discrete-log oracle"

    race("groth16_prove_dev", list(zip(dst, real, poison)), [], lambda: prove.create_proof_dev(pk, *dst), False, check=check)


def test_groth16_assemble_dev(net, prover):
    import torch
    _, pk = prover

    def partials(seed):
        g1 = _xyzz_partials(net, False, seed, 4)
        return [g1[0], _xyzz_partials(net, True, seed + 50, 1)[0], g1[1], g1[2], g1[3]]

    real, poison = partials(0x52300000), partials(0x52310000)
    dst = [torch.empty_like(t) for t in real]
    r = np.zeros(4, dtype=np.uint64)
    s = np.zeros(4, dtype=np.uint64)

    def call():
        out = (ctypes.c_uint8 * 128)()
        a, b2, l_, h, b1 = (c_vp(t.data_ptr()) for t in dst)
        net.check(net._lib.b200zk_groth16_assemble_dev(net._h, pk._h, a, b2, l_, h, b1, c_vp(r.ctypes.data), c_vp(s.ctypes.data), 1,
                                                       out))
        return bytes(out)

    race("groth16_assemble_dev", list(zip(dst, real, poison)), [], call, False)


def test_group_groth16_prove_r1cs_dev(net, cref):
    """Group([0, 0]): two contexts on one GPU; the witness is written late on device 0's torch stream"""
    import torch
    from distributed_groth16_b200.group import Group, GroupConstraintMatrices, GroupProvingKey
    log_m, nc, ni, n_vars = 12, 3000, 3, 2500
    m = 1 << log_m
    rng = np.random.default_rng(0x5240)
    vals = cref.fr_generate(0x5241, 5 * nc)
    a_csr, b_csr = _csr(rng, nc, n_vars, vals), _csr(rng, nc, n_vars, vals[::-1])
    coo = lambda csr: (np.repeat(np.arange(nc, dtype=np.uint32), np.diff(csr[0].astype(np.int64))), csr[1], csr[2])
    spec = po.KeySpec(m, n_vars, ni, 0x5242 << 8)
    pts = {k: v if isinstance(v, np.ndarray) else _host(v) for k, v in spec.device_points(net).items()}
    zs = []
    for seed in (0x5243, 0x5244):
        z = cref.fr_generate(seed, n_vars)
        z[0] = ONE_M
        zs.append(z)
    want = po.proof_bytes(po.exponents(spec, zs[0], po.expected_h(cref, *cref.qap(a_csr, b_csr, zs[0], nc, ni, m))), 0, 0)
    grp = Group([0, 0])
    gpk = GroupProvingKey(grp, pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], ni, pts["vk1"][0], pts["vk1"][1], pts["vk1"][2],
                          pts["vk2"][0], pts["vk2"][1])
    mats = GroupConstraintMatrices(grp, ni, nc, coo(a_csr), coo(b_csr), values_montgomery_depth=0, log_m=log_m, n_vars=n_vars)
    try:
        real, poison = _dev(net, zs[0]), _dev(net, zs[1])
        z_dev = torch.empty_like(real)

        def check(ref):
            assert ref[0] == want, "reference run: not the proof of the discrete-log oracle"

        race("group_groth16_prove_r1cs_dev", [(z_dev, real, poison)], [], lambda: gpk.create_proof_r1cs(mats, z_dev), False,
             check=check)
    finally:
        mats.free()
        gpk.free()
        grp.close()


# ---- B. two host-staged MSMs on one slot ------------------------------------------------------------------------------
def _host_array(arr, pinned):
    import torch
    if not pinned:
        return np.array(arr, copy=True)
    t = torch.empty(arr.shape, dtype=torch.int64, pin_memory=True)
    out = t.numpy().view(np.uint64)
    out[...] = arr
    return out


@pytest.mark.parametrize("second", ["staged", "host"])
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("n", [3001, 1 << 20], ids=["3001", "2^20"])
def test_staged_msm_twice_on_one_slot(net, n, pinned, second):
    """call 1's kernels wait behind a sleep on slot 0's stream; call 2 (same scalars, other bases) must not overwrite the
    staging buffer they read.  n = 2^20 runs in five parts with the side stream, 3001 in one part; the second call is
    b200zk_msm_staged_dev again or the host entry b200zk_msm_g1, which stages through the same buffer"""
    import torch
    s1, s2 = 0x53000000 + n % 9973 + 2 * pinned, 0x53100000 + n % 9973 + 2 * pinned
    scalars = _host_array(_host(net.generate_fr(s1 ^ 0x55, n)), pinned)
    b1, b2 = (_host_array(_host(net.generate_g1(s, n)), pinned) for s in (s1, s2))
    want1, want2 = dl.expected_msm(s1, scalars), dl.expected_msm(s2, scalars)
    out1 = torch.empty(16, dtype=torch.int64, device=net._dev())
    out2 = torch.empty(16, dtype=torch.int64, device=net._dev())
    net.msm_staged(b1, scalars, out_xyzz=out1)                       # warm the staging buffer and workspaces at this size
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    net.msm(b1, scalars)
    op_ms = (time.perf_counter() - t0) * 1e3
    net._t0()
    torch.cuda._sleep(_delay_cycles(op_ms))
    net.msm_staged(b1, scalars, out_xyzz=out1)
    if second == "staged":
        net.msm_staged(b2, scalars, out_xyzz=out2)
    else:
        got2 = net.msm(b2, scalars)
    early1, early2 = out1.clone(), out2.clone()
    torch.cuda.synchronize()
    got1 = _xyzz_to_affine(net, _host(early1), False)
    if second == "staged":
        got2 = _xyzz_to_affine(net, _host(early2), False)
    (p1, i1), (p2, i2) = got1, got2
    hint = " (it is the answer for call 2's bases)" if i1 == want2[1] and (np.asarray(p1) == want2[0]).all() else ""
    assert i1 == want1[1] and (np.asarray(p1) == want1[0]).all(), "call 1 of two staged MSMs is wrong%s" % hint
    _assert_point(got2, want2, "call 2 of two staged MSMs")


@pytest.mark.parametrize("n", [3001, 1 << 20], ids=["3001", "2^20"])
def test_staged_msm_host_buffers_reusable_on_return(net, n):
    """b200zk_msm_staged_dev returns once the host buffers may be reused, also when its copies wait behind earlier work"""
    import torch
    seed = 0x53200000 + n % 9973
    scalars = _host_array(_host(net.generate_fr(seed ^ 0x55, n)), True)
    bases = _host_array(_host(net.generate_g1(seed, n)), True)
    want = dl.expected_msm(seed, scalars)
    other_s, other_b = _host(net.generate_fr(seed ^ 0x56, n)), _host(net.generate_g1(seed + 1, n))
    out = torch.empty(16, dtype=torch.int64, device=net._dev())
    net.msm_staged(bases, scalars, out_xyzz=out)
    torch.cuda.synchronize()
    net._t0()
    torch.cuda._sleep(_delay_cycles(10.0))
    net.msm_staged(bases, scalars, out_xyzz=out)
    bases[...] = other_b
    scalars[...] = other_s
    torch.cuda.synchronize()
    _assert_point(_xyzz_to_affine(net, _host(out), False), want, "staged MSM after its host buffers were overwritten")


# ---- C. re-binding slot 0 from one stream to another --------------------------------------------------------------------
@pytest.fixture
def rebind_back(net):
    yield
    net._t0()                                # slot 0 follows the default stream again


def _switch(net, run, what):
    """on stream A: a sleep, run(1), event eA; on stream B: run(2), event eB.  `_t0` re-binds slot 0 from A to B, and B's
    call uses the same slot buffers, so it must wait for A's"""
    import torch
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    eA, eB = torch.cuda.Event(), torch.cuda.Event()
    with torch.cuda.stream(A):
        run(0)                                # warm: plans, workspace size
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run(0)
        torch.cuda.synchronize()
        op_ms = (time.perf_counter() - t0) * 1e3
        torch.cuda._sleep(_delay_cycles(op_ms))
        run(1)
        eA.record()
    with torch.cuda.stream(B):
        run(2)
        eB.record()
    eB.synchronize()
    a_done = eA.query()
    torch.cuda.synchronize()
    assert a_done, "%s: the call on stream B finished while the earlier call through the slot on stream A had not" % what


def test_stream_switch_ntt(net, cref, rebind_back):
    log_n = 20
    xs = [net.generate_fr(0x54000000 + k, 1 << log_n) for k in range(3)]
    outs = [None, None, None]

    def run(k):
        outs[k] = net.ntt_dev(xs[k])

    _switch(net, run, "ntt_fr_dev")
    for k in (1, 2):
        assert (_host(outs[k]).reshape(-1, 4) == cref.ntt(_host(xs[k]))).all(), "NTT %d on its stream" % k


def test_stream_switch_h_circom(net, cref, rebind_back):
    m = 1 << 18
    ins = [[net.generate_fr(0x54100000 + 4 * k + j, m) for j in range(3)] for k in range(3)]
    outs = [None, None, None]

    def run(k):
        outs[k] = net.h_circom_dev(*ins[k])

    _switch(net, run, "h_circom_dev")
    for k in (1, 2):
        assert (_host(outs[k]).reshape(-1, 4) == cref.h_circom(*(_host(t) for t in ins[k]))).all(), "h %d on its stream" % k


# ---- D. the prover's other slots behind the caller's work on slot 1 -------------------------------------------------------
def test_prover_slots_behind_callers_slot1_work(cref):
    """slot 1 bound to a torch side stream S1 holding a sleep and a 2^20 MSM; the prover (slot 0, late inputs) uses slots 1
    and 2 as well.  Both results are exact.  A context of its own, so the session context keeps its slot 1"""
    import torch
    from distributed_groth16_b200 import Net
    from distributed_groth16_b200.groth16 import prove
    from distributed_groth16_b200.groth16.proving_key import ProvingKey
    net = Net(0)
    pk = None
    try:
        m, n_vars, ni = PROVE_SHAPE
        spec = po.KeySpec(m, n_vars, ni, 0x5500 << 8)
        pts = spec.device_points(net)
        pk = ProvingKey.from_device(net, pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], ni, po.vk_array(pts))
        n, seed = 1 << 20, 0x55100000
        bases, scalars = net.generate_g1(seed, n), net.generate_fr(seed ^ 0x5, n)
        want_msm = dl.expected_msm(seed, _host(scalars))
        inst = _prove_instance(cref, 0x5520)
        real = [_dev(net, v) for v in inst]
        poison = [_dev(net, v) for v in _prove_instance(cref, 0x5530)]
        dst = [torch.empty_like(t) for t in real]
        want = _expected_proof(cref, spec, inst)
        for d, p in zip(dst, poison):
            d.copy_(p)
        out1 = torch.empty(16, dtype=torch.int64, device=net._dev())
        S1 = torch.cuda.Stream()
        with torch.cuda.stream(S1):
            net.use_torch_stream(1)
        net.msm_dev(bases, scalars, out_xyzz=out1, sid=1)            # warm slot 1 at this size
        prove.create_proof_dev(pk, *real)                             # warm the prover's plans
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        prove.create_proof_dev(pk, *real)
        op_ms = (time.perf_counter() - t0) * 1e3
        cycles = _delay_cycles(op_ms)
        with torch.cuda.stream(S1):
            torch.cuda._sleep(cycles)
        net.msm_dev(bases, scalars, out_xyzz=out1, sid=1)
        _late_write(list(zip(dst, real)), cycles)
        got = prove.create_proof_dev(pk, *dst)
        torch.cuda.synchronize()
        assert got == want, "proof with slot 1 busy on the caller's side stream"
        _assert_point(net.sum_points_dev(out1, 1, sid=1), want_msm, "the caller's MSM on slot 1")
    finally:
        if pk is not None:
            pk.free()
        net.close()


# ---- control: a missing edge on purpose ------------------------------------------------------------------------------------
def test_control_missing_edge_reads_the_poison(net):
    """the input is written late on a side stream the library is not told about: fr_convert_dev (pure arithmetic, no
    index data) must then read the poison -- the harness turns a missing edge into a wrong answer"""
    import torch
    n = 1 << 16
    real, poison = net.generate_fr(0x56000000, n), net.generate_fr(0x56000001, n)
    x = torch.empty_like(real)
    out = torch.empty_like(real)

    def convert(src):
        y = torch.empty_like(src)
        net.check(net._lib.b200zk_fr_convert_dev(net._h, 0, c_vp(src.data_ptr()), c_vp(y.data_ptr()), n, 0, 1))
        torch.cuda.synchronize()
        return _host(y).copy()

    want_real, want_poison = convert(real), convert(poison)
    assert not np.array_equal(want_real, want_poison)
    x.copy_(poison)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        ev = _late_write([(x, real)], _delay_cycles(1.0))
    net.check(net._lib.b200zk_fr_convert_dev(net._h, 0, c_vp(x.data_ptr()), c_vp(out.data_ptr()), n, 0, 1))
    early = out.clone()
    pending = not ev.query()
    torch.cuda.synchronize()
    assert pending, "the late write on the side stream had completed before the call returned"
    assert np.array_equal(_host(early), want_poison), "the control did not see the poison"
