"""The MSM (csrc/msm.cu) against exact answers at every window width and size up to 2^26.

The bases are generated with known discrete logs, P_i = k_i G (tests/dlog_oracle.py), so MSM(P, s) = (sum_i k_i s_i) G
is known exactly at any size without running another MSM.  Covered here:
  - the default configuration at 2^20 .. 2^26 (device-resident with its window groups, host-staged in parts, fixed-base
    table), with the generated points themselves spot-checked against k_i G, and host-staged MSMs of 1, 5 and 15 pairs;
  - every window width B200ZK_MSM_WINDOW = 2..23 on G1 and 2..20 on G2 (read on every call), each with digit-pattern
    scalar families that put B, B + 1 or 2^c - 1 into every window of both GLV halves; at 2^20 the small widths
    (c <= 8) also run task lengths above 128 and block-level merges of the giant buckets.  Width 24 needs about 33 GB of
    G1 bucket workspace (10^8 buckets with their task sums) and is left out;
  - adversarial bucket contents: one point n times, P and -P, s and r - s, and +-G bases whose bucket counts make a
    running sum of the segment reduction hit the identity and equal the bucket it adds (quad and thread reduction);
  - the W * n >= 2^32 guard, which must refuse before any allocation;
  - fixed-base tables at every window c = 2..24 (G1) and 2..20 (G2) with digit-pattern families, reaching all three
    `wsplit` branches, a G2 table at 2^20, and the fold path's W * n >= 2^31 guard.
A failure names the configuration, the family and the size.

Measured on one H100 80GB HBM3 at a 700 W power limit: 180 s for the file, host oracle included."""
import os

import numpy as np
import pytest

from oracle import bn254 as o, layout

import dlog_oracle as dl

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

G1_WINDOWS = list(range(2, 24))
G2_WINDOWS = list(range(2, 21))


# ---- helpers ----------------------------------------------------------------------------------------------------
def _host(t):
    return t.cpu().numpy().view(np.uint64)


def _assert_canonical(sh):
    """every Montgomery scalar read back from the device is < r"""
    r = np.array([(o.R >> (64 * i)) & dl.MASK64 for i in range(4)], dtype=np.uint64)
    lt = np.zeros(sh.shape[0], dtype=bool)
    eq = np.ones(sh.shape[0], dtype=bool)
    for i in (3, 2, 1, 0):
        lt |= eq & (sh[:, i] < r[i])
        eq &= sh[:, i] == r[i]
    assert lt.all(), "scalar >= r at %s" % np.nonzero(~lt)[0][:8]


def _msm_dev(net, bases, scalars, g2):
    return net.sum_points_dev(net.msm_dev(bases, scalars, g2=g2), 1, g2=g2)


def _check_point(got, want, what):
    (gp, ginf), (wp, winf) = got, want
    assert ginf == winf and (np.asarray(gp) == wp).all(), "MSM mismatch: %s (got inf=%s, want inf=%s)" % (what, ginf, winf)


def _check_generated(net, seed, n, g2, what, staged=False):
    """device-generated bases and scalars, exact answer from the logs"""
    bases = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
    scalars = net.generate_fr(seed ^ 0x5CA1A4, n)
    sh = _host(scalars)
    _assert_canonical(sh)
    want = dl.expected_msm(seed, sh, g2)
    got = net.msm(_host(bases), sh, g2=g2) if staged else _msm_dev(net, bases, scalars, g2)
    _check_point(got, want, what)
    return bases


def _family_scalars(c):
    fams = dl.digit_families(c, True)
    fams["glv_halves"] = [dl.glv_compose(a, b) for a, b in dl.glv_designed_halves()] + list(_extremes())
    return fams


_EXT = []


def _extremes():
    if not _EXT:
        _EXT.extend(dl.glv_extremes(1 << 14))
    return _EXT


def _check_families(net, c, g2, what):
    """one MSM per scalar family on the first generated bases; the designed GLV halves are confirmed first"""
    import torch
    fams = _family_scalars(c)
    for a, b in dl.glv_designed_halves():
        assert dl.glv_decompose(dl.glv_compose(a, b)) == (a, b)
    seed = 0xFA000000 + c
    m = max(len(v) for v in fams.values())
    bases = net.generate_g2(seed, m) if g2 else net.generate_g1(seed, m)
    for name, ks in fams.items():
        sc = layout.fr_to_arr(ks)
        want = dl.expected_msm(seed, sc, g2)
        got = _msm_dev(net, bases[: len(ks)].contiguous(), torch.from_numpy(sc.view(np.int64)).to(bases.device), g2)
        _check_point(got, want, "%s family %s" % (what, name))


def _sweep_one(net, c, g2, big=True):
    os.environ["B200ZK_MSM_WINDOW"] = str(c)
    try:
        what = "%s c=%d" % ("G2" if g2 else "G1", c)
        for n in (3001, 40000) + (((1 << 20),) if big and c <= 8 else ()):
            _check_generated(net, 0xC0000000 + 1000 * c + n % 997, n, g2, "%s n=%d" % (what, n))
        _check_families(net, c, g2, what)
    finally:
        del os.environ["B200ZK_MSM_WINDOW"]


def _g_arr(g2, neg=False):
    curve, gen = (o.G2, o.G2_GEN) if g2 else (o.G1, o.G1_GEN)
    return (layout.g2_to_arr if g2 else layout.g1_to_arr)([curve.neg(gen) if neg else gen])[0]


# Bucket counts m_d (multiples of G in bucket d) of the +-G collision case, top bucket of every 8-bucket block first: the
# running sum of the segment reduction goes 1, 0 (identity: G + (-G)), 1, 2 (doubling: G + G), 2, 4, 0 (4G + (-4G)), 3, ...
COLLIDE_BLOCK = [1, -1, 1, 1, 0, 2, -4, 3]


def collision_counts(B):
    m = [0] * (B + 1)                                   # m[d], digit d = 1..B
    for b in range(B):                                   # bucket b holds digit b + 1; blocks of 8 from the top down
        j = 7 - (b % 8)
        m[b + 1] = COLLIDE_BLOCK[j]
    return m


def simulate_segments(m, B, seg_len):
    """(identity hits, doubling hits) of run = run + bucket in k_msm_reduce_segments(_quad), buckets of G multiples"""
    ident = dbl = 0
    for lo in range(0, B, seg_len):
        run = 0
        for b in range(lo + seg_len - 1, lo - 1, -1):
            mb = m[b + 1]
            if run and mb and run + mb == 0:
                ident += 1
            if run and run == mb:
                dbl += 1
            run += mb
    return ident, dbl


def check_collisions(net, g2, seg_len, c=5):
    """+-G bases with scalars 1..B at window c: every bucket is a known multiple of G (k = d < 2^c: window 0 only, and the
    GLV split leaves k2 = 0)."""
    import torch
    B = 1 << (c - 1)
    m = collision_counts(B)
    ident, dbl = simulate_segments(m, B, seg_len)
    assert ident > 0 and dbl > 0, (ident, dbl)
    logs, scal, rows = [], [], []
    gp, gn = _g_arr(g2), _g_arr(g2, True)
    for d in range(1, B + 1):
        for _ in range(abs(m[d])):
            rows.append(gp if m[d] > 0 else gn)
            logs.append(1 if m[d] > 0 else -1)
            scal.append(d)
    sc = layout.fr_to_arr(scal)
    want = dl.expected_from_logs(logs, sc, g2)
    assert want[0].any() and not want[1]
    os.environ["B200ZK_MSM_WINDOW"] = str(c)
    try:
        got = _msm_dev(net, torch.from_numpy(np.stack(rows).view(np.int64)).cuda(), torch.from_numpy(sc.view(np.int64)).cuda(), g2)
    finally:
        del os.environ["B200ZK_MSM_WINDOW"]
    _check_point(got, want, "+-G bucket collisions %s seg_len=%d" % ("G2" if g2 else "G1", seg_len))


# ---- 1. size ladder, default configuration ------------------------------------------------------------------------
def _spot_check_points(bases, seed, g2):
    n = bases.shape[0]
    rng = np.random.default_rng(n)
    cnt = 64 if g2 else 256
    idx = np.unique(np.concatenate([[0, n - 1], rng.integers(0, n, cnt - 2)]))
    import torch
    got = _host(bases[torch.from_numpy(idx).to(bases.device)])
    logs = dl.base_logs(seed, n)[idx]
    curve, gen = (o.G2, o.G2_GEN) if g2 else (o.G1, o.G1_GEN)
    want = (layout.g2_to_arr if g2 else layout.g1_to_arr)([curve.mul(gen, int(k)) for k in logs])
    assert (got == want).all()


@pytest.mark.parametrize("g2,n", [(False, 1 << 20), (False, (1 << 22) + 1), (False, (1 << 23) - 1), (False, 1 << 24),
                                  (False, 1 << 26), (True, 1 << 20), (True, 1 << 22)])
def test_size_ladder_device_resident(net, g2, n):
    """also the window groups: one Horner step per group, 1 group below 2^22 and 4 from there up"""
    import torch
    seed = 0xA1000000 + n
    net.profile(True)
    net.profile_reset()
    bases = _check_generated(net, seed, n, g2, "default %s n=%d" % ("G2" if g2 else "G1", n))
    rep = net.profile_report()
    net.profile(False)
    assert rep["msm_combine"]["launches"] == (4 if n >= 1 << 22 else 1), rep["msm_combine"]
    _spot_check_points(bases, seed, g2)
    del bases
    torch.cuda.empty_cache()


@pytest.mark.parametrize("g2", [False, True])
@pytest.mark.parametrize("log_n", [20, 22])
def test_size_ladder_host_staged(net, g2, log_n):
    """b200zk_msm_g1/g2 on host buffers: five input parts adding into one bucket set"""
    net.profile(True)
    net.profile_reset()
    _check_generated(net, 0xA2000000 + log_n, 1 << log_n, g2, "host-staged log_n=%d" % log_n, staged=True)
    rep = net.profile_report()
    net.profile(False)
    assert rep["msm_digits"]["launches"] == 5                 # one sort per part


@pytest.mark.parametrize("g2", [False, True], ids=["g1", "g2"])
def test_host_staged_tiny(net, g2):
    """host-staged MSMs of 1, 5 and 15 pairs: one part each"""
    for n in (1, 5, 15):
        _check_generated(net, 0xB2000000 + n, n, g2, "tiny %s n=%d host-staged" % ("G2" if g2 else "G1", n), staged=True)


def test_fixed_base_table_2_22_c20(net):
    import torch
    n, seed = 1 << 22, 0xA3000022
    bases = net.generate_g1(seed, n)
    scalars = net.generate_fr(seed, n)
    sh = _host(scalars)
    _assert_canonical(sh)
    table = net.msm_table_build(bases, 20)
    del bases
    got = net.sum_points_dev(net.msm_table_dev(table, scalars, 20), 1)
    _check_point(got, dl.expected_msm(seed, sh), "fixed-base table n=2^22 c=20")
    del table
    torch.cuda.empty_cache()


# ---- 2. window sweep ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", G1_WINDOWS)
def test_window_sweep_g1(net, c):
    _sweep_one(net, c, False)


@pytest.mark.parametrize("c", G2_WINDOWS)
def test_window_sweep_g2(net, c):
    _sweep_one(net, c, True, big=False)


# ---- 3. adversarial bucket contents ---------------------------------------------------------------------------------
@pytest.mark.parametrize("g2", [False, True])
def test_one_point_many_times(net, g2):
    """one point 2^16 + 5 times with one scalar: one giant bucket per window whose tasks all have the same sum"""
    import torch
    n, seed = (1 << 16) + 5, 0xA4000001
    p = net.generate_g2(seed, 1) if g2 else net.generate_g1(seed, 1)
    s = net.generate_fr(seed, 1)
    bases, scalars = p.repeat(n, 1).contiguous(), s.repeat(n, 1).contiguous()
    k0 = dl.base_logs(seed, 1)
    want = dl.point_from_exponent(dl.exponent(np.repeat(k0, n), _host(scalars)), g2)
    _check_point(_msm_dev(net, bases, scalars, g2), want, "one point n times")
    # the same point with alternating P, -P and one scalar, and with s, r - s: both sum to infinity
    neg = torch.from_numpy(_neg_points(_host(p), g2).view(np.int64)).to(p.device)
    alt = torch.cat([p, neg]).repeat(n // 2, 1).contiguous()
    got = _msm_dev(net, alt, s.repeat(alt.shape[0], 1).contiguous(), g2)
    assert got[1], "P and -P with one scalar must give infinity"
    sv = layout.arr_to_fr(_host(s))[0]
    pair = torch.from_numpy(layout.fr_to_arr([sv, o.R - sv]).view(np.int64)).to(p.device)
    got = _msm_dev(net, bases[: 2 * (n // 2)].contiguous(), pair.repeat(n // 2, 1).contiguous(), g2)
    assert got[1], "s and r - s on one point must give infinity"


def _neg_points(arr, g2):
    pts = (layout.arr_to_g2 if g2 else layout.arr_to_g1)(arr)
    curve = o.G2 if g2 else o.G1
    return (layout.g2_to_arr if g2 else layout.g1_to_arr)([curve.neg(q) for q in pts])


@pytest.mark.parametrize("g2", [False, True])
def test_bucket_running_sum_collisions_quad_reduce(net, g2):
    check_collisions(net, g2, seg_len=8)                  # small bucket sets: one quad per 8-bucket segment


@pytest.mark.parametrize("g2", [False, True], ids=["g1", "g2"])
def test_bucket_running_sum_collisions_thread_reduce(net, g2):
    """c = 16: 2 x 8 GLV bucket sets of 2048 16-bucket segments, more than the 8192 the quad reduction takes, so one thread
    reduces each 16-bucket segment"""
    c, seg_len = 16, 16
    assert 2 * (-(-128 // c)) * ((1 << (c - 1)) // seg_len) > 8192
    check_collisions(net, g2, seg_len, c=c)


def test_size_guard_refuses_before_launch(net, monkeypatch):
    """c = 2 gives W = 128 digit windows: 2^25 points make W * n = 2^32 entries, past the 32-bit offsets"""
    import torch
    from distributed_groth16_b200 import B200zkError
    n = 1 << 25
    bases = net.generate_g1(7, n)
    scalars = net.generate_fr(7, n)
    monkeypatch.setenv("B200ZK_MSM_WINDOW", "2")
    with pytest.raises(B200zkError):
        net.msm_dev(bases, scalars)
    del bases, scalars
    torch.cuda.empty_cache()


# ---- 4. fixed-base tables: window sweep, G2 at 2^20, the fold guard -----------------------------------------------------
TABLE_G1_WINDOWS = list(range(2, 25))
TABLE_G2_WINDOWS = list(range(2, 21))
PROVER_TABLE_WINDOWS = (7, 16, 22)           # B200ZK_PK_TABLE_WINDOW in test_gpu_prove_exact.py (32-bucket segment hint)


def table_seg_len(c, hint=0):
    """segment length of a fixed-base table MSM (one bucket set), as msm_dev_impl picks it"""
    B = 1 << (c - 1)
    seg = min(B, 16)
    if B // seg <= 8192:                     # quad reduction: 8-bucket segments whatever the hint
        return min(B, 8)
    return hint if hint and hint <= B else seg


def table_wsplit(c, seg_len):
    """blocks that sum the segment partials of the single bucket set (msm_dev_impl, `wsplit`)"""
    nseg = (1 << (c - 1)) // seg_len
    return 16 if nseg >= 16 * 256 else (4 if nseg >= 1024 else 1)


def test_table_sweep_reaches_every_wsplit():
    pairs = [(c, table_seg_len(c)) for c in TABLE_G1_WINDOWS] + [(c, table_seg_len(c, 32)) for c in PROVER_TABLE_WINDOWS]
    assert {table_wsplit(c, s) for c, s in pairs} == {1, 4, 16}, pairs
    assert {table_wsplit(c, table_seg_len(c)) for c in TABLE_G2_WINDOWS} == {1, 4, 16}


def _table_msm(net, bases, scalars, c, g2):
    table = net.msm_table_build(bases, c, g2=g2)
    return net.sum_points_dev(net.msm_table_dev(table, scalars, c, g2=g2), 1, g2=g2)


def _table_sweep_one(net, c, g2):
    import torch
    what = "table %s c=%d wsplit=%d" % ("G2" if g2 else "G1", c, table_wsplit(c, table_seg_len(c)))
    for n in (3001, 40000):
        seed = 0xD0000000 + 1000 * c + n % 997 + (1 << 20) * g2
        bases = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
        scalars = net.generate_fr(seed ^ 0x7AB1E, n)
        _check_point(_table_msm(net, bases, scalars, c, g2), dl.expected_msm(seed, _host(scalars), g2), "%s n=%d" % (what, n))
    fams = dl.digit_families(c, glv=False)
    seed = 0xD8000000 + c + (1 << 20) * g2
    cnt = max(len(v) for v in fams.values())
    bases = net.generate_g2(seed, cnt) if g2 else net.generate_g1(seed, cnt)
    for name, ks in fams.items():
        sc = layout.fr_to_arr(ks)
        got = _table_msm(net, bases[: len(ks)].contiguous(), torch.from_numpy(sc.view(np.int64)).to(bases.device), c, g2)
        _check_point(got, dl.expected_msm(seed, sc, g2), "%s family %s" % (what, name))


@pytest.mark.parametrize("c", TABLE_G1_WINDOWS)
def test_table_window_sweep_g1(net, c):
    _table_sweep_one(net, c, False)


@pytest.mark.parametrize("c", TABLE_G2_WINDOWS)
def test_table_window_sweep_g2(net, c):
    _table_sweep_one(net, c, True)


def test_fixed_base_table_g2_2_20_c20(net):
    import torch
    n, seed = 1 << 20, 0xA3000020
    bases = net.generate_g2(seed, n)
    scalars = net.generate_fr(seed, n)
    got = _table_msm(net, bases, scalars, 20, True)
    _check_point(got, dl.expected_msm(seed, _host(scalars), True), "fixed-base table G2 n=2^20 c=20")
    del bases
    torch.cuda.empty_cache()


def test_table_fold_guard_refuses_before_launch(net):
    """c = 2 has 128 windows: 2^24 scalars make W * n = 2^31 table entries, past the fold path's 31-bit entry indices.
    msm_dev_impl refuses before it allocates or launches anything, so the table buffer here is a placeholder."""
    import ctypes
    import torch
    from distributed_groth16_b200 import _native
    n = 1 << 24
    assert net.msm_table_windows(2) * n == 1 << 31
    scalars = net.generate_fr(11, n)
    table = torch.zeros((16, 8), dtype=torch.int64, device=scalars.device)
    out = torch.empty(16, dtype=torch.int64, device=scalars.device)
    rc = net._lib.b200zk_msm_table_dev(net._h, 0, 0, ctypes.c_void_p(table.data_ptr()), ctypes.c_void_p(scalars.data_ptr()), n, 2,
                                       ctypes.c_void_p(out.data_ptr()))
    assert rc == _native.ERR_ARG, rc
    assert "W * n" in net._lib.b200zk_last_error(net._h).decode()
    del scalars
    torch.cuda.empty_cache()
