"""The R1CS -> QAP mat-vec (csrc/qap.cu) and the setup's Fr and fixed-base kernels (csrc/setup.cu, csrc/packexp.cu) against
exact answers.

Every result is compared word for word with an answer computed without the library: the CPU twin (oracle/cref.py:
fr_spmv, qap, fixed_base_mul, the MSM, the point generator), Python ints, or the known-log identity of tests/dlog_oracle.py
(Net.generate_g1/g2(seed, n) are k_i G with known k_i).  Device outputs start as all-ones words, so a row a kernel never
writes cannot pass as zero.  Covered here:
  - qap_dev through ConstraintMatrices and groth16.qap.qap on both kernels: one warp per row (m <= 2^18) and one thread per
    row (above), m = 2^0 .. 2^24; row lengths 0, 1, 2, 31, 32, 33, 64, 65 and one row of 2^16 terms on both; coefficients
    0, 1, r - 1 and full width; full-width and sha256-like (0 / 1) witnesses; every padding case (none, one row, nc = 0,
    n_inputs 1, 2, 17 and 2^18 + 1, an empty B row under a non-empty A row); the three coefficient encodings (r1cs
    canonical, Montgomery, zkey x R^2); the ERR_DOMAIN refusals, before any launch;
  - r1cs_check_dev at full width on both kernels, with planted failures counted and located;
  - fr_spmv_dev, fr_lincomb_dev (with the aliased call (a, b, a)), fr_powers_dev and fr_convert_dev (in place too);
  - fixed_base_mul_dev on G1 and G2: every table entry, edge scalars, 2^20 / 2^18 points by the known-log identity, and the
    lazily built tables of a fresh context;
  - points_matmul_dev on G1 and G2 at non-square shapes with infinity points and 0 / 1 / r - 1 entries, and its ERR_ARG
    guards, before any launch;
  - circom.prove_from_matrices at m = 2^20 (the thread-per-row QAP kernel) against the exact proof of a known-log key, and
    at m = 2^19 from zkey bytes.
A failure names the kernel, the size and the case.

Measured on one H100 80GB HBM3 at a 700 W power limit: 106 s and 117 s for the file in two runs, most of it host-side (the
zkey writer at 2^19, the 2^24 matrices and the 2^24 Python-int power chain)."""
import os
import sys

import numpy as np
import pytest

from distributed_groth16_b200._native import ERR_ARG, ERR_DOMAIN, c_vp
from oracle import bn254 as o, layout

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import dlog_oracle as dl          # noqa: E402
import prove_dlog_oracle as po    # noqa: E402

pytestmark = pytest.mark.gpu
R = o.R
MASK64 = (1 << 64) - 1
R_TOP = np.uint64(R >> 192)
SPECIAL_LENGTHS = (0, 1, 2, 31, 32, 33, 64, 65)
LONG_ROW = 1 << 16
WARP_PATH_MAX = 1 << 18                 # qap_dev and r1cs_check_dev: one warp per row up to here, one thread per row above


# ---- helpers ----------------------------------------------------------------------------------------------------------
def raw(vals) -> np.ndarray:
    """ints -> (n, 4) u64 words as given (no Montgomery conversion)"""
    return np.array([[(int(v) >> (64 * i)) & MASK64 for i in range(4)] for v in vals], dtype=np.uint64).reshape(-1, 4)


def mont(vals) -> np.ndarray:
    return layout.fr_to_arr([int(v) for v in vals])


ZERO_M, ONE_M, MINUS_ONE_M = mont([0, 1, R - 1])
R2_RAW = raw([o.MONT_R * o.MONT_R % R])[0]
ONE_RAW = raw([1])[0]


def rand_words(rng, n) -> np.ndarray:
    """(n, 4) field elements below r, every limb full width (the top limb reduced below r's)"""
    w = rng.integers(0, 1 << 64, (n, 4), dtype=np.uint64, endpoint=False)
    w[:, 3] %= R_TOP
    return w


def mul_const(cref, vals, k_raw) -> np.ndarray:
    """Montgomery product of every row with the constant k (raw words), by the CPU twin's mat-vec with one term per row:
    k = R^2 turns values into Montgomery form, k = 1 takes them out"""
    vals = np.ascontiguousarray(vals, dtype=np.uint64).reshape(-1, 4)
    n = vals.shape[0]
    return cref.fr_spmv(np.arange(n + 1, dtype=np.uint32), np.zeros(n, dtype=np.uint32), vals, np.asarray(k_raw).reshape(1, 4))


def host(t) -> np.ndarray:
    return t.cpu().numpy().view(np.uint64)


def filled(net, shape):
    """a device tensor of all-ones words"""
    import torch
    return torch.full(shape, -1, dtype=torch.int64, device=net._dev())


def assert_rows(got, want, what):
    got = np.asarray(got, dtype=np.uint64).reshape(want.shape[0], -1)
    want = np.asarray(want, dtype=np.uint64).reshape(want.shape[0], -1)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, "%s: %d of %d rows differ, first %s" % (what, bad.size, want.shape[0], bad[:8].tolist())


# ---- the CSR generator shared by qap_dev, r1cs_check_dev and fr_spmv_dev ------------------------------------------------------
def make_csr(rng, n_rows, n_vars, mean=2.0, long_row=True, empty_rows=()):
    """(ptr u32, idx u32, val (nnz, 4) Montgomery) with Poisson(mean) terms per row, the SPECIAL_LENGTHS at rows 1.. and at
    the last rows, a row of LONG_ROW terms at n_rows // 2 (when n_rows >= 32), `empty_rows` without terms; columns 0 and
    n_vars - 1 both used, row 3 (two terms) holding one (row, col) pair twice; coefficients 0, 1, r - 1 (10 % each) and
    full width"""
    cnt = rng.poisson(mean, n_rows).astype(np.int64)
    if n_rows:
        cnt[0] = 3
    k = min(len(SPECIAL_LENGTHS), n_rows - 1)
    if k > 0:
        cnt[1:1 + k] = SPECIAL_LENGTHS[:k]
    if n_rows > 3 * len(SPECIAL_LENGTHS):
        cnt[-len(SPECIAL_LENGTHS):] = SPECIAL_LENGTHS           # the last row has 65 terms
    if long_row and n_rows >= 32:
        cnt[n_rows // 2] = LONG_ROW
    cnt[list(empty_rows)] = 0
    ptr = np.zeros(n_rows + 1, dtype=np.int64)
    ptr[1:] = np.cumsum(cnt)
    nnz = int(ptr[-1])
    assert nnz < 1 << 32
    idx = rng.integers(0, n_vars, nnz, dtype=np.uint32)
    val = rand_words(rng, nnz)
    pick = rng.random(nnz)
    val[pick < 0.1] = ZERO_M
    val[(pick >= 0.1) & (pick < 0.2)] = ONE_M
    val[(pick >= 0.2) & (pick < 0.3)] = MINUS_ONE_M
    if n_rows:
        idx[0], idx[1], idx[2] = 0, n_vars - 1, 0                # row 0: both end columns
        val[0], val[1] = rand_words(rng, 2)
    if n_rows > 3 and cnt[3] == 2:
        idx[ptr[3] + 1] = idx[ptr[3]]                            # one (row, col) pair twice
    return ptr.astype(np.uint32), idx, val


def coo(csr):
    ptr, idx, val = csr
    return np.repeat(np.arange(ptr.shape[0] - 1, dtype=np.uint32), np.diff(ptr.astype(np.int64))), idx, val


def witness(rng, n, kind, seed):
    if kind == "0/1":
        return po.sha256_like_witness(n, seed)
    z = rand_words(rng, n)
    z[0] = ONE_M
    return z


def encode(cref, val, depth):
    """coefficients as ConstraintMatrices takes them at values_montgomery_depth `depth`: -1 canonical, 0 Montgomery, 1 times
    R^2 (zkey)"""
    if depth < 0:
        return mul_const(cref, val, ONE_RAW)
    return mul_const(cref, val, R2_RAW) if depth > 0 else val


# ---- qap_dev ------------------------------------------------------------------------------------------------------------
def run_qap(net, mats, z_dev, log_m):
    """b200zk_qap_dev into all-ones outputs, and groth16.qap.qap on the same matrices; both must agree"""
    from distributed_groth16_b200.groth16.qap import qap
    m = 1 << log_m
    nc, ni = mats.num_constraints, mats.num_instance_variables
    outs = [filled(net, (m, 4)) for _ in range(3)]
    (ap, ac, av), (bp, bc, bv) = mats.csr
    net.check(net._lib.b200zk_qap_dev(net._h, 0, c_vp(ap.data_ptr()), c_vp(ac.data_ptr()), c_vp(av.data_ptr()),
                                      c_vp(bp.data_ptr()), c_vp(bc.data_ptr()), c_vp(bv.data_ptr()), nc, ni,
                                      c_vp(z_dev.data_ptr()), log_m, *(c_vp(t.data_ptr()) for t in outs)))
    got = [host(t) for t in outs]
    q = qap(mats, z_dev, net)
    assert q.domain.size() == m
    for name, g, t in zip("abc", got, (q.a, q.b, q.c)):
        assert_rows(host(t), g, "groth16.qap.qap vs b200zk_qap_dev, vector %s" % name)
    return got


# (log_m, nc, n_inputs, n_vars, witness, mean terms per row)
QAP_CASES = {
    "m=2^0 nc=0": (0, 0, 1, 1, "random", 2.0),
    "m=2^1": (1, 1, 1, 3, "random", 2.0),
    "m=2^5 no padding": (5, 31, 1, 40, "random", 2.0),
    "m=2^5 n_inputs=17": (5, 14, 17, 50, "0/1", 2.0),
    "m=2^5 nc=0 n_inputs=17": (5, 0, 17, 17, "random", 2.0),
    "m=2^10 one below 2^10": (10, 1021, 2, 700, "random", 2.0),
    "m=2^18 no padding": (18, (1 << 18) - 2, 2, 1 << 17, "random", 2.0),
    "m=2^18 n_inputs=17 0/1": (18, 200000, 17, 150000, "0/1", 2.0),
    "m=2^19 one below 2^19": (19, (1 << 19) - 18, 17, 1 << 19, "random", 2.0),
    "m=2^19 nc=0": (19, 0, (1 << 18) + 1, (1 << 18) + 1, "random", 2.0),
    "m=2^19 no padding 0/1": (19, (1 << 19) - 1, 1, 3000, "0/1", 2.0),
    "m=2^20 0/1": (20, (1 << 20) - 2, 2, 1 << 19, "0/1", 2.0),
    "m=2^22": (22, 3000000, 1, 1 << 21, "random", 2.0),
    "m=2^24": (24, (1 << 24) - 2, 2, 1 << 22, "random", 1.5),
}


@pytest.mark.parametrize("case", list(QAP_CASES))
def test_qap_dev(net, cref, case):
    from distributed_groth16_b200.groth16.qap import ConstraintMatrices
    log_m, nc, ni, n_vars, wkind, mean = QAP_CASES[case]
    assert (nc + ni > (1 << log_m) // 2 or log_m == 0) and nc + ni <= 1 << log_m
    rng = np.random.default_rng(0x9A9 + log_m * 1000 + nc)
    a_csr = make_csr(rng, nc, n_vars, mean)
    b_csr = make_csr(rng, nc, n_vars, mean, long_row=False, empty_rows=[nc - 1] if nc > 24 else [])
    if nc > 24:
        assert a_csr[0][nc] > a_csr[0][nc - 1] and b_csr[0][nc] == b_csr[0][nc - 1]       # B's last row empty, A's not
    z = witness(rng, n_vars, wkind, 0x9A90 + log_m)
    want = cref.qap(a_csr, b_csr, z, nc, ni, 1 << log_m)
    mats = ConstraintMatrices(net, ni, nc, coo(a_csr), coo(b_csr), values_montgomery_depth=0)
    got = run_qap(net, mats, net.to_device(z), log_m)
    path = "warp" if (1 << log_m) <= WARP_PATH_MAX else "thread"
    for name, g, w in zip("abc", got, want):
        assert_rows(g, w, "qap_dev %s (%s path) vector %s" % (case, path, name))


@pytest.mark.parametrize("log_m", [10, 19])
def test_qap_dev_coefficient_encodings_agree(net, cref, log_m):
    """The same matrix as r1cs values (canonical, depth -1), Montgomery (0) and zkey values (x R^2, depth 1)."""
    from distributed_groth16_b200.groth16.qap import ConstraintMatrices
    m = 1 << log_m
    nc, ni, n_vars = m - 3, 3, m // 4
    rng = np.random.default_rng(0xE7C + log_m)
    a_csr, b_csr = make_csr(rng, nc, n_vars), make_csr(rng, nc, n_vars, long_row=False)
    z = witness(rng, n_vars, "random", 0)
    want = cref.qap(a_csr, b_csr, z, nc, ni, m)
    z_dev = net.to_device(z)
    for depth in (-1, 0, 1):
        ea, eb = ((r, c, encode(cref, v, depth)) for r, c, v in (coo(a_csr), coo(b_csr)))
        got = run_qap(net, ConstraintMatrices(net, ni, nc, ea, eb, values_montgomery_depth=depth), z_dev, log_m)
        for name, g, w in zip("abc", got, want):
            assert_rows(g, w, "qap_dev m=2^%d values_montgomery_depth=%d vector %s" % (log_m, depth, name))


def test_qap_dev_refuses_before_any_launch(net):
    import torch
    dummy = torch.zeros((64, 4), dtype=torch.int64, device=net._dev())
    p = c_vp(dummy.data_ptr())
    for nc, ni, log_m in ((0, 1, 29), (1, 0, 40), (10, 7, 4), (17, 0, 4), (0, 17, 4), ((1 << 20), 1, 20)):
        before = net.launch_count()
        rc = net._lib.b200zk_qap_dev(net._h, 0, p, p, p, p, p, p, nc, ni, p, log_m, p, p, p)
        assert rc == ERR_DOMAIN, (nc, ni, log_m, rc)
        assert net.launch_count() == before, (nc, ni, log_m)
    assert "domain" in net._lib.b200zk_last_error(net._h).decode()


# ---- r1cs_check_dev at full width ------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [16, 20])
def test_r1cs_check_dev_full_width(net, cref, log_n):
    """A, B full width, C one term per row at column 0 (w[0] = 1) holding the twin's a_i b_i.  2^16 rows take the
    warp-per-row kernel, 2^20 the thread-per-row one."""
    from distributed_groth16_b200.groth16 import snarkjs
    n, n_vars = 1 << log_n, 1 << 15
    rng = np.random.default_rng(0xC4EC + log_n)
    a_csr, b_csr = make_csr(rng, n, n_vars), make_csr(rng, n, n_vars, long_row=False)
    w = witness(rng, n_vars, "random", 0)
    a = cref.fr_spmv(*a_csr, w)
    b = cref.fr_spmv(*b_csr, w)
    diag = np.arange(n + 1, dtype=np.uint32)
    c = cref.fr_spmv(diag, diag[:n], a, b)
    long_row = n // 2
    assert int(a_csr[0][long_row + 1]) - int(a_csr[0][long_row]) == LONG_ROW
    c_ptr, c_idx = diag, np.zeros(n, dtype=np.uint32)
    dev = lambda p, i, v: (net.to_device(p.view(np.int32)), net.to_device(i.view(np.int32)), net.to_device(v))
    A, B = dev(*a_csr), dev(*b_csr)
    w_dev = net.to_device(w)
    assert snarkjs.r1cs_check(net, [A, B, dev(c_ptr, c_idx, c)], w_dev, n) == (0, n), "every row holds"
    run = np.arange(n // 3, n // 3 + 300)
    for planted in (np.array([0]), np.array([n - 1]), run, np.array([long_row]),
                    np.concatenate([[0, 5, long_row], run, [n - 1]])):
        planted = np.unique(planted)
        bad = c.copy()
        bad[planted, 0] ^= np.uint64(2)
        assert (bad[planted] != c[planted]).any(axis=1).all()
        got = snarkjs.r1cs_check(net, [A, B, dev(c_ptr, c_idx, bad)], w_dev, n)
        assert got == (planted.size, int(planted[0])), ("r1cs_check_dev n=2^%d" % log_n, planted[:4].tolist(), got)


# ---- fr_spmv_dev ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [10, 14, 18, 22])
def test_fr_spmv_dev(net, cref, log_n):
    n = 1 << log_n
    n_vars = n // 2 + 7
    rng = np.random.default_rng(0x5B3 + log_n)
    ptr, idx, val = make_csr(rng, n, n_vars, empty_rows=[n - 5])
    x = witness(rng, n_vars, "random", 0)
    want = cref.fr_spmv(ptr, idx, val, x)
    out = filled(net, (n, 4))
    d = [net.to_device(ptr.view(np.int32)), net.to_device(idx.view(np.int32)), net.to_device(val), net.to_device(x)]
    net.check(net._lib.b200zk_fr_spmv_dev(net._h, *(c_vp(t.data_ptr()) for t in d), n, c_vp(out.data_ptr())))
    assert_rows(host(out), want, "fr_spmv_dev n=2^%d" % log_n)


# ---- fr_lincomb_dev ---------------------------------------------------------------------------------------------------
LINCOMB_S = {
    "distinct": [0x1111 * 3 + 1, 0x2222 * 5 + 7, (1 << 200) + 0x33, R - 12345],
    "zeros and r-1": [R - 1, 0, 5, R - 1],
    "scale zero": [7, 11, 13, 0],
}


def lincomb_dev(net, a, b, c, s, n):
    out = filled(net, (n, 4))
    sl = mont(s).reshape(-1)
    net.check(net._lib.b200zk_fr_lincomb_dev(net._h, c_vp(a.data_ptr()), c_vp(b.data_ptr()), c_vp(c.data_ptr()),
                                             c_vp(sl.ctypes.data), n, c_vp(out.data_ptr())))
    return host(out)


def lincomb_expected(cref, a, b, c, s, sample=None):
    """(a s0 + b s1 + c s2) s3: Python ints on `sample` rows (all when None); the twin's three-term mat-vec for the rest"""
    n = a.shape[0]
    if sample is not None:
        rows = [layout.arr_to_fr(v[sample]) for v in (a, b, c)]
        return mont([(x * s[0] + y * s[1] + z * s[2]) * s[3] for x, y, z in zip(*rows)])
    ptr = np.arange(0, 3 * n + 1, 3, dtype=np.uint32)
    idx = (np.arange(n, dtype=np.uint32)[:, None] + np.array([0, n, 2 * n], dtype=np.uint32)).reshape(-1)
    val = np.tile(mont([s[0] * s[3], s[1] * s[3], s[2] * s[3]]), (n, 1))
    return cref.fr_spmv(ptr, idx, val, np.concatenate([a, b, c]))


@pytest.mark.parametrize("n", [1, 255, 256, 257, 1 << 20])
def test_fr_lincomb_dev(net, cref, n):
    rng = np.random.default_rng(0x71C + n)
    a, b, c = (rand_words(rng, n) for _ in range(3))
    for v, k in ((a, 0), (b, 1), (c, 2)):
        v[:3][k % min(n, 3)] = (ZERO_M, ONE_M, MINUS_ONE_M)[k]
    da, db, dc = (net.to_device(v) for v in (a, b, c))
    sample = np.unique(np.concatenate([[0, n - 1], rng.integers(0, n, 64)])) if n > 257 else np.arange(n)
    for sname, s in LINCOMB_S.items():
        for call, (x, y, zz, hx, hy, hz) in (("(a, b, c)", (da, db, dc, a, b, c)), ("aliased (a, b, a)", (da, db, da, a, b, a))):
            got = lincomb_dev(net, x, y, zz, s, n)
            what = "fr_lincomb_dev n=%d s=%s %s" % (n, sname, call)
            assert_rows(got[sample], lincomb_expected(cref, hx, hy, hz, s, sample), what + " (Python ints)")
            if n > 257:
                assert_rows(got, lincomb_expected(cref, hx, hy, hz, s), what)


# ---- fr_powers_dev ----------------------------------------------------------------------------------------------------
OMEGA_LOG = 10
POWERS_CASES = {
    "(0, s)": (0, 0xABCDEF12345),
    "(1, s)": (1, R - 77),
    "(r-1, s)": (R - 1, 0x5555 << 180),
    "(omega_2^10, 1)": (o.fr_root_of_unity(1 << OMEGA_LOG), 1),
    "(random, 0)": (0x1F2E3D4C5B6A79881726354453627180 * 0x9ABC % R, 0),
    "(random, random)": (0x0123456789ABCDEF0123456789ABCDEF01 * 0x77 % R, (1 << 251) + 0x5EED),
}
_CHAIN = {}


def powers_chain(base, scale, n) -> np.ndarray:
    """scale base^i, i < n, as Montgomery limbs from the iterative Python-int chain y_{i+1} = y_i base (y in Montgomery
    form); cached per case at the longest n asked"""
    key = (base, scale)
    if key not in _CHAIN or _CHAIN[key].shape[0] < n:
        y, out = scale * o.MONT_R % R, bytearray()
        for _ in range(n):
            out += y.to_bytes(32, "little")
            y = y * base % R
        _CHAIN[key] = np.frombuffer(bytes(out), dtype=np.uint64).reshape(n, 4)
    return _CHAIN[key][:n]


def powers_expected(case, n) -> np.ndarray:
    base, scale = POWERS_CASES[case]
    if case == "(0, s)":
        out = np.zeros((n, 4), dtype=np.uint64)
        out[0] = mont([scale])[0]
        return out
    if case == "(1, s)":
        return np.tile(mont([scale]), (n, 1))
    if case == "(r-1, s)":
        return np.tile(mont([scale, R - scale]), ((n + 1) // 2, 1))[:n]
    if case == "(random, 0)":
        return np.zeros((n, 4), dtype=np.uint64)
    if case == "(omega_2^10, 1)":
        period = powers_chain(base, scale, 1 << OMEGA_LOG)
        return np.tile(period, ((n >> OMEGA_LOG) + 1, 1))[:n]
    return powers_chain(base, scale, n)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 1 << 20, 1 << 24])
def test_fr_powers_dev(net, n):
    for case, (base, scale) in POWERS_CASES.items():
        out = filled(net, (n, 4))
        b, s = mont([base])[0], mont([scale])[0]
        net.check(net._lib.b200zk_fr_powers_dev(net._h, c_vp(b.ctypes.data), c_vp(s.ctypes.data), n, c_vp(out.data_ptr())))
        got = host(out)
        assert_rows(got, powers_expected(case, n), "fr_powers_dev n=%d %s" % (n, case))
        if case.startswith("(omega") and n > 1 << OMEGA_LOG:
            assert (got[1 << (OMEGA_LOG - 1)] == MINUS_ONE_M).all() and (got[1 << OMEGA_LOG] == ONE_M).all()
    if n == 1 << 24:
        _CHAIN.clear()


# ---- fr_convert_dev ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 255, 256, 257, 1 << 20])
def test_fr_convert_dev(net, cref, n):
    import torch
    rng = np.random.default_rng(0xC0 + n)
    x = rand_words(rng, n)
    if n > 3:                                                 # n = 1 keeps a full-width value: 0 converts to itself
        x[:3] = raw([0, 1, R - 1])
    dx = net.to_device(x)
    for to_mont in (0, 1):
        want = x
        for times in range(4):
            what = "fr_convert_dev n=%d to_mont=%d times=%d" % (n, to_mont, times)
            out = filled(net, (n, 4))
            net.check(net._lib.b200zk_fr_convert_dev(net._h, 0, c_vp(dx.data_ptr()), c_vp(out.data_ptr()), n, to_mont, times))
            assert_rows(host(out), want, what)
            inplace = dx.clone()
            net.check(net._lib.b200zk_fr_convert_dev(net._h, 0, c_vp(inplace.data_ptr()), c_vp(inplace.data_ptr()), n, to_mont,
                                                     times))
            assert_rows(host(inplace), want, what + " in place")
            want = mul_const(cref, want, R2_RAW if to_mont else ONE_RAW)
    assert torch.equal(dx, net.to_device(x)), "the input was modified"
    if n > 3:                                                 # the first rows against Python ints
        conv = net.fr_convert(dx, to_mont=True, times=2)
        assert layout.arr_to_fr(host(conv)[:3]) == [0, o.MONT_R % R, (R - 1) * o.MONT_R % R]


# ---- fixed_base_mul_dev -----------------------------------------------------------------------------------------------
def gen_arr(g2):
    return layout.g2_to_arr([o.G2_GEN])[0] if g2 else layout.g1_to_arr([o.G1_GEN])[0]


def fixed_base_dev(net, scalars_m, g2, n=None):
    n = scalars_m.shape[0] if n is None else n
    out = filled(net, (max(n, 1), 16 if g2 else 8))
    sc = net.to_device(scalars_m) if scalars_m.shape[0] else filled(net, (1, 4))
    net.check(net._lib.b200zk_fixed_base_mul_dev(net._h, int(g2), c_vp(sc.data_ptr()), n, c_vp(out.data_ptr())))
    return out


def table_and_edge_scalars(rng):
    """d 16^w for every table entry (d in 1..15, w < 64, below r), then the edge scalars and random ones"""
    table = [d << (4 * w) for w in range(64) for d in range(1, 16) if d << (4 * w) < R]
    assert len(table) == 63 * 15 + 3                      # window 63 holds d <= 3 only: 4 * 16^63 > r
    edges = [0, 1, R - 1, R - 2, (R - 1) // 2, (R + 1) // 2, 1 << 252, 3 << 252] + [(1 << (4 * w)) - 1 for w in range(1, 64)]
    return table + edges + [int.from_bytes(rng.bytes(32), "little") % R for _ in range(200)]


@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
def test_fixed_base_mul_dev_every_table_entry_and_edges(net, cref, g2):
    scalars = table_and_edge_scalars(np.random.default_rng(0xFB + g2))
    sm = mont(scalars)
    got = host(fixed_base_dev(net, sm, g2))
    want = cref.fixed_base_mul(gen_arr(g2), sm, g2=g2)
    bad = [scalars[i] for i in np.nonzero((got != want).any(axis=1))[0][:4]]
    assert not bad, "fixed_base_mul_dev %s: scalars %s" % ("G2" if g2 else "G1", [hex(s) for s in bad])
    assert not got[scalars.index(0)].any() and got[scalars.index(1)].tolist() == gen_arr(g2).tolist()


@pytest.mark.parametrize("g2,log_n", [(False, 20), (True, 18)], ids=["G1 2^20", "G2 2^18"])
def test_fixed_base_mul_dev_known_logs(net, cref, g2, log_n):
    """fixed_base_mul(k_i) == generate(seed, n) with k_i the generator's known logs; the first 4096 also against the twin's
    generator."""
    import torch
    n, seed = 1 << log_n, 0xF1BA5E + log_n
    logs = dl.base_logs(seed, n)
    k = np.zeros((n, 4), dtype=np.uint64)
    k[:, 0] = logs
    got = fixed_base_dev(net, mul_const(cref, k, R2_RAW), g2)
    gen = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
    diff = torch.nonzero((got != gen).any(dim=1)).reshape(-1)
    assert diff.numel() == 0, "fixed_base_mul_dev vs generate (%s, n=2^%d): %d rows differ, first %s" % (
        "G2" if g2 else "G1", log_n, diff.numel(), diff[:8].tolist())
    twin = (cref.g2_generate if g2 else cref.g1_generate)(seed, 4096)
    assert_rows(host(got[:4096]), twin, "fixed_base_mul_dev vs the twin's generator")


def test_fixed_base_mul_dev_lazy_tables_of_a_fresh_context(cref):
    """The first call of a fresh context has n = 0 (it builds the table and launches nothing else), the next n = 1; G1
    then G2 in the same context, then G1 again on the table it kept."""
    from distributed_groth16_b200 import Net
    fresh = Net(0)
    fresh.use_torch_stream(0)
    try:
        k = mont([0x1234567890ABCDEF1234567890ABCDEF * 31 % R])
        for g2, table_launches in ((False, 1), (True, 1), (False, 0)):
            what = "fresh context %s" % ("G2" if g2 else "G1")
            first = fresh.launch_count()
            fixed_base_dev(fresh, k[:0], g2, n=0)
            assert fresh.launch_count() - first == table_launches, what + ": n = 0 builds the table once and nothing else"
            got = host(fixed_base_dev(fresh, k, g2))
            assert_rows(got, cref.fixed_base_mul(gen_arr(g2), k, g2=g2), what)
            assert fresh.launch_count() - first == table_launches + 1, what
    finally:
        fresh.close()


# ---- points_matmul_dev ------------------------------------------------------------------------------------------------
# (n_chunks, l, rows); l = 1024 only with few rows, rows = 4096 only with l = 1
MATMUL_SHAPES = [(1, 1, 1), (7, 2, 5), (7, 3, 5), (1, 3, 2), (7, 5, 3), (1, 1024, 1), (1, 1024, 5), (1, 1, 4096), (7, 1, 4096)]


def matmul_dev(net, pts, n_chunks, l, matrix, rows, g2):
    out = filled(net, (n_chunks * rows, 16 if g2 else 8))
    dp, dm = net.to_device(pts), net.to_device(matrix)
    net.check(net._lib.b200zk_points_matmul_dev(net._h, 0, int(g2), c_vp(dp.data_ptr()), n_chunks, l, c_vp(dm.data_ptr()),
                                                rows, c_vp(out.data_ptr())))
    return host(out)


@pytest.mark.parametrize("g2", [False, True], ids=["G1", "G2"])
@pytest.mark.parametrize("shape", MATMUL_SHAPES, ids=["chunks=%d l=%d rows=%d" % s for s in MATMUL_SHAPES])
def test_points_matmul_dev(net, cref, shape, g2):
    n_chunks, l, rows = shape
    rng = np.random.default_rng(0x9A7 + 97 * n_chunks + 13 * l + rows + g2)
    pts = (cref.g2_generate if g2 else cref.g1_generate)(0x9A70 + l, n_chunks * l)
    pts[3::4] = 0                                                   # infinity points
    matrix = rand_words(rng, rows * l)
    matrix[: min(3, rows * l)] = np.stack([ZERO_M, ONE_M, MINUS_ONE_M])[: min(3, rows * l)]
    matrix[-1] = MINUS_ONE_M
    got = matmul_dev(net, pts, n_chunks, l, matrix, rows, g2).reshape(n_chunks, rows, -1)
    msm = cref.msm_g2 if g2 else cref.msm_g1
    m2 = matrix.reshape(rows, l, 4)
    for k in range(n_chunks):
        chunk = pts[k * l:(k + 1) * l]
        if l == 1:
            want = cref.fixed_base_mul(chunk[0], m2[:, 0], g2=g2)
        else:
            want = np.stack([msm(chunk, m2[j])[0] for j in range(rows)])
        assert_rows(got[k], want, "points_matmul_dev %s chunks=%d l=%d rows=%d, chunk %d" % ("G2" if g2 else "G1",
                                                                                            n_chunks, l, rows, k))


def test_points_matmul_dev_refuses_before_any_launch(net):
    dummy = filled(net, (64, 16))
    p = c_vp(dummy.data_ptr())
    for g2 in (0, 1):
        for n_chunks, l, rows in ((1, 0, 1), (3, 0, 5), (1, 1025, 1), (2, 1025, 3), (1, 1, 4097), (1, 3, 4097)):
            before = net.launch_count()
            rc = net._lib.b200zk_points_matmul_dev(net._h, 0, g2, p, n_chunks, l, p, rows, p)
            assert rc == ERR_ARG, (g2, n_chunks, l, rows, rc)
            assert net.launch_count() == before, (g2, n_chunks, l, rows)


# ---- end to end on the thread-per-row QAP kernel ----------------------------------------------------------------------
RS_RANDOM = (0x2F1E3D4C5B6A79881726354453627180 % R, 0x0A1B2C3D4E5F60718293A4B5C6D7E8F9 * 7 % R)


def test_prove_from_matrices_on_the_thread_path(net, cref):
    """m = 2^20, nc + n_inputs > 2^18: qap_dev runs k_qap.  The key is made of known-log points (prove_dlog_oracle.KeySpec),
    so the expected proof needs the twin's QAP and h, and no curve MSM."""
    import torch
    from distributed_groth16_b200.groth16 import ProvingKey, circom
    from distributed_groth16_b200.groth16.qap import ConstraintMatrices
    m, nc, ni, n_vars = 1 << 20, 700000, 3, 1 << 19
    rng = np.random.default_rng(0xE2E)
    a_csr, b_csr = make_csr(rng, nc, n_vars), make_csr(rng, nc, n_vars, long_row=False, empty_rows=[nc - 1])
    z = witness(rng, n_vars, "random", 0)
    h = cref.h_circom(*cref.qap(a_csr, b_csr, z, nc, ni, m))
    spec = po.KeySpec(m, n_vars, ni, 0xE2E000)
    pts = spec.device_points(net)
    pk = ProvingKey.from_device(net, pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], ni, po.vk_array(pts))
    del pts
    mats = ConstraintMatrices(net, ni, nc, coo(a_csr), coo(b_csr), values_montgomery_depth=0)
    z_dev = net.to_device(z)
    e = po.exponents(spec, z, h)
    try:
        for r, s in ((0, 0), RS_RANDOM):
            got = circom.prove_from_matrices(pk, mats, z_dev, mont([r])[0], mont([s])[0])
            assert got == po.proof_bytes(e, r, s), "prove_from_matrices m=2^20 r=%#x s=%#x" % (r, s)
    finally:
        pk.free()
        torch.cuda.empty_cache()


def test_prove_zkey_bytes_on_the_thread_path(net, cref):
    """m = 2^19 through zkey bytes (tests/artefact_writer.py): the coefficients are stored times R^2 and turned back into
    Montgomery form on the device (values_montgomery_depth = 1) before qap_dev runs k_qap."""
    import artefact_writer as aw
    import torch
    from distributed_groth16_b200.groth16 import circom
    m, nc, n_public, n_vars = 1 << 19, 300000, 2, 1 << 18
    ni = n_public + 1
    rng = np.random.default_rng(0x2E19)
    a_csr, b_csr = make_csr(rng, nc, n_vars), make_csr(rng, nc, n_vars, long_row=False)
    z = witness(rng, n_vars, "0/1", 0x2E19)
    h = cref.h_circom(*cref.qap(a_csr, b_csr, z, nc, ni, m))
    spec = po.KeySpec(m, n_vars, ni, 0x2E1900)
    pts = {k: v if isinstance(v, np.ndarray) else host(v) for k, v in spec.device_points(net).items()}
    d = dict(dims=np.array([n_vars, n_public, m, nc]), vk_g1=pts["vk1"], ic=cref.g1_generate(0x2E1901, ni),
             vk_g2=np.concatenate([pts["vk2"], layout.g2_to_arr([o.G2_GEN])]), a_query=pts["a"], b_g1_query=pts["b1"],
             b_g2_query=pts["b2"], l_query=pts["l"], h_query=pts["h"])
    for name, csr in (("a", a_csr), ("b", b_csr)):
        d[name + "_rows"], d[name + "_cols"], d[name + "_vals"] = coo(csr)
    pk, mats, zk = circom.load_zkey(net, aw.write_zkey(d))
    assert (mats.num_constraints, mats.num_instance_variables, pk.m) == (nc, ni, m)
    e = po.exponents(spec, z, h)
    try:
        for r, s in ((0, 0), RS_RANDOM):
            got = circom.prove_from_matrices(pk, mats, net.to_device(z), mont([r])[0], mont([s])[0])
            assert got == po.proof_bytes(e, r, s), "prove_from_matrices from zkey bytes m=2^19 r=%#x s=%#x" % (r, s)
    finally:
        pk.free()
        torch.cuda.empty_cache()
