"""The bucket reduction of the MSM (csrc/msm.cu, section 5) against exact answers from known discrete logs.

Bucket sets of more than 8192 segments are reduced in three launches: one thread per segment writes the pair
(R_s, A_s) = (sum of its L buckets, their running-sum total); k_msm_window_bits sums, per set, the A_s and for every bit
b of the segment index the R_s whose index has that bit set (C_b), each in `bsplit` parts, and doubles each C_b part
b + log2 L times; k_msm_window_sum adds a set's parts up to S_w = sum A_s + sum_b 2^(b + log2 L) C_b.  Covered here, each
against dlog_oracle's exact answer:
  - one segment per set (L = B: no C_b at all), 8 segments, 512 and 4096, through the segment-length override
    B200ZK_MSM_SEG; B <= L at c = 2..5 (the quad reduction);
  - bucket sets whose C_b sums are all empty (every digit in the lowest windows);
  - segment sums designed so that the sums of k_msm_window_bits add a point to its negative and to itself, checked by an
    integer model of the kernel first;
  - fixed-base tables at c = 16 (quad reduction), 20 and 24 (C_b sums in 8 and 128 parts);
  - the prover with segment lengths 8, 16, 32 and 64 over its generic MSMs."""
import os

import numpy as np
import pytest

from oracle import bn254 as o, layout

import dlog_oracle as dl

pytestmark = pytest.mark.gpu
THREADS = {False: 256, True: 128}       # k_msm_window_bits block size on G1 / G2


def _host(t):
    return t.cpu().numpy().view(np.uint64)


def _check(got, want, what):
    (gp, ginf), (wp, winf) = got, want
    assert ginf == winf and (np.asarray(gp) == wp).all(), "MSM mismatch: %s (got inf=%s, want inf=%s)" % (what, ginf, winf)


class _env:
    """environment variables for the duration of a block (the MSM reads B200ZK_MSM_WINDOW / B200ZK_MSM_SEG on every call)"""

    def __init__(self, **kv):
        self.kv = {k: str(v) for k, v in kv.items() if v is not None}

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        os.environ.update(self.kv)

    def __exit__(self, *exc):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _msm(net, bases, scalars, g2):
    return net.sum_points_dev(net.msm_dev(bases, scalars, g2=g2), 1, g2=g2)


def _generated(net, seed, n, g2, what, c=None, seg=None):
    bases = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
    scalars = net.generate_fr(seed ^ 0x5E6, n)
    with _env(B200ZK_MSM_WINDOW=c, B200ZK_MSM_SEG=seg):
        got = _msm(net, bases, scalars, g2)
    _check(got, dl.expected_msm(seed, _host(scalars), g2), what)


def plan(c, seg=0, fold=False):
    """(nseg, nterms, bsplit) of the thread reduction as msm_plan picks them, or None for the quad reduction"""
    B = 1 << (c - 1)
    WB = 1 if fold else 2 * (-(-128 // c))
    if WB * (B // min(B, 16)) <= 8192:
        return None
    L = 1 << (seg.bit_length() - 1) if seg and seg <= B else min(B, 16)
    nseg = B // L
    bsplit = 1
    while nseg // 2 // bsplit > 2048:
        bsplit *= 2
    return nseg, nseg.bit_length(), bsplit


def test_plan_reaches_every_branch():
    """host only: the cases below take a set without C_b terms, C_b sums in one part and in several parts"""
    plans = [plan(16, s) for s in (1 << 15, 1 << 12, 64, 8)] + [plan(c, fold=True) for c in (20, 24)]
    assert plan(16, 1 << 15) == (1, 1, 1)
    assert any(p[2] == 1 and p[1] > 1 for p in plans) and any(p[2] > 1 for p in plans)
    assert plan(16, fold=True) is None and plan(14, 64) is not None


# ---- 1. segment lengths and empty sums --------------------------------------------------------------------------------
@pytest.mark.parametrize("g2", [False, True], ids=["g1", "g2"])
@pytest.mark.parametrize("seg", [1 << 15, 1 << 12, 64, 8])
def test_segment_lengths_at_c16(net, g2, seg):
    """c = 16 (2 x 8 GLV sets of 2^15 buckets): 1, 8, 512 and 4096 segments per set"""
    p = plan(16, seg)
    assert p is not None and p[0] == (1 << 15) // seg
    _generated(net, 0x5E000000 + seg + g2, 40000, g2, "%s c=16 L=%d plan=%s" % ("G2" if g2 else "G1", seg, p), c=16, seg=seg)


@pytest.mark.parametrize("c", [2, 3, 4, 5])
def test_bucket_set_not_longer_than_segment(net, c):
    """B <= L: every set is one segment (quad reduction), with and without a longer hint"""
    for g2 in (False, True):
        for seg in (None, 64):
            _generated(net, 0x5F000000 + 16 * c + g2, 3001, g2, "%s c=%d seg=%s" % ("G2" if g2 else "G1", c, seg), c=c, seg=seg)


def test_empty_sums(net):
    """scalars below 2^16 at c = 16: the second GLV half is zero and the first has digits in its two lowest windows only,
    so every sum of 14 of the 16 bucket sets is empty and the other two are sparse"""
    import torch
    for g2 in (False, True):
        n, seed = 5000, 0x5A000000 + g2
        bases = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
        rng = np.random.default_rng(seed)
        sc = layout.fr_to_arr([int(v) for v in rng.integers(1, 1 << 16, n)])
        with _env(B200ZK_MSM_WINDOW=16):
            got = _msm(net, bases, torch.from_numpy(sc.view(np.int64)).to(bases.device), g2)
        _check(got, dl.expected_msm(seed, sc, g2), "%s scalars < 2^16 c=16" % ("G2" if g2 else "G1"))


# ---- 2. collisions in the sums -------------------------------------------------------------------------------------------
def window_bits_model(R, A, T, bsplit, log2L, stats):
    """integer model of k_msm_window_bits + k_msm_window_sum for one set of segment pairs (multiples of G): returns S_w;
    `stats` counts the additions whose operands are both non-zero and add to zero ("ident") or are equal ("dbl")"""
    def add(a, b):
        if a and b:
            stats["ident"] += a + b == 0
            stats["dbl"] += a == b
        return a + b

    def block_sum(vals):
        acc = [0] * T
        for k, v in enumerate(vals):
            acc[k % T] = add(acc[k % T], v)
        s = T // 2
        while s:
            for i in range(s):
                acc[i] = add(acc[i], acc[i + s])
            s //= 2
        return acc[0]

    nseg = len(R)
    nbits = nseg.bit_length() - 1
    parts = []
    for b in range(nbits + 1):
        vals = A if b == nbits else [R[s] for s in range(nseg) if s >> b & 1]
        cnt = len(vals) // bsplit
        for h in range(bsplit):
            v = block_sum(vals[h * cnt:(h + 1) * cnt])
            parts.append(v if b == nbits else v << (b + log2L))
    return block_sum(parts)


@pytest.mark.parametrize("g2", [False, True], ids=["g1", "g2"])
def test_window_bits_collisions(net, g2):
    """c = 16, L = 16: the top bucket of segment s holds R_s G (a digit of the lowest window of the first GLV half), so
    A_s = 16 R_s; the model confirms that the sums meet P + (-P) and P + P before the device runs them"""
    import torch
    c, L = 16, 16
    B = 1 << (c - 1)
    nseg, _, bsplit = plan(c, L)
    rng = np.random.default_rng(0xC0111DE + g2)
    R = [int(v) for v in rng.integers(-2, 3, nseg)]
    stats = {"ident": 0, "dbl": 0}
    sw = window_bits_model(R, [L * r for r in R], THREADS[g2], bsplit, 4, stats)
    assert stats["ident"] > 0 and stats["dbl"] > 0, stats
    assert sw == sum((k + 1) * (R[k // L] if k % L == L - 1 else 0) for k in range(B))
    curve, gen = (o.G2, o.G2_GEN) if g2 else (o.G1, o.G1_GEN)
    to_arr = layout.g2_to_arr if g2 else layout.g1_to_arr
    gp, gn = to_arr([gen])[0], to_arr([curve.neg(gen)])[0]
    rows, logs, scal = [], [], []
    for s, r in enumerate(R):
        for _ in range(abs(r)):
            rows.append(gp if r > 0 else gn)
            logs.append(1 if r > 0 else -1)
            scal.append(s * L + L)                              # digit s L + L: bucket s L + L - 1, the segment's top
    sc = layout.fr_to_arr(scal)
    want = dl.expected_from_logs(logs, sc, g2)
    with _env(B200ZK_MSM_WINDOW=c, B200ZK_MSM_SEG=L):
        got = _msm(net, torch.from_numpy(np.stack(rows).view(np.int64)).cuda(), torch.from_numpy(sc.view(np.int64)).cuda(), g2)
    _check(got, want, "%s designed segment sums, %s" % ("G2" if g2 else "G1", stats))


# ---- 3. fixed-base tables -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("g2,c", [(False, 16), (False, 20), (False, 24), (True, 16), (True, 20)])
def test_fold_tables(net, g2, c):
    """one bucket set of 2^(c-1) buckets: c = 16 takes the quad reduction, c = 20 and 24 sum their C_b in 8 and 128 parts"""
    import torch
    p = plan(c, fold=True)
    n, seed = 40000, 0x7B000000 + c + (g2 << 8)
    bases = net.generate_g2(seed, n) if g2 else net.generate_g1(seed, n)
    scalars = net.generate_fr(seed ^ 0x7AB, n)
    table = net.msm_table_build(bases, c, g2=g2)
    got = net.sum_points_dev(net.msm_table_dev(table, scalars, c, g2=g2), 1, g2=g2)
    _check(got, dl.expected_msm(seed, _host(scalars), g2), "table %s c=%d plan=%s" % ("G2" if g2 else "G1", c, p))
    del table
    torch.cuda.empty_cache()


# ---- 4. the prover's generic MSMs at every segment length -------------------------------------------------------------------
@pytest.mark.parametrize("seg", [8, 16, 32, 64])
def test_prover_segment_lengths(net, cref, seg):
    """a 2^18-constraint proof over the generic MSMs (no tables): its MSMs run at c = 14 (2 x 10 sets of 8192 buckets)
    through the thread reduction, with the prover's 32-bucket hint overridden"""
    import torch
    import prove_dlog_oracle as po
    from distributed_groth16_b200.groth16 import ProvingKey, prove
    m = 1 << 18
    assert plan(14, seg) is not None
    a, b, c = (net.generate_fr(0x6C000000 + 8 * m + k, m) for k in range(3))
    h = po.expected_h(cref, _host(a), _host(b), _host(c))
    z = net.generate_fr(0x6D000000 + seg, m)
    z[0] = torch.from_numpy(po.ONE.view(np.int64)).to(z.device)
    spec = po.KeySpec(m, m, 2, 0x6E000000 + seg)
    e = po.exponents(spec, _host(z), h)
    pts = spec.device_points(net)
    with _env(B200ZK_PK_TABLES=0):
        pk = ProvingKey.from_device(net, pts["a"], pts["b1"], pts["b2"], pts["l"], pts["h"], spec.n_inputs, po.vk_array(pts))
    del pts
    assert pk.table_bytes == 0
    rs = (0x2F1E3D4C5B6A79881726354453627180 % o.R, 0x0A1B2C3D4E5F60718293A4B5C6D7E8F9 * 7 % o.R)
    with _env(B200ZK_MSM_SEG=seg):
        got = prove.create_proof_dev(pk, z, a, b, c, layout.fr_to_arr([rs[0]])[0], layout.fr_to_arr([rs[1]])[0])
    pk.free()
    torch.cuda.empty_cache()
    assert got == po.proof_bytes(e, *rs), "proof mismatch at m=2^18 with B200ZK_MSM_SEG=%d" % seg
