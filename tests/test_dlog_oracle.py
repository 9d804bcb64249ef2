"""tests/dlog_oracle.py against the CPU twin: the splitmix mirror reproduces the generated bases (last index included,
and across the 2^64 wrap of seed + i), and the exact dot product gives the same point as cref's MSM."""
import numpy as np
import pytest

from oracle import bn254 as o, layout

import dlog_oracle as dl


def _gen_arr(g2):
    return (layout.g2_to_arr if g2 else layout.g1_to_arr)([o.G2_GEN if g2 else o.G1_GEN])[0]


@pytest.mark.parametrize("g2", [False, True])
@pytest.mark.parametrize("seed,n", [(0xB2000001, 3000), (0, 2), ((1 << 64) - 5, 17)])
def test_mirror_reproduces_the_generated_bases(cref, g2, seed, n):
    pts = (cref.g2_generate if g2 else cref.g1_generate)(seed, n)
    idx = sorted(set(list(range(min(n, 64))) + list(range(max(0, n - 64), n))))
    logs = dl.base_logs(seed, n)[idx]
    assert (logs & np.uint64(1)).all()
    want = cref.fixed_base_mul(_gen_arr(g2), layout.fr_to_arr([int(k) for k in logs]), g2=g2)
    assert (pts[idx] == want).all()
    m = min(n, 8)
    assert (dl.base_logs(seed, m, start=n - m) == dl.base_logs(seed, n)[n - m:]).all()


def test_splitmix_known_values():
    """splitmix64's first outputs from state 0 (published test vector of the generator)."""
    x = np.array([0, 0x9E3779B97F4A7C15], dtype=np.uint64)
    assert [int(v) for v in dl.splitmix64(x)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4]


@pytest.mark.parametrize("g2", [False, True])
@pytest.mark.parametrize("n", [1, 5, 300, 4096])
def test_exact_dot_matches_cref_msm(cref, g2, n):
    seed = 0xD106 + n
    bases = (cref.g2_generate if g2 else cref.g1_generate)(seed, n)
    scalars = cref.fr_generate(seed, n)
    if n >= 5:
        scalars[:5] = layout.fr_to_arr([0, 1, o.R - 1, 1 << 253, 7])
    got, inf = dl.expected_msm(seed, scalars, g2)
    want, winf = (cref.msm_g2 if g2 else cref.msm_g1)(bases, scalars)
    assert inf == winf and (got == want).all()


def test_exact_dot_edges(cref):
    """A zero sum gives infinity; limbs at their maximum do not overflow the 16-bit split."""
    n = 4
    logs = np.full(n, (1 << 64) - 1, dtype=np.uint64)
    v = np.full((n, 4), (1 << 64) - 1, dtype=np.uint64)
    assert dl.exact_dot(logs, v) == n * ((1 << 64) - 1) * ((1 << 256) - 1)
    scalars = layout.fr_to_arr([5, o.R - 5])
    _, inf = dl.expected_from_logs([3, 3], scalars)
    assert inf
    pt, inf = dl.expected_from_logs([1, -1, 2], layout.fr_to_arr([4, 1, 1]))
    assert not inf and (pt == layout.g1_to_arr([o.G1.mul(o.G1_GEN, 5)])[0]).all()


def test_glv_mirror_constants_and_families():
    """The split constants describe the lattice {(a, b): a + b lambda = 0 mod r}, and every designed scalar family splits
    back into the halves it was built from."""
    g, lam = dl.GLV, dl.LAMBDA
    assert (lam * lam + lam + 1) % o.R == 0
    assert (g["a1"] - g["nb1"] * lam) % o.R == 0 and (g["a2"] + g["b2"] * lam) % o.R == 0
    assert g["g1"] == (g["b2"] << 256) // o.R and g["g2"] == (g["nb1"] << 256) // o.R
    for h1, h2 in dl.glv_designed_halves():
        assert dl.glv_decompose(dl.glv_compose(h1, h2)) == (h1, h2)
    for c in range(2, 25):
        h = [dl.repeat_digit(d, c, dl.GLV_HALF_BITS) for d in ((1 << (c - 1)), (1 << (c - 1)) + 1, (1 << c) - 1)]
        for v in h:
            for s1 in (1, -1, 0):
                for s2 in (1, -1, 0):
                    assert dl.glv_decompose(dl.glv_compose(s1 * v, s2 * v)) == (s1 * v, s2 * v), (c, v, s1, s2)
