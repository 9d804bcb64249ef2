"""The two-level NTT twiddle tables, the path transforms above 2^24 and a device without room for the single-level table
fall back to, reached below 2^25 with B200ZK_NTT_BIGTAB=0 (read once per process) and checked against the oracle in a fresh
process."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import sys
sys.path.insert(0, %r)
import numpy as np
from oracle import cref
from distributed_groth16_b200 import Net
from distributed_groth16_b200.dist_primitives import d_msm
cref.build()
net = Net(0)
for log_n in (9, 12, 17):
    x = cref.fr_generate(40 + log_n, 1 << log_n)
    for inv in (False, True):
        for coset in (False, True):
            assert (net.ntt(x, inverse=inv, coset=coset) == cref.ntt(x, inverse=inv, coset=coset)).all(), (log_n, inv, coset)
a = cref.fr_generate(7, 1 << 10)
assert (net.h_circom(a, a[::-1].copy(), a) == cref.h_circom(a, a[::-1].copy(), a, 1)).all()
for g2 in (False, True):
    for n in (300, 5000):
        bases = (cref.g2_generate if g2 else cref.g1_generate)(50 + n, n)
        scalars = cref.fr_generate(60 + n, n)
        scalars[0] = 0
        scalars[1] = np.array([1, 0, 0, 0], dtype=np.uint64)        # not a Montgomery one: just another scalar
        got = d_msm(bases, scalars, None, net, g2=g2)
        exp, inf = (cref.msm_g2 if g2 else cref.msm_g1)(bases, scalars)
        assert (np.asarray(got.limbs) == exp).all() and bool(got.infinity) == bool(inf), (g2, n)
print("fallback paths ok")
"""


@pytest.mark.parametrize("env", [{"B200ZK_NTT_BIGTAB": "0"}], ids=["two-level-twiddles"])
def test_switchable_paths_match_the_oracle(env):
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, "-c", SCRIPT % ROOT], env=e, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "fallback paths ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
