"""The CPU twin's batched NTT with post factors (cref.ntt_batched_post) against the Python restatement the gloo test drives
parallel.py with (mgpu_common.OracleBackend.batched_ntt_post).  tests/test_gpu_sharded_exact.py compares the device kernel
with the twin at sizes the Python backend is too slow for, so this pin closes the chain parallel.py -> OracleBackend ->
twin -> kernel."""
import numpy as np
import pytest
import torch

from mgpu_common import OracleBackend

# (log_t, batch, inverse, log_base, shift, b0, alpha, beta, gamma): every tuple shape parallel.sharded_ntt passes (column
# step of rank g: b0 = g cg, alpha = 1; shifted row step: b0 = g rl, beta = 1, gamma = rows), the single-GPU plain post
# (0, 0, 1), and exponents past the order of the base (the twin reduces them; the device refuses them)
CASES = [
    (3, 4, False, 5, False, 0, 1, 0, 0),
    (3, 2, False, 5, False, 2, 1, 0, 0),
    (3, 2, True, 5, False, 6, 1, 0, 0),
    (2, 2, True, 5, True, 4, 0, 1, 8),
    (2, 1, True, 5, True, 7, 0, 1, 8),
    (4, 3, False, 4, False, 0, 0, 0, 1),
    (4, 3, True, 6, False, 5, 3, 7, 11),
    (1, 2, False, 2, False, 9, 5, 1, 3),
    (2, 3, True, 3, True, (1 << 64) - 2, 1 << 40, 5, (1 << 63) + 1),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "t%d_b%d_inv%d_base%d_shift%d_b0=%d" % c[:6])
def test_twin_batched_post_equals_oracle_backend(cref, case):
    log_t, batch, inverse, log_base, shift, b0, alpha, beta, gamma = case
    x = cref.fr_generate(0xBA7C + log_t + 7 * batch, batch << log_t)
    want = OracleBackend().batched_ntt_post(torch.from_numpy(x.view(np.int64)), log_t, batch, inverse, log_base=log_base, shift=shift,
                                            b0=b0, alpha=alpha, beta=beta, gamma=gamma).numpy().view(np.uint64)
    got = cref.ntt_batched_post(x, log_t, batch, inverse, log_base, shift, b0, alpha, beta, gamma)
    assert (got == want).all()


def test_twin_batched_post_without_post_factor_is_the_batched_ntt(cref):
    x = cref.fr_generate(0xBA7D, 4 << 5)
    for inverse in (False, True):
        got = cref.ntt_batched_post(x, 5, 4, inverse, 0)
        want = np.concatenate([cref.ntt(x[b << 5:(b + 1) << 5], inverse=inverse) for b in range(4)])
        assert (got == want).all(), inverse
