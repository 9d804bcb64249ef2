"""NTTs at 2^23..2^26 bit for bit against the CPU twin, and a closed form at 2^26 that pins the root of unity without it.

Up to 2^24 the first pass boundary and the coset tables are single-level; above 2^24 they are two-level by default
(B200ZK_NTT_BIGTAB, csrc/ntt.cu).  Elsewhere the suite checks 2^24 and 2^26 only by iNTT(NTT(x)) == x, which a transform
with a consistently wrong root passes.  Forward, inverse and coset transforms are compared with `cref.ntt`; the impulse
e_k transforms to NTT(e_k)[j] = w^{jk} (coset: g^k w^{jk}; inverse: w^{-jk} / n, coset inverse also times g^{-j}), checked
at 4096 indices j with exponents jk spread over the whole range, the high table half included.

Measured on one H100 80GB HBM3 at a 700 W power limit: 155 s for the file, most of it the CPU twin at 2^25 and 2^26."""
import numpy as np
import pytest

from oracle import bn254 as o, layout

pytestmark = pytest.mark.gpu


def _ntt_dev(net, x, inverse=False, coset=False):
    import torch
    y = net.ntt_dev(x, inverse=inverse, coset=coset)
    torch.cuda.synchronize()
    return y.cpu().numpy().view(np.uint64)


@pytest.mark.parametrize("log_n", [23, 24, 25, 26])
def test_large_ntt_matches_cref(net, cref, log_n):
    import torch
    n = 1 << log_n
    x = net.generate_fr(0xE4AC7000 + log_n, n)
    xh = x.cpu().numpy().view(np.uint64)
    for inverse, coset in ((False, False), (True, False), (False, True)):
        got = _ntt_dev(net, x, inverse, coset)
        want = cref.ntt(xh, inverse=inverse, coset=coset)
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert bad.size == 0, (log_n, inverse, coset, bad.size, bad[:8])
        del got, want
    del x, xh
    torch.cuda.empty_cache()


def test_impulse_closed_form_2_26(net):
    import torch
    log_n = 26
    n = 1 << log_n
    w = o.fr_root_of_unity(n)
    g = o.FR_GENERATOR
    rng = np.random.default_rng(26)
    js = np.unique(np.concatenate([rng.integers(0, n, 4090), [0, 1, 2, n // 2, n - 2, n - 1]]))
    for k in (1, (1 << 24) + 3, n - 1, int(rng.integers(1 << 25, n)) | 1):
        x = torch.zeros((n, 4), dtype=torch.int64, device="cuda")
        x[k] = torch.from_numpy(layout.fr_to_arr([1]).view(np.int64)[0]).cuda()
        for inverse, coset in ((False, False), (False, True), (True, False), (True, True)):
            y = net.ntt_dev(x, inverse=inverse, coset=coset)
            torch.cuda.synchronize()
            got = layout.arr_to_fr(y[torch.from_numpy(js).cuda()].cpu().numpy().view(np.uint64))
            if not inverse:
                scale = pow(g, k, o.R) if coset else 1
                want = [scale * pow(w, int(j) * k % n, o.R) % o.R for j in js]
            else:
                ninv = pow(n, -1, o.R)
                want = [ninv * pow(w, (n - int(j) * k % n) % n, o.R) % o.R for j in js]
                if coset:
                    want = [v * pow(g, -int(j), o.R) % o.R for v, j in zip(want, js)]
            bad = [int(j) for j, a, b in zip(js, got, want) if a != b]
            assert not bad, (k, inverse, coset, len(bad), bad[:8])
            del y
        del x
        torch.cuda.empty_cache()
