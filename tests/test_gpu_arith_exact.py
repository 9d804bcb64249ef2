"""Every device primitive of fp.cuh, codec.cuh, pairing.cuh, glv.cuh and ec.cuh on the H100, element by element through
b200zk_test_arith (csrc/selftest.cu), against the big-integer answers of tests/arith_oracle.py, record for record.

The operands reach each reduction branch on purpose (final subtractions, both redc<2> subtractions of Fq2::mul's c0, every
iteration count of Fp::inv, the c1 = 0 square roots, ...): on sm_90a the carry chains are separate PTX statements sharing the
carry flag, which the host run of the same bodies (tests/test_host_arith.py) cannot show.  The quad-cooperative group law
runs with the eight quads of a warp on eight different relations (P + P, P - P, O, ...), i.e. different early returns and
__syncwarp masks in one launch."""
import ctypes

import numpy as np
import pytest

import arith_oracle as A

pytestmark = pytest.mark.gpu


def _run(net, name):
    op = A.OPS[name]
    recs = A.corpus()[name]
    inp = np.ascontiguousarray(np.array([r for _, r in recs], dtype=np.uint64))
    out = np.zeros((len(recs), op.n_out), dtype=np.uint64)
    net.check(net._lib.b200zk_test_arith(net._h, op.code, ctypes.c_void_p(inp.ctypes.data), len(recs),
                                         ctypes.c_void_p(out.ctypes.data)))
    return out


@pytest.mark.parametrize("name", list(A.OPS))
def test_device_arith_exact(net, name):
    got = _run(net, name)
    bad = A.mismatches(name, got)
    assert not bad, "%d of %d records wrong, first:\n%s" % (len(bad), len(got), "\n".join(bad[:3]))


def test_unknown_op_is_refused(net):
    from distributed_groth16_b200 import B200zkError
    one = np.zeros(64, dtype=np.uint64)
    with pytest.raises(B200zkError):
        net.check(net._lib.b200zk_test_arith(net._h, 63, ctypes.c_void_p(one.ctypes.data), 1, ctypes.c_void_p(one.ctypes.data)))
