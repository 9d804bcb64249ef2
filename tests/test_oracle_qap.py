"""The CPU twin's CSR mat-vec and QAP (oracle/bn254_ref.cpp orc_fr_spmv, oracle/cref.py fr_spmv / qap) against Python ints
and oracle/bn254.py's qap: the expected values of the device's R1CS -> QAP tests (tests/test_gpu_qap_setup_exact.py)."""
import numpy as np

from oracle import bn254 as o, layout as L

R = o.R


def _rand_ints(rng, n):
    return [int.from_bytes(rng.bytes(32), "little") % R for _ in range(n)]


def _matrix(rng, n_rows, n_vars, lengths):
    """rows as [(coeff, wire)] lists: coefficients 0, 1, r - 1 and full width; wires 0 and n_vars - 1 appear, and row 2
    holds one (row, col) pair twice"""
    specials = [0, 1, R - 1]
    rows = []
    for i in range(n_rows):
        k = lengths[i % len(lengths)]
        cols = [int(c) for c in rng.integers(0, n_vars, k)]
        vals = [specials[j % 3] if (i + j) % 4 == 0 else v for j, v in enumerate(_rand_ints(rng, k))]
        rows.append(list(zip(vals, cols)))
    rows[0] = [(_rand_ints(rng, 1)[0], 0), (R - 1, n_vars - 1)]
    rows[2] = [(_rand_ints(rng, 1)[0], 7 % n_vars), (_rand_ints(rng, 1)[0], 7 % n_vars)]
    return rows


def _csr(rows):
    ptr = np.zeros(len(rows) + 1, dtype=np.uint32)
    ptr[1:] = np.cumsum([len(r) for r in rows])
    idx = np.array([w for r in rows for _, w in r], dtype=np.uint32)
    val = L.fr_to_arr([c for r in rows for c, _ in r])
    return ptr, idx, val


def test_fr_spmv_against_python_int_dot_products(cref):
    rng = np.random.default_rng(11)
    n_vars = 300
    lengths = [0, 1, 2, 31, 32, 33, 64, 65, 3, 0]
    rows = _matrix(rng, 200, n_vars, lengths)
    rows[5] = [(v, int(c)) for v, c in zip(_rand_ints(rng, 5000), rng.integers(0, n_vars, 5000))]     # one long row
    z = _rand_ints(rng, n_vars)
    z[0] = 1
    got = L.arr_to_fr(cref.fr_spmv(*_csr(rows), L.fr_to_arr(z), nthreads=4))
    want = [sum(c * z[w] for c, w in r) % R for r in rows]
    assert got == want
    assert want[9] == 0 and rows[9] == [] and len(rows[2]) == 2 and rows[2][0][1] == rows[2][1][1]
    # no rows, and rows without terms
    assert cref.fr_spmv(np.zeros(1, dtype=np.uint32), np.zeros(0, dtype=np.uint32), np.zeros((0, 4), dtype=np.uint64),
                        L.fr_to_arr(z)).shape == (0, 4)
    empty = cref.fr_spmv(np.zeros(9, dtype=np.uint32), np.zeros(0, dtype=np.uint32), np.zeros((0, 4), dtype=np.uint64),
                         L.fr_to_arr(z))
    assert empty.shape == (8, 4) and not empty.any()


def test_qap_against_the_python_oracle(cref):
    rng = np.random.default_rng(12)
    for nc, n_inputs, n_vars, wit in ((0, 1, 1, "random"), (1, 1, 2, "random"), (31, 1, 40, "random"), (14, 17, 60, "0/1"),
                                      (45, 2, 90, "random"), (61, 3, 64, "0/1")):
        a_rows = _matrix(rng, nc, n_vars, [0, 1, 2, 33, 65, 4]) if nc > 2 else [[(5, 0)]] * nc
        b_rows = _matrix(rng, nc, n_vars, [1, 0, 32, 2, 64]) if nc > 2 else [[]] * nc
        if nc > 7:
            b_rows[7] = []                                           # B's row empty while A's is not
            assert a_rows[7]
        z = _rand_ints(rng, n_vars) if wit == "random" else [int(v) for v in rng.integers(0, 2, n_vars)]
        z[0] = 1
        m = o.next_pow2(nc + n_inputs)
        want = o.qap(a_rows, b_rows, n_inputs, nc, z)
        got = cref.qap(_csr(a_rows), _csr(b_rows), L.fr_to_arr(z), nc, n_inputs, m, nthreads=3)
        assert all(g.shape == (m, 4) for g in got)
        assert [L.arr_to_fr(g) for g in got] == list(want), (nc, n_inputs)
