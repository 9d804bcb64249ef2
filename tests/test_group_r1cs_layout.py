"""The host-side reorder behind GroupConstraintMatrices (b200zk_group_r1cs_local_row_ptr): GPU g of P keeps, at local slot
c rows + r, the CSR row of global constraint r cols + g cols / P + c, the column layout the sharded h pipeline reads
(csrc/group.cu).  Checked against a NumPy restatement of that layout, without a device."""
import numpy as np
import pytest

from distributed_groth16_b200._native import ERR_ARG, ERR_DOMAIN, B200zkError
from distributed_groth16_b200.group import local_row_ptr


def column_layout(log_m, P):
    """global row index held by every local slot, per GPU: the row-major rows x cols matrix of 0..m-1, GPU g's column slab
    stored column after column"""
    rows, cols = 1 << ((log_m + 1) // 2), 1 << (log_m // 2)
    x = np.arange(1 << log_m).reshape(rows, cols)
    cg = cols // P
    return [x[:, g * cg:(g + 1) * cg].T.reshape(-1) for g in range(P)]


def row_ptr_with_lengths(lengths):
    ptr = np.zeros(len(lengths) + 1, dtype=np.uint32)
    ptr[1:] = np.cumsum(lengths)
    return ptr


@pytest.mark.parametrize("P", [1, 2, 4, 8])
@pytest.mark.parametrize("log_m", [6, 7, 8, 9])
@pytest.mark.parametrize("fill", ["full", "minus3", "five"])
def test_every_constraint_lands_in_one_slot_of_the_column_layout(log_m, P, fill):
    m = 1 << log_m
    nc = {"full": m, "minus3": m - 3, "five": 5}[fill]
    ptr = row_ptr_with_lengths(np.arange(1, nc + 1))          # row i has i + 1 terms: a slot's length names its row
    layout = column_layout(log_m, P)
    seen = []
    for g in range(P):
        lptr = local_row_ptr(ptr, nc, log_m, P, g)
        assert lptr.shape == (m // P + 1,) and lptr[0] == 0
        lengths = np.diff(lptr.astype(np.int64))
        want = np.where(layout[g] < nc, layout[g] + 1, 0)     # rows >= nc (padding and instance rows) have no terms
        assert (lengths == want).all(), g
        seen.append(lengths[lengths > 0] - 1)
    seen = np.sort(np.concatenate(seen))
    assert (seen == np.arange(nc)).all()                      # every constraint exactly once over the GPUs


def test_empty_rows_stay_empty():
    log_m, P, nc = 8, 4, 200
    lengths = np.zeros(nc, dtype=np.int64)
    lengths[::7] = 3
    ptr = row_ptr_with_lengths(lengths)
    layout = column_layout(log_m, P)
    for g in range(P):
        got = np.diff(local_row_ptr(ptr, nc, log_m, P, g).astype(np.int64))
        want = np.where(layout[g] < nc, lengths[np.minimum(layout[g], nc - 1)], 0)
        assert (got == want).all(), g


@pytest.mark.parametrize("case,code", [((4, 8, 0), ERR_ARG),           # cols = 4 < 8 GPUs
                                       ((28, 1, 0), ERR_DOMAIN),       # log_m > 27
                                       ((6, 3, 0), ERR_ARG),           # not a power of two
                                       ((6, 2, 2), ERR_ARG)])          # rank out of range
def test_refusals(case, code):
    log_m, P, rank = case
    with pytest.raises(B200zkError) as e:
        local_row_ptr(np.zeros(1, dtype=np.uint32), 0, log_m, P, rank)
    assert e.value.code == code


def test_more_constraints_than_the_domain_is_a_domain_error():
    with pytest.raises(B200zkError) as e:
        local_row_ptr(np.zeros(66, dtype=np.uint32), 65, 6, 1, 0)
    assert e.value.code == ERR_DOMAIN
