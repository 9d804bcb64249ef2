"""ctypes binding of oracle/liboracle.so (TEST INFRASTRUCTURE ONLY -- see bn254_ref.cpp).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  Arrays are numpy uint64 in the b200zk.h layout (Montgomery limbs)."""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")
_lib = None

_u64p = ctypes.POINTER(ctypes.c_uint64)


def build(force: bool = False) -> str:
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(
            os.path.join(_HERE, "bn254_ref.cpp")):
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = ctypes.CDLL(_LIB_PATH)
        _lib.orc_num_threads.restype = ctypes.c_int
    return _lib


def _p(a: np.ndarray):
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(_u64p)


def num_threads() -> int:
    return lib().orc_num_threads()


def constants() -> dict:
    out = np.zeros(26, dtype=np.uint64)
    lib().orc_constants(_p(out))
    f = lambda s: int.from_bytes(out[s].tobytes(), "little")
    return dict(q=f(slice(0, 4)), r=f(slice(4, 8)), inv_q=int(out[8]), inv_r=int(out[9]),
                r1_q=f(slice(10, 14)), r1_r=f(slice(14, 18)), r2_q=f(slice(18, 22)), r2_r=f(slice(22, 26)))


def field_op(field: int, op: int, a: np.ndarray, b: np.ndarray | None = None) -> np.ndarray:
    out = np.zeros(4, dtype=np.uint64)
    lib().orc_field_op(field, op, _p(a), _p(b) if b is not None else None, _p(out))
    return out


def g1_generate(seed: int, n: int, nthreads: int = 0) -> np.ndarray:
    out = np.zeros((n, 8), dtype=np.uint64)
    lib().orc_g1_generate(ctypes.c_uint64(seed), ctypes.c_size_t(n), _p(out), nthreads)
    return out


def g2_generate(seed: int, n: int, nthreads: int = 0) -> np.ndarray:
    out = np.zeros((n, 16), dtype=np.uint64)
    lib().orc_g2_generate(ctypes.c_uint64(seed), ctypes.c_size_t(n), _p(out), nthreads)
    return out


def fixed_base_mul(base, scalars, g2: bool = False, nthreads: int = 0) -> np.ndarray:
    """scalars[i] * base for one affine base point (Montgomery limbs) and (n, 4) Montgomery scalars."""
    w = 16 if g2 else 8
    b = np.ascontiguousarray(base, dtype=np.uint64).reshape(w)
    s = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, 4)
    out = np.zeros((s.shape[0], w), dtype=np.uint64)
    fn = lib().orc_g2_fixed_base_mul if g2 else lib().orc_g1_fixed_base_mul
    fn(_p(b), _p(s), ctypes.c_size_t(s.shape[0]), _p(out), int(nthreads))
    return out


def fr_generate(seed: int, n: int) -> np.ndarray:
    out = np.zeros((n, 4), dtype=np.uint64)
    lib().orc_fr_generate(ctypes.c_uint64(seed), ctypes.c_size_t(n), _p(out))
    return out


def _msm(fn, bases, scalars, width, nthreads=None):
    bases = np.ascontiguousarray(bases, dtype=np.uint64)
    scalars = np.ascontiguousarray(scalars, dtype=np.uint64)
    n = min(bases.shape[0], scalars.shape[0])
    out = np.zeros(width, dtype=np.uint64)
    inf = ctypes.c_int(0)
    if nthreads is None:
        fn(_p(bases), _p(scalars), ctypes.c_size_t(n), _p(out), ctypes.byref(inf))
    else:
        fn(_p(bases), _p(scalars), ctypes.c_size_t(n), _p(out), ctypes.byref(inf), nthreads)
    return out, bool(inf.value)


def msm_g1(bases, scalars, nthreads: int = 0):
    return _msm(lib().orc_msm_g1, bases, scalars, 8, nthreads)


def msm_g2(bases, scalars, nthreads: int = 0):
    return _msm(lib().orc_msm_g2, bases, scalars, 16, nthreads)


def msm_g1_naive(bases, scalars):
    return _msm(lib().orc_msm_g1_naive, bases, scalars, 8)


def msm_g2_naive(bases, scalars):
    return _msm(lib().orc_msm_g2_naive, bases, scalars, 16)


def g1_on_curve(pts) -> bool:
    pts = np.ascontiguousarray(pts, dtype=np.uint64)
    return bool(lib().orc_g1_on_curve(_p(pts), ctypes.c_size_t(pts.shape[0])))


def g2_on_curve(pts) -> bool:
    pts = np.ascontiguousarray(pts, dtype=np.uint64)
    return bool(lib().orc_g2_on_curve(_p(pts), ctypes.c_size_t(pts.shape[0])))


def ntt(data, inverse: bool = False, coset: bool = False, nthreads: int = 0) -> np.ndarray:
    out = np.array(data, dtype=np.uint64, copy=True, order="C")
    n = out.shape[0]
    log_n = n.bit_length() - 1
    assert 1 << log_n == n
    rc = lib().orc_ntt(_p(out), log_n, int(inverse), int(coset), nthreads)
    assert rc == 0
    return out


def ntt_batched_post(data, log_t: int, batch: int, inverse: bool, log_base: int, shift: bool = False, b0: int = 0, alpha: int = 0,
                     beta: int = 0, gamma: int = 0, nthreads: int = 0) -> np.ndarray:
    """b200zk_ntt_fr_batched_post_dev: `batch` contiguous NTTs of 2^log_t elements, output k of transform b times
    base^((b + b0)(alpha k + beta) + gamma k), base = w_{2^log_base} (inverted for an inverse transform unless `shift`).
    data: (batch * 2^log_t, 4) Montgomery limbs; the same as tests/mgpu_common.OracleBackend.batched_ntt_post."""
    out = np.array(data, dtype=np.uint64, copy=True, order="C").reshape(-1, 4)
    assert out.shape[0] == batch << log_t
    rc = lib().orc_ntt_batched_post(_p(out), log_t, ctypes.c_size_t(batch), int(inverse), log_base, int(shift), ctypes.c_uint64(b0),
                                    ctypes.c_uint64(alpha), ctypes.c_uint64(beta), ctypes.c_uint64(gamma), nthreads)
    assert rc == 0
    return out


def bitrev(data) -> np.ndarray:
    out = np.array(data, dtype=np.uint64, copy=True, order="C")
    n = out.shape[0]
    lib().orc_bitrev(_p(out), n.bit_length() - 1)
    return out


def fr_spmv(ptr, idx, val, x, nthreads: int = 0) -> np.ndarray:
    """CSR mat-vec over Fr: out[r] = sum_k val[k] x[idx[k]], k in [ptr[r], ptr[r+1]).  ptr (n_rows + 1,) and idx (nnz,)
    u32, val (nnz, 4) and x (n, 4) Montgomery limbs; -> (n_rows, 4)."""
    ptr = np.ascontiguousarray(ptr, dtype=np.uint32).reshape(-1)
    idx = np.ascontiguousarray(idx, dtype=np.uint32).reshape(-1)
    val = np.ascontiguousarray(val, dtype=np.uint64).reshape(-1, 4)
    x = np.ascontiguousarray(x, dtype=np.uint64).reshape(-1, 4)
    n_rows = ptr.shape[0] - 1
    nnz = int(ptr[-1])
    assert n_rows >= 0 and (np.diff(ptr.astype(np.int64)) >= 0).all() and idx.shape[0] >= nnz and val.shape[0] >= nnz
    assert nnz == 0 or int(idx[:nnz].max()) < x.shape[0]
    out = np.zeros((n_rows, 4), dtype=np.uint64)
    u32p = ctypes.POINTER(ctypes.c_uint32)
    lib().orc_fr_spmv(ptr.ctypes.data_as(u32p), idx.ctypes.data_as(u32p), _p(val), _p(x), ctypes.c_size_t(n_rows), _p(out),
                      int(nthreads))
    return out


def qap(a_csr, b_csr, z, nc: int, n_inputs: int, m: int, nthreads: int = 0):
    """qap::qap (groth16/src/qap.rs:44-91) on CSR matrices: a_i = <A_i, z>, b_i = <B_i, z> for i < nc, a[nc + j] = z[j] for
    j < n_inputs, c = a * b, zero up to m.  a_csr / b_csr: (ptr, idx, val) as fr_spmv takes them, nc + 1 row pointers each;
    z: (n_vars, 4) Montgomery limbs.  -> a, b, c as (m, 4) Montgomery limbs."""
    assert nc + n_inputs <= m
    z = np.ascontiguousarray(z, dtype=np.uint64).reshape(-1, 4)
    a, b, c = (np.zeros((m, 4), dtype=np.uint64) for _ in range(3))
    a[:nc] = fr_spmv(*a_csr, z, nthreads=nthreads)
    b[:nc] = fr_spmv(*b_csr, z, nthreads=nthreads)
    a[nc:nc + n_inputs] = z[:n_inputs]
    diag = np.arange(nc + 1, dtype=np.uint32)                # c_i = a_i b_i: the diagonal matrix of a times b
    c[:nc] = fr_spmv(diag, diag[:nc], a[:nc], b, nthreads=nthreads)
    return a, b, c


def h_circom(a, b, c, nthreads: int = 0) -> np.ndarray:
    a, b, c = (np.ascontiguousarray(x, dtype=np.uint64) for x in (a, b, c))
    m = a.shape[0]
    out = np.zeros((m, 4), dtype=np.uint64)
    lib().orc_h_circom(_p(a), _p(b), _p(c), m.bit_length() - 1, _p(out), nthreads)
    return out


def groth16_prove(a_query, b_g1_query, b_g2_query, l_query, h_query, vk_pts, n_inputs, z, h, r, s,
                  mirror_bg1: bool = False, nthreads: int = 0) -> bytes:
    arrs = [np.ascontiguousarray(x, dtype=np.uint64) for x in
            (a_query, b_g1_query, b_g2_query, l_query, h_query, vk_pts, z, h, r, s)]
    aq, b1, b2, lq, hq, vk, zz, hh, rr, ss = arrs
    n_vars = aq.shape[0]
    m = hq.shape[0]
    assert hh.shape[0] == m and zz.shape[0] == n_vars and lq.shape[0] == n_vars - n_inputs
    out = (ctypes.c_uint8 * 128)()
    rc = lib().orc_groth16_prove(_p(aq), _p(b1), _p(b2), _p(lq), _p(hq), ctypes.c_size_t(n_vars),
                                 ctypes.c_size_t(n_inputs), ctypes.c_size_t(m), _p(vk), _p(zz), _p(hh),
                                 _p(rr), _p(ss), int(mirror_bg1), out, nthreads)
    assert rc == 0
    return bytes(out)
