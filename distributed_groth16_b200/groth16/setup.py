"""Circuit-specific Groth16 setup on the GPU (SURVEY 8f3).

What the reference's drivers obtain from `Groth16::<Bn254, CircomReduction>::circuit_specific_setup(circuit, rng)`
(/root/reference/groth16/examples/sha256.rs:133-137, mpc-api/src/main.rs:148-152): a proving key whose h-query
follows `CircomReduction::h_query_scalars` (ark-circom/src/circom/qap.rs:94-110) so that it pairs with the odd-coset h of
`ext_wit::h`.  The toxic waste (tau, alpha, beta, gamma, delta) is supplied by the caller as canonical integers -- this is a
development / benchmarking setup (known trapdoor), exactly like the reference's fixed-seed one.

Every field / group operation runs on the device: QAP evaluations at tau = Lagrange coefficients (an iNTT of the powers
of tau) times the transposed constraint matrices (CSR mat-vec), query scalars by a fused linear combination, query points
by fixed-base multiplication of the generators.  The host only reorders index arrays and builds small scalar vectors."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from .._native import c_vp
from ..formats import FR_MODULUS
from .proving_key import ProvingKey
from .qap import ConstraintMatrices

R = FR_MODULUS
_MONT = 1 << 256


def _mont_limbs(v: int) -> np.ndarray:
    """canonical int -> Montgomery limbs.  Integer arithmetic on the handful of setup constants only."""
    x = (v % R) * _MONT % R
    return np.array([(x >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)], dtype=np.uint64)


@dataclass
class VerifyingKey:
    alpha_g1: np.ndarray
    beta_g2: np.ndarray
    gamma_g2: np.ndarray
    delta_g2: np.ndarray
    gamma_abc_g1: np.ndarray      # (n_inputs, 8)


def _fixed_base(net, scalars, g2=False):
    import torch
    n = int(scalars.shape[0])
    out = torch.empty((n, 16 if g2 else 8), dtype=torch.int64, device=scalars.device)
    net.check(net._lib.b200zk_fixed_base_mul_dev(net._h, int(g2), c_vp(scalars.data_ptr()), n, c_vp(out.data_ptr())))
    return out


def _fixed_base_custom(net, base, scalars, g2=False):
    """scalars[i] * base for an arbitrary base point (the reference draws its generators at random, ark-groth16's
    `generate_random_parameters_with_reduction`): `b200zk_points_matmul_dev` with a one-point chunk, i.e. one thread per
    scalar, in slabs of 4096 rows (its limit).  One-off setup work."""
    import torch
    n, w = int(scalars.shape[0]), 16 if g2 else 8
    out = torch.empty((n, w), dtype=torch.int64, device=scalars.device)
    pt = net.to_device(np.ascontiguousarray(base, dtype=np.uint64).reshape(1, w))
    scalars = scalars.contiguous()
    for lo in range(0, n, 4096):
        rows = min(4096, n - lo)
        net.check(net._lib.b200zk_points_matmul_dev(net._h, 0, int(g2), c_vp(pt.data_ptr()), 1, 1,
                                                    c_vp(scalars[lo:lo + rows].data_ptr()), rows,
                                                    c_vp(out[lo:lo + rows].data_ptr())))
    net.sync(0)
    return out


def _powers(net, base: int, scale: int, n: int):
    import torch
    out = torch.empty((n, 4), dtype=torch.int64, device=torch.device("cuda", net.device))
    b, s = _mont_limbs(base), _mont_limbs(scale)
    net.check(net._lib.b200zk_fr_powers_dev(net._h, c_vp(b.ctypes.data), c_vp(s.ctypes.data), n, c_vp(out.data_ptr())))
    return out


def _transpose_csr(net, rows, cols, vals_dev_order, n_cols, extra=None):
    """CSR of the TRANSPOSE (one row per variable): index-only host work; `vals_dev_order` are device values in the
    original COO order, gathered on the device."""
    import torch
    rows = np.asarray(rows, dtype=np.int64)
    cols = np.asarray(cols, dtype=np.int64)
    order = np.argsort(cols, kind="stable")
    counts = np.bincount(cols, minlength=n_cols)
    ptr = np.zeros(n_cols + 1, dtype=np.uint32)
    ptr[1:] = np.cumsum(counts).astype(np.uint32)
    idx = rows[order].astype(np.uint32)
    d_order = torch.from_numpy(order).to(vals_dev_order.device)
    return net.to_device(ptr.view(np.int32)), net.to_device(idx.view(np.int32)), vals_dev_order[d_order].contiguous()


def _points_spmv(net, csr, points, n_rows: int, g2=False):
    """out[r] = sum_k val[k] * points[idx[k]] over a CSR (ptr, idx, val) on the device (b200zk_points_spmv_dev)."""
    import torch
    ptr, idx, val = csr
    out = torch.empty((n_rows, 16 if g2 else 8), dtype=torch.int64, device=points.device)
    net.check(net._lib.b200zk_points_spmv_dev(net._h, 0, int(g2), c_vp(ptr.data_ptr()), c_vp(idx.data_ptr()),
                                              c_vp(val.data_ptr()), c_vp(points.data_ptr()), n_rows, c_vp(out.data_ptr())))
    return out


def ptau_key_points(net, r1cs, ptau) -> dict:
    """What snarkjs `zkey new` computes from an r1cs (formats.R1CS) and a prepared Powers-of-Tau file (formats.PTau), as
    CUDA tensors (the query vectors, ic) and host limb arrays (the six header points).  With L, L2, alpha L, beta L the
    Lagrange bases of the circuit's domain 2^k and H those of 2^(k+1):

      a_query[s] = sum_c A[c,s] L_c (+ L_{nc+s} for s <= n_public: the input-consistency rows, groth16/src/qap.rs:69-73)
      b_g1_query[s] / b_g2_query[s] = sum_c B[c,s] L_c / L2_c
      K[s] = sum_c (A[c,s] beta L_c + B[c,s] alpha L_c + C[c,s] L_c)  ->  ic = K[:n_public + 1], l_query = K[n_public + 1:]
      h_query[i] = H_{2i+1}   (ark-circom/src/circom/qap.rs:11-15, 94-110)

    alpha_1, beta_1, beta_2 come from the ceremony, gamma_2 = delta_2 and delta_1 are the generators: gamma = delta = 1
    until a phase-2 contribution.  Every product runs as b200zk_points_spmv_dev over one CSR per query (K over the stacked
    points [L | alpha L | beta L]); the host only reorders indices and moves the needed ceremony levels to the device."""
    import torch
    from .. import formats
    n_vars, nc = int(r1cs.n_wires), int(r1cs.n_constraints)
    n_public = int(r1cs.n_pub_out + r1cs.n_pub_in)
    n_inputs = n_public + 1
    k = formats.zkey_cir_power(nc, n_public)
    m = 1 << k
    net.use_torch_stream(0)
    lag, lag2, alag, blag = (net.to_device(ptau.lagrange(sid, k)) for sid in (12, 13, 14, 15))
    h_query = net.to_device(np.ascontiguousarray(ptau.lagrange(12, k + 1)[1::2]))
    dev = lag.device
    one = torch.from_numpy(_mont_limbs(1).view(np.int64)).to(dev).reshape(1, 4)

    def coo(i):
        rows, cols = np.asarray(r1cs.rows[i], np.int64), np.asarray(r1cs.cols[i], np.int64)
        vals = net.fr_convert(net.to_device(np.ascontiguousarray(r1cs.vals[i], dtype=np.uint64).reshape(-1, 4)), to_mont=True)
        return rows, cols, vals

    (ar, ac, av), (br, bc, bv), (cr, cc, cv) = coo(0), coo(1), coo(2)
    ar = np.concatenate([ar, np.arange(nc, nc + n_inputs)])          # input-consistency rows a[nc + j] = z[j]
    ac = np.concatenate([ac, np.arange(n_inputs)])
    av = torch.cat([av, one.expand(n_inputs, 4)], dim=0).contiguous()
    a_csr = _transpose_csr(net, ar, ac, av, n_vars)
    b_csr = _transpose_csr(net, br, bc, bv, n_vars)
    k_csr = _transpose_csr(net, np.concatenate([cr, br + m, ar + 2 * m]), np.concatenate([cc, bc, ac]),
                           torch.cat([cv, bv, av], dim=0), n_vars)
    a_query = _points_spmv(net, a_csr, lag, n_vars)
    b_g1_query = _points_spmv(net, b_csr, lag, n_vars)
    b_g2_query = _points_spmv(net, b_csr, lag2, n_vars, g2=True)
    kq = _points_spmv(net, k_csr, torch.cat([lag, alag, blag], dim=0), n_vars)
    g1 = _fixed_base(net, one).cpu().numpy().view(np.uint64)[0]
    g2 = _fixed_base(net, one, g2=True).cpu().numpy().view(np.uint64)[0]
    return dict(n_vars=n_vars, n_public=n_public, domain_size=m, a_query=a_query, b_g1_query=b_g1_query,
                b_g2_query=b_g2_query, ic=kq[:n_inputs].contiguous(), l_query=kq[n_inputs:].contiguous(), h_query=h_query,
                alpha_g1=ptau.alpha_g1, beta_g1=ptau.beta_g1, beta_g2=ptau.beta_g2, gamma_g2=g2, delta_g1=g1, delta_g2=g2)


def setup_from_ptau(net, r1cs, ptau):
    """Groth16 setup from a ceremony instead of known toxic waste: snarkjs `zkey new` (what the reference's
    scripts/phase2_proving_key.sh runs before proving) on the GPU.  r1cs: formats.R1CS; ptau: formats.PTau (read_ptau).
    Returns (ProvingKey on the device, VerifyingKey as host limb arrays, ConstraintMatrices) like circuit_specific_setup.
    The key has delta = 1: it needs a phase-2 contribution before production use."""
    q = ptau_key_points(net, r1cs, ptau)
    n_inputs = q["n_public"] + 1
    vk_points = np.concatenate([q["alpha_g1"], q["beta_g1"], q["delta_g1"], q["beta_g2"], q["delta_g2"]])
    pk = ProvingKey.from_device(net, q["a_query"], q["b_g1_query"], q["b_g2_query"], q["l_query"], q["h_query"], n_inputs,
                                vk_points)
    vk = VerifyingKey(alpha_g1=q["alpha_g1"], beta_g2=q["beta_g2"], gamma_g2=q["gamma_g2"], delta_g2=q["delta_g2"],
                      gamma_abc_g1=q["ic"].cpu().numpy().view(np.uint64))
    coo = lambda i: (r1cs.rows[i], r1cs.cols[i], r1cs.vals[i])
    mats = ConstraintMatrices(net, n_inputs, int(r1cs.n_constraints), coo(0), coo(1), values_montgomery_depth=-1)
    return pk, vk, mats


def circuit_specific_setup(net, n_vars: int, n_inputs: int, num_constraints: int, a_coo, b_coo, c_coo, toxic,
                           values_montgomery_depth: int = -1, g1_generator=None, g2_generator=None):
    """a_coo / b_coo / c_coo: (rows, cols, vals (nnz, 4) u64) of the R1CS matrices; toxic = (tau, alpha, beta, gamma, delta)
    canonical ints.  g1_generator / g2_generator: affine Montgomery limbs (8 / 16 u64) of the group elements every query
    is a multiple of -- ark-groth16 draws them at random (`E::G1::rand(rng)`), None = the standard generators.
    Returns (ProvingKey on the device, VerifyingKey as host limb arrays, ConstraintMatrices)."""
    import torch
    tau, alpha, beta, gamma, delta = (int(x) % R for x in toxic)
    m = 1
    while m < num_constraints + n_inputs:
        m <<= 1
    dev = torch.device("cuda", net.device)
    net.use_torch_stream(0)
    # Lagrange coefficients L_i(tau) = iNTT(tau^k)[i]
    u = net.ntt_dev(_powers(net, tau, 1, m), inverse=True)

    def conv(vals):
        d = net.to_device(np.ascontiguousarray(vals, dtype=np.uint64).reshape(-1, 4))
        if values_montgomery_depth < 0:
            return net.fr_convert(d, to_mont=True, times=-values_montgomery_depth)
        if values_montgomery_depth > 0:
            return net.fr_convert(d, to_mont=False, times=values_montgomery_depth)
        return d

    one = torch.from_numpy(_mont_limbs(1).view(np.int64)).to(dev).reshape(1, 4)
    evals = []
    for k, (rows, cols, vals) in enumerate((a_coo, b_coo, c_coo)):
        rows, cols = np.asarray(rows, dtype=np.int64), np.asarray(cols, dtype=np.int64)
        keep = rows < num_constraints
        rows, cols = rows[keep], cols[keep]
        dv = conv(np.asarray(vals)[keep])
        if k == 0:      # input-consistency rows: a[num_constraints + j] = z[j]   (groth16/src/qap.rs:69-73)
            rows = np.concatenate([rows, np.arange(num_constraints, num_constraints + n_inputs)])
            cols = np.concatenate([cols, np.arange(n_inputs)])
            dv = torch.cat([dv, one.expand(n_inputs, 4)], dim=0).contiguous()
        ptr, idx, tv = _transpose_csr(net, rows, cols, dv, n_vars)
        out = torch.empty((n_vars, 4), dtype=torch.int64, device=dev)
        net.check(net._lib.b200zk_fr_spmv_dev(net._h, c_vp(ptr.data_ptr()), c_vp(idx.data_ptr()), c_vp(tv.data_ptr()),
                                              c_vp(u.data_ptr()), n_vars, c_vp(out.data_ptr())))
        evals.append(out)
    a_t, b_t, c_t = evals

    def lincomb(s3):
        s = np.concatenate([_mont_limbs(beta), _mont_limbs(alpha), _mont_limbs(1), _mont_limbs(s3)])
        out = torch.empty_like(a_t)
        net.check(net._lib.b200zk_fr_lincomb_dev(net._h, c_vp(a_t.data_ptr()), c_vp(b_t.data_ptr()), c_vp(c_t.data_ptr()),
                                                 c_vp(s.ctypes.data), n_vars, c_vp(out.data_ptr())))
        return out

    l_all = lincomb(pow(delta, -1, R))              # (beta A_j + alpha B_j + C_j) / delta
    ic_all = lincomb(pow(gamma, -1, R))             # ... / gamma  (public inputs)
    # h-query scalars: iNTT over the 2m-domain of delta^-1 tau^k (k < 2m - 1), odd entries   (qap.rs:94-110)
    hs = _powers(net, tau, pow(delta, -1, R), 2 * m)
    hs[2 * m - 1] = 0
    hs = net.ntt_dev(hs, inverse=True)[1::2].contiguous()
    custom = g1_generator is not None or g2_generator is not None
    if custom and (g1_generator is None or g2_generator is None):
        raise ValueError("give both generators or neither")
    _fb = (lambda sc, g2=False: _fixed_base_custom(net, g2_generator if g2 else g1_generator, sc, g2)) if custom else \
        (lambda sc, g2=False: _fixed_base(net, sc, g2))
    a_query = _fb(a_t)
    b_g1_query = _fb(b_t)
    b_g2_query = _fb(b_t, g2=True)
    l_query = _fb(l_all[n_inputs:].contiguous())
    h_query = _fb(hs)
    ic = _fb(ic_all[:n_inputs].contiguous())
    consts = torch.from_numpy(np.stack([_mont_limbs(v) for v in (alpha, beta, delta, gamma)]).view(np.int64)).to(dev)
    g1c = _fb(consts).cpu().numpy().view(np.uint64)          # alpha, beta, delta, gamma in G1
    g2c = _fb(consts, g2=True).cpu().numpy().view(np.uint64)
    vk_points = np.concatenate([g1c[0], g1c[1], g1c[2], g2c[1], g2c[2]])
    pk = ProvingKey.from_device(net, a_query, b_g1_query, b_g2_query, l_query, h_query, n_inputs, vk_points)
    vk = VerifyingKey(alpha_g1=g1c[0], beta_g2=g2c[1], gamma_g2=g2c[3], delta_g2=g2c[2],
                      gamma_abc_g1=ic.cpu().numpy().view(np.uint64))
    mats = ConstraintMatrices(net, n_inputs, num_constraints, a_coo, b_coo, values_montgomery_depth=values_montgomery_depth)
    return pk, vk, mats
