"""Several GPUs of one box behind single calls: the Python face of `b200zk_group_*` (csrc/group.cu).

The reference reaches its parties through `Net: MpcSerNet` (dist-primitives/src/channel/mod.rs:8-56); `Group` is that handle
for "all the GPUs of this box, one host process".  The sharded MSM / four-step NTT / h pipeline / Groth16 prover run inside
the library (peer stores over NVLink instead of the king/client star), so the Rust prover flow of
groth16/src/prove.rs:106-136 can reach BASELINE config 5 through FFI without torch.distributed.  `parallel.py` keeps the
one-process-per-GPU (torchrun + NCCL) orchestration that bench.py's scaling runs use."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _native, formats
from ._native import B200zkError, c_vp
from .context import MpcNetError, _as_u64, _ptr
from .dist_primitives.dmsm import GroupElement

ZERO_FR = np.zeros(4, dtype=np.uint64)


class Group:
    def __init__(self, devices):
        self._lib = _native.lib()
        devs = (ctypes.c_int * len(devices))(*[int(d) for d in devices])
        h = c_vp()
        rc = self._lib.b200zk_group_create(devs, len(devices), ctypes.byref(h))
        if rc != 0:
            raise B200zkError(rc, "cannot create a GPU group on devices %r (1, 2, 4 or 8 peer-connected GPUs; no CPU fallback)"
                              % (list(devices),))
        self._h = h
        self.devices = [int(d) for d in devices]
        self._bound0 = None

    def size(self) -> int:
        return int(self._lib.b200zk_group_size(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b200zk_group_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc: int):
        if rc != 0:
            msg = self._lib.b200zk_group_last_error(self._h).decode()
            if rc == _native.ERR_LENGTH:
                raise MpcNetError("Generic", msg)
            raise B200zkError(rc, msg)

    def _t0(self):
        """Slot 0 of device 0's context follows torch's current stream there, as `context.Net` binds its own: a tensor that torch
        wrote on device 0 is ready when the group's calls read it, and the group's writes are ready for torch."""
        import torch
        h = torch.cuda.current_stream(self.devices[0]).cuda_stream
        if h != self._bound0:
            ctx0 = self._lib.b200zk_group_ctx(self._h, 0)
            rc = self._lib.b200zk_ctx_set_stream(ctx0, 0, c_vp(h))
            if rc != 0:
                raise B200zkError(rc, self._lib.b200zk_last_error(ctx0).decode())
            self._bound0 = h

    def witness_to_device(self, w):
        """canonical (n, 4) u64 limbs (a .wtns witness) -> CUDA int64 (n, 4) tensor on device 0 in Montgomery form; the
        conversion runs on device 0 (b200zk_fr_convert_dev through the group's context there)."""
        import torch
        w = _as_u64(w, 4)
        self._t0()
        x = torch.from_numpy(w.view(np.int64)).to(torch.device("cuda", self.devices[0]))
        out = torch.empty_like(x)
        ctx0 = self._lib.b200zk_group_ctx(self._h, 0)
        rc = self._lib.b200zk_fr_convert_dev(ctx0, 0, c_vp(x.data_ptr()), c_vp(out.data_ptr()), w.shape[0], 1, 1)
        if rc != 0:
            raise B200zkError(rc, self._lib.b200zk_last_error(ctx0).decode())
        return out

    # -- d_msm -----------------------------------------------------------------------------------------------------------------
    def d_msm(self, bases, scalars, g2: bool | None = None) -> GroupElement:
        width = int(np.asarray(bases).shape[-1]) if np.asarray(bases).ndim == 2 else None
        if g2 is None:
            g2 = width == 16
        w = 16 if g2 else 8
        b, s = _as_u64(bases, w), _as_u64(scalars, 4)
        out = np.zeros(w, dtype=np.uint64)
        inf = ctypes.c_int(0)
        fn = self._lib.b200zk_group_msm_g2 if g2 else self._lib.b200zk_group_msm_g1
        self.check(fn(self._h, _ptr(b), b.shape[0] if b.size else 0, _ptr(s), s.shape[0] if s.size else 0, _ptr(out), ctypes.byref(inf)))
        return GroupElement(out, bool(inf.value), g2)

    # -- d_fft / d_ifft ----------------------------------------------------------------------------------------------------------
    def d_fft(self, x, inverse: bool = False) -> np.ndarray:
        buf = np.array(_as_u64(x, 4), dtype=np.uint64, copy=True)
        n = buf.shape[0]
        log_n = n.bit_length() - 1
        if n == 0 or (1 << log_n) != n:
            raise B200zkError(_native.ERR_DOMAIN, "length must be a power of two")
        self.check(self._lib.b200zk_group_ntt_fr(self._h, _ptr(buf), log_n, int(inverse)))
        return buf

    def d_ifft(self, x) -> np.ndarray:
        return self.d_fft(x, inverse=True)

    # -- ext_wit::h --------------------------------------------------------------------------------------------------------------
    def h(self, a, b, c) -> np.ndarray:
        a, b, c = (_as_u64(v, 4) for v in (a, b, c))
        m = a.shape[0]
        log_m = m.bit_length() - 1
        if m == 0 or (1 << log_m) != m or b.shape[0] != m or c.shape[0] != m:
            raise B200zkError(_native.ERR_DOMAIN, "a, b, c must share one power-of-two length")
        out = np.zeros((m, 4), dtype=np.uint64)
        self.check(self._lib.b200zk_group_h_circom(self._h, _ptr(a), _ptr(b), _ptr(c), log_m, _ptr(out)))
        return out


def local_row_ptr(row_ptr, num_constraints: int, log_m: int, n_gpus: int, rank: int) -> np.ndarray:
    """The CSR row_ptr (2^log_m / n_gpus + 1 entries) GPU `rank` of a group of n_gpus keeps of a matrix with `row_ptr`: local slot
    c rows + r holds global row r cols + rank cols / n_gpus + c (rows = 2^ceil(log_m / 2), cols = 2^floor(log_m / 2)).  Host
    only: the reorder GroupConstraintMatrices runs (b200zk_group_r1cs_local_row_ptr)."""
    ptr = np.ascontiguousarray(row_ptr, dtype=np.uint32)
    if ptr.shape != (int(num_constraints) + 1,):
        raise B200zkError(_native.ERR_ARG, "row_ptr must have num_constraints + 1 entries")
    out = np.zeros((1 << int(log_m)) // max(int(n_gpus), 1) + 1, dtype=np.uint32)
    lib = _native.lib()
    rc = lib.b200zk_group_r1cs_local_row_ptr(_ptr(ptr), int(num_constraints), int(log_m), int(n_gpus), int(rank), _ptr(out))
    if rc != 0:
        raise B200zkError(rc, "local_row_ptr(num_constraints=%d, log_m=%d, n_gpus=%d, rank=%d) refused"
                          % (num_constraints, log_m, n_gpus, rank))
    return out


class GroupConstraintMatrices:
    """A and B of a circuit (arguments as groth16.qap.ConstraintMatrices) sharded over the GPUs of a Group: GPU g keeps the
    rows of its slice of the column layout of the 2^log_m domain, so the QAP of a proof is computed where the sharded h
    pipeline reads it."""

    def __init__(self, group: Group, num_inputs: int, num_constraints: int, a_coo, b_coo, values_montgomery_depth: int,
                 log_m: int, n_vars: int):
        self.group = group
        self.num_instance_variables, self.num_constraints = int(num_inputs), int(num_constraints)
        self.log_m, self.n_vars = int(log_m), int(n_vars)
        csr = []
        for rows, cols, vals in (a_coo, b_coo):
            ptr, col, val = formats.coo_to_csr(np.asarray(rows), np.asarray(cols), _as_u64(vals, 4), self.num_constraints)
            csr.append((ptr, col, np.ascontiguousarray(val.reshape(-1, 4))))
        (ap, ac, av), (bp, bc, bv) = csr
        h = c_vp()
        group.check(group._lib.b200zk_group_r1cs_upload(group._h, _ptr(ap), _ptr(ac), _ptr(av), _ptr(bp), _ptr(bc), _ptr(bv),
                                                        self.num_constraints, self.num_instance_variables, self.n_vars, self.log_m,
                                                        int(values_montgomery_depth), ctypes.byref(h)))
        self._h = h

    def free(self):
        if getattr(self, "_h", None):
            self.group._lib.b200zk_group_r1cs_free(self.group._h, self._h)
            self._h = None


def load_zkey(group: Group, zkey_bytes: bytes):
    """circom.load_zkey on a Group -> (GroupProvingKey, GroupConstraintMatrices, formats.ZKey).  The public-input rows snarkjs
    appends to A are dropped as there (ZKey.num_constraints): the QAP puts z[0..n_inputs) after the constraints itself."""
    from .groth16.circom import zkey_matrices_coo
    zk = formats.read_zkey(zkey_bytes)
    gpk = GroupProvingKey(group, zk.a_query, zk.b_g1_query, zk.b_g2_query, zk.l_query, zk.h_query, zk.n_inputs, zk.alpha_g1,
                          zk.beta_g1, zk.delta_g1, zk.beta_g2, zk.delta_g2)
    try:
        a_coo, b_coo = zkey_matrices_coo(zk)
        mats = GroupConstraintMatrices(group, zk.n_inputs, zk.num_constraints, a_coo, b_coo, values_montgomery_depth=1,
                                       log_m=gpk.m.bit_length() - 1, n_vars=zk.n_vars)
    except Exception:
        gpk.free()
        raise
    return gpk, mats, zk


class GroupProvingKey:
    """A proving key sharded over the GPUs of a Group (arguments as groth16.ProvingKey)."""

    def __init__(self, group: Group, a_query, b_g1_query, b_g2_query, l_query, h_query, n_inputs: int, alpha_g1, beta_g1, delta_g1,
                 beta_g2, delta_g2):
        aq, b1, b2, hq = _as_u64(a_query, 8), _as_u64(b_g1_query, 8), _as_u64(b_g2_query, 16), _as_u64(h_query, 8)
        lq = _as_u64(l_query, 8)
        self.group = group
        self.n_vars, self.m, self.n_inputs = aq.shape[0], hq.shape[0], int(n_inputs)
        vk = np.concatenate([np.asarray(p, dtype=np.uint64).reshape(-1) for p in (alpha_g1, beta_g1, delta_g1, beta_g2, delta_g2)])
        assert vk.size == 56
        h = c_vp()
        group.check(group._lib.b200zk_group_pk_upload(group._h, _ptr(aq), _ptr(b1), _ptr(b2), _ptr(lq) if lq.size else None, _ptr(hq),
                                                      self.n_vars, self.n_inputs, self.m, _ptr(vk), ctypes.byref(h)))
        self._h = h

    @property
    def table_bytes(self) -> int:
        return int(self.group._lib.b200zk_group_pk_table_bytes(self._h))

    def free(self):
        if getattr(self, "_h", None):
            self.group._lib.b200zk_group_pk_free(self.group._h, self._h)
            self._h = None

    def create_proof(self, z, a, b, c, r=None, s=None) -> bytes:
        """128 compressed proof bytes, identical to groth16.prove.create_proof on one GPU."""
        z, a, b, c = (_as_u64(v, 4) for v in (z, a, b, c))
        assert z.shape[0] == self.n_vars and a.shape[0] == self.m and b.shape[0] == self.m and c.shape[0] == self.m
        r = ZERO_FR if r is None else np.ascontiguousarray(r, dtype=np.uint64)
        s = ZERO_FR if s is None else np.ascontiguousarray(s, dtype=np.uint64)
        out = (ctypes.c_uint8 * 128)()
        self.group.check(self.group._lib.b200zk_group_groth16_prove(self.group._h, self._h, _ptr(z), _ptr(a), _ptr(b), _ptr(c), _ptr(r),
                                                                    _ptr(s), out))
        return bytes(out)

    def create_proof_r1cs(self, matrices: GroupConstraintMatrices, z_dev, r=None, s=None) -> bytes:
        """128 compressed proof bytes from the witness: z_dev is the full assignment as a CUDA int64 (n_vars, 4) tensor on
        cuda:devices[0], Montgomery form.  The QAP runs sharded on the group (b200zk_group_groth16_prove_r1cs_dev); the bytes
        equal create_proof's on the QAP of the same matrices."""
        import torch
        g = self.group
        if not isinstance(z_dev, torch.Tensor) or not z_dev.is_cuda or z_dev.device.index != g.devices[0] or z_dev.dtype != torch.int64:
            raise B200zkError(_native.ERR_ARG, "z_dev must be a CUDA int64 tensor on cuda:%d" % g.devices[0])
        if tuple(z_dev.shape) != (self.n_vars, 4):
            raise B200zkError(_native.ERR_ARG, "witness has %d entries, the key expects %d" % (int(z_dev.shape[0]), self.n_vars))
        z_dev = z_dev.contiguous()
        r = ZERO_FR if r is None else np.ascontiguousarray(r, dtype=np.uint64)
        s = ZERO_FR if s is None else np.ascontiguousarray(s, dtype=np.uint64)
        out = (ctypes.c_uint8 * 128)()
        g._t0()
        g.check(g._lib.b200zk_group_groth16_prove_r1cs_dev(g._h, self._h, matrices._h, c_vp(z_dev.data_ptr()), _ptr(r), _ptr(s), out))
        return bytes(out)
