"""snarkjs `groth16 prove` through the library's own file path (b200zk_zkey_load / b200zk_zkey_prove): the zkey is parsed and
its coefficient section sorted into CSR in C++ / CUDA, the witness read from the .wtns bytes and the JSON written by the
library, with no numpy on the way.  circom.groth16_prove is the Python path to the same texts.  GroupZKeyProver is the same on
a group.Group (b200zk_group_zkey_*), whose Python path is circom.groth16_prove_group."""
from __future__ import annotations

import ctypes

import numpy as np

from .. import _native
from ..context import Net, _as_u64

NO_TABLES = 0xFFFFFFFF
PROOF_JSON_MAX = 810                             # B200ZK_PROOF_JSON_MAX: the longest proof.json plus its NUL


def public_json_max(n_public: int) -> int:
    """B200ZK_PUBLIC_JSON_MAX: the longest public.json of n_public signals plus its NUL."""
    return 3 + 82 * int(n_public)


def _prove(check, call, n_public: int, wtns_bytes: bytes, r, s):
    """one b200zk_zkey_prove-shaped call(wtns, len, r, s, proof, proof.json, len, public.json, len) with buffers that always
    suffice -> (proof.json, public.json, proof bytes)"""
    w = bytes(wtns_bytes)
    rs = [None if v is None else np.ascontiguousarray(_as_u64(v, 4).reshape(4)) for v in (r, s)]
    ptr = lambda a: None if a is None else a.ctypes.data
    proof = (ctypes.c_uint8 * 128)()
    plen, ulen = ctypes.c_size_t(PROOF_JSON_MAX), ctypes.c_size_t(public_json_max(n_public))
    pbuf, ubuf = ctypes.create_string_buffer(plen.value), ctypes.create_string_buffer(ulen.value)
    check(call(w, len(w), ptr(rs[0]), ptr(rs[1]), proof, pbuf, ctypes.byref(plen), ubuf, ctypes.byref(ulen)))
    return pbuf.raw[:plen.value].decode(), ubuf.raw[:ulen.value].decode(), bytes(proof)


def _info(check, call) -> dict:
    v = [ctypes.c_size_t(0) for _ in range(4)]
    check(call(*(ctypes.byref(x) for x in v)))
    return dict(zip(("n_vars", "n_public", "domain_size", "num_constraints"), (int(x.value) for x in v)))


class ZKeyProver:
    """A .zkey resident in HBM.  table_window as b200zk_pk_precompute's c: 0 = the automatic table policy, NO_TABLES = none."""

    def __init__(self, net: Net, zkey_bytes: bytes, table_window: int = 0):
        self.net = net
        buf = bytes(zkey_bytes)                  # the library keeps nothing of it after the load
        h = _native.c_vp()
        self._h = None
        net.check(net._lib.b200zk_zkey_load(net._h, buf, len(buf), int(table_window), ctypes.byref(h)))
        self._h = h
        self._n_public = self.info()["n_public"]

    def info(self) -> dict:
        return _info(self.net.check, lambda *a: self.net._lib.b200zk_zkey_info(self._h, *a))

    def prove(self, wtns_bytes: bytes, r=None, s=None):
        """-> (text of proof.json, text of public.json, 128 proof bytes).  r, s: 4 Montgomery limbs each; None = drawn by the
        library from the OS."""
        return _prove(self.net.check, lambda *a: self.net._lib.b200zk_zkey_prove(self.net._h, self._h, *a), self._n_public,
                      wtns_bytes, r, s)

    def free(self):
        if self._h is not None:
            self.net._lib.b200zk_zkey_free(self.net._h, self._h)
            self._h = None

    def __del__(self):                           # a handle dropped without free() gives its HBM back
        try:
            self.free()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.free()


class GroupZKeyProver:
    """A .zkey resident on a Group (b200zk_group_zkey_*): the coefficient section sorted on GPU 0 straight into every GPU's
    QAP output slots, the point sections sharded from the bytes.  Methods as ZKeyProver's; errors through Group.check."""

    def __init__(self, group, zkey_bytes: bytes, table_window: int = 0):
        self.group = group
        buf = bytes(zkey_bytes)                  # the library keeps nothing of it after the load
        h = _native.c_vp()
        self._h = None
        group.check(group._lib.b200zk_group_zkey_load(group._h, buf, len(buf), int(table_window), ctypes.byref(h)))
        self._h = h
        self._n_public = self.info()["n_public"]

    def info(self) -> dict:
        return _info(self.group.check, lambda *a: self.group._lib.b200zk_group_zkey_info(self._h, *a))

    @property
    def table_bytes(self) -> int:
        return int(self.group._lib.b200zk_group_zkey_table_bytes(self._h))

    def prove(self, wtns_bytes: bytes, r=None, s=None):
        """-> (text of proof.json, text of public.json, 128 proof bytes), as ZKeyProver.prove."""
        return _prove(self.group.check, lambda *a: self.group._lib.b200zk_group_zkey_prove(self.group._h, self._h, *a),
                      self._n_public, wtns_bytes, r, s)

    def free(self):
        if self._h is not None:
            self.group._lib.b200zk_group_zkey_free(self.group._h, self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.free()
