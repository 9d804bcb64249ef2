"""ctypes loader for libb200zk.so -- the only compute backend of this package.

There is deliberately no fallback: if the CUDA library cannot be loaded or no GPU is present,
every operation raises (`B200zkError`)."""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200zk.so")

OK, ERR_LENGTH, ERR_DOMAIN, ERR_CUDA, ERR_ARG, ERR_OOM, ERR_SHORT_BUFFER = range(7)
_ERR_NAMES = {1: "BAD_LENGTH", 2: "BAD_DOMAIN", 3: "CUDA", 4: "BAD_ARG", 5: "OOM", 6: "SHORT_BUFFER"}


class B200zkError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__("b200zk error %d (%s): %s" % (code, _ERR_NAMES.get(code, "?"), message))
        self.code = code
        self.message = message


_lib = None

c_u64p = ctypes.POINTER(ctypes.c_uint64)
c_vp = ctypes.c_void_p

# name -> (restype, argtypes); must list every symbol declared in include/b200zk.h
SIGNATURES = {
    "b200zk_version": (ctypes.c_char_p, []),
    "b200zk_ctx_create": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(c_vp)]),
    "b200zk_ctx_destroy": (None, [c_vp]),
    "b200zk_last_error": (ctypes.c_char_p, [c_vp]),
    "b200zk_ctx_set_stream": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp]),
    "b200zk_ctx_sync": (ctypes.c_int, [c_vp, ctypes.c_int]),
    "b200zk_profile_enable": (ctypes.c_int, [c_vp, ctypes.c_int]),
    "b200zk_profile_reset": (ctypes.c_int, [c_vp]),
    "b200zk_profile_json": (ctypes.c_int, [c_vp, ctypes.c_char_p, ctypes.c_size_t]),
    "b200zk_launch_count": (ctypes.c_uint64, [c_vp]),
    "b200zk_msm_g1": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp, ctypes.c_size_t, c_vp,
                                     ctypes.POINTER(ctypes.c_int)]),
    "b200zk_msm_g2": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp, ctypes.c_size_t, c_vp,
                                     ctypes.POINTER(ctypes.c_int)]),
    "b200zk_msm_staged_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_msm_g1_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_msm_g2_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_msm_table_windows": (ctypes.c_uint, [ctypes.c_uint]),
    "b200zk_msm_table_auto_window": (ctypes.c_uint, [ctypes.c_size_t]),
    "b200zk_msm_table_build_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, ctypes.c_uint, c_vp]),
    "b200zk_msm_table_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, ctypes.c_size_t, ctypes.c_uint, c_vp]),
    "b200zk_g1_sum_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp, ctypes.POINTER(ctypes.c_int)]),
    "b200zk_g2_sum_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp, ctypes.POINTER(ctypes.c_int)]),
    "b200zk_ntt_fr": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, ctypes.c_uint, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                     ctypes.c_int, ctypes.c_uint]),
    "b200zk_ntt_fr_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, ctypes.c_uint, ctypes.c_int, ctypes.c_int,
                                         ctypes.c_uint]),
    "b200zk_ntt_fr_fourstep_cols_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, ctypes.c_uint, ctypes.c_uint,
                                                       ctypes.c_uint, ctypes.c_uint64, ctypes.c_int]),
    "b200zk_ntt_fr_fourstep_cols_p2p_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, ctypes.POINTER(c_vp), ctypes.c_uint,
                                                           ctypes.c_uint, ctypes.c_uint, ctypes.c_uint, ctypes.c_uint64,
                                                           ctypes.c_int]),
    "b200zk_peer_alloc": (ctypes.c_int, [c_vp, ctypes.c_size_t, ctypes.POINTER(c_vp), c_vp]),
    "b200zk_peer_open": (ctypes.c_int, [c_vp, c_vp, ctypes.POINTER(c_vp)]),
    "b200zk_peer_close": (ctypes.c_int, [c_vp, c_vp]),
    "b200zk_peer_free": (ctypes.c_int, [c_vp, c_vp]),
    "b200zk_msm_exchange_sum_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.POINTER(c_vp), ctypes.c_uint,
                                                   ctypes.c_uint, ctypes.c_uint64, c_vp]),
    "b200zk_ntt_fr_batched_post_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, ctypes.c_uint, ctypes.c_uint,
                                                      ctypes.c_int, ctypes.c_uint, ctypes.c_int, ctypes.c_uint64,
                                                      ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64]),
    "b200zk_fr_mul_sub_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t]),
    "b200zk_h_circom": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, ctypes.c_uint, c_vp]),
    "b200zk_h_circom_dev": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, ctypes.c_uint, c_vp]),
    "b200zk_qap_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, ctypes.c_size_t,
                                      c_vp, ctypes.c_uint, c_vp, c_vp, c_vp]),
    "b200zk_fr_convert_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, ctypes.c_size_t, ctypes.c_int, ctypes.c_int]),
    "b200zk_r1cs_check_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                             ctypes.c_size_t, c_vp, c_u64p, c_u64p]),
    "b200zk_pk_upload": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, ctypes.c_size_t,
                                        ctypes.c_size_t, c_vp, ctypes.POINTER(c_vp)]),
    "b200zk_pk_upload_dev": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, ctypes.c_size_t,
                                            ctypes.c_size_t, c_vp, ctypes.POINTER(c_vp)]),
    "b200zk_groth16_prove_dev": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_int, c_vp]),
    "b200zk_pk_free": (None, [c_vp, c_vp]),
    "b200zk_pk_precompute": (ctypes.c_int, [c_vp, c_vp, ctypes.c_uint]),
    "b200zk_pk_table_bytes": (ctypes.c_size_t, [c_vp]),
    "b200zk_groth16_prove": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_int, c_vp]),
    "b200zk_points_matmul_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, ctypes.c_size_t, c_vp,
                                                ctypes.c_size_t, c_vp]),
    "b200zk_groth16_verify": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, c_vp, c_vp, c_vp, c_vp,
                                             ctypes.POINTER(ctypes.c_int)]),
    "b200zk_vk_alphabeta_12": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp]),
    "b200zk_points_compress_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_points_decompress_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, ctypes.c_int, c_vp,
                                                    ctypes.POINTER(ctypes.c_size_t)]),
    "b200zk_zkey_load": (ctypes.c_int, [c_vp, c_vp, ctypes.c_size_t, ctypes.c_uint, ctypes.POINTER(c_vp)]),
    "b200zk_zkey_free": (None, [c_vp, c_vp]),
    "b200zk_zkey_info": (ctypes.c_int, [c_vp] + [ctypes.POINTER(ctypes.c_size_t)] * 4),
    "b200zk_zkey_prove": (ctypes.c_int, [c_vp, c_vp, c_vp, ctypes.c_size_t, c_vp, c_vp, c_vp, ctypes.c_char_p,
                                         ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p, ctypes.POINTER(ctypes.c_size_t)]),
    "b200zk_xyzz_sum_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, ctypes.c_size_t, c_vp]),
    "b200zk_groth16_assemble_dev": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_int, c_vp]),
    "b200zk_fixed_base_mul_dev": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_fr_powers_dev": (ctypes.c_int, [c_vp, c_vp, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_fr_spmv_dev": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_points_spmv_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_points_scale_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp, c_vp]),
    "b200zk_points_intt_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_uint, c_vp]),
    "b200zk_points_ntt_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_uint, c_vp]),
    "b200zk_points_mul_powers_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp, c_vp, c_vp]),
    "b200zk_points_sub_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_points_encode_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, ctypes.c_int, c_vp]),
    "b200zk_points_decode_dev": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, ctypes.c_size_t, ctypes.c_int, ctypes.c_int,
                                                c_vp, ctypes.POINTER(ctypes.c_size_t), ctypes.POINTER(ctypes.c_size_t)]),
    "b200zk_blake2b512_init": (ctypes.c_int, [c_vp]),
    "b200zk_blake2b512_update": (ctypes.c_int, [c_vp, c_vp, ctypes.c_size_t]),
    "b200zk_blake2b512_final": (ctypes.c_int, [c_vp, c_vp]),
    "b200zk_fr_lincomb_dev": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, c_vp]),
    "b200zk_g1_generate_dev": (ctypes.c_int, [c_vp, ctypes.c_uint64, ctypes.c_size_t, c_vp]),
    "b200zk_g2_generate_dev": (ctypes.c_int, [c_vp, ctypes.c_uint64, ctypes.c_size_t, c_vp]),
    "b200zk_fr_generate_dev": (ctypes.c_int, [c_vp, ctypes.c_uint64, ctypes.c_size_t, c_vp]),
    "b200zk_group_create": (ctypes.c_int, [ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.POINTER(c_vp)]),
    "b200zk_group_destroy": (None, [c_vp]),
    "b200zk_group_size": (ctypes.c_int, [c_vp]),
    "b200zk_group_ctx": (c_vp, [c_vp, ctypes.c_int]),
    "b200zk_group_last_error": (ctypes.c_char_p, [c_vp]),
    "b200zk_group_msm_g1": (ctypes.c_int, [c_vp, c_vp, ctypes.c_size_t, c_vp, ctypes.c_size_t, c_vp, ctypes.POINTER(ctypes.c_int)]),
    "b200zk_group_msm_g2": (ctypes.c_int, [c_vp, c_vp, ctypes.c_size_t, c_vp, ctypes.c_size_t, c_vp, ctypes.POINTER(ctypes.c_int)]),
    "b200zk_group_ntt_fr": (ctypes.c_int, [c_vp, c_vp, ctypes.c_uint, ctypes.c_int]),
    "b200zk_group_h_circom": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, ctypes.c_uint, c_vp]),
    "b200zk_group_pk_upload": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, ctypes.c_size_t,
                                              ctypes.c_size_t, c_vp, ctypes.POINTER(c_vp)]),
    "b200zk_group_pk_free": (None, [c_vp, c_vp]),
    "b200zk_group_pk_table_bytes": (ctypes.c_size_t, [c_vp]),
    "b200zk_group_groth16_prove": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b200zk_group_r1cs_upload": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, ctypes.c_size_t, ctypes.c_size_t,
                                                ctypes.c_size_t, ctypes.c_uint, ctypes.c_int, ctypes.POINTER(c_vp)]),
    "b200zk_group_r1cs_free": (None, [c_vp, c_vp]),
    "b200zk_group_r1cs_local_row_ptr": (ctypes.c_int, [c_vp, ctypes.c_size_t, ctypes.c_uint, ctypes.c_int, ctypes.c_int, c_vp]),
    "b200zk_group_groth16_prove_r1cs_dev": (ctypes.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b200zk_group_zkey_load": (ctypes.c_int, [c_vp, c_vp, ctypes.c_size_t, ctypes.c_uint, ctypes.POINTER(c_vp)]),
    "b200zk_group_zkey_free": (None, [c_vp, c_vp]),
    "b200zk_group_zkey_info": (ctypes.c_int, [c_vp] + [ctypes.POINTER(ctypes.c_size_t)] * 4),
    "b200zk_group_zkey_table_bytes": (ctypes.c_size_t, [c_vp]),
    "b200zk_group_zkey_prove": (ctypes.c_int, [c_vp, c_vp, c_vp, ctypes.c_size_t, c_vp, c_vp, c_vp, ctypes.c_char_p,
                                               ctypes.POINTER(ctypes.c_size_t), ctypes.c_char_p, ctypes.POINTER(ctypes.c_size_t)]),
    "b200zk_fr_op": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, c_vp, c_vp, ctypes.c_size_t]),
    "b200zk_test_field_op": (ctypes.c_int, [c_vp, ctypes.c_int, ctypes.c_int, c_vp, c_vp, c_vp, ctypes.c_size_t]),
    "b200zk_test_arith": (ctypes.c_int, [c_vp, ctypes.c_int, c_vp, ctypes.c_size_t, c_vp]),
}


def lib():
    """Load libb200zk.so (built by distributed_groth16_b200.build). Raises if missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200zkError(ERR_CUDA, "libb200zk.so not built (run `python -m distributed_groth16_b200.build`); "
                                        "there is no CPU fallback")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)            # AttributeError if the ABI and this table drift apart
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib
