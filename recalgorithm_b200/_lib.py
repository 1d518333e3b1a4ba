"""ctypes binding of libctr_b200.so -- the C ABI declared in include/ctr_b200.h.

There is deliberately no fallback: if the library has not been built, or a compute entry point
fails, the caller gets an exception.  Nothing here imports ``oracle``.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_int, c_int64, c_void_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libctr_b200.so")

CTR_OK, CTR_ERR_INVALID_ARG, CTR_ERR_UNSUPPORTED, CTR_ERR_CUDA = 0, -1, -2, -3

_P = c_void_p       # device pointers travel as integers / None
_I = c_int64

# name -> (restype, argtypes); mirrors include/ctr_b200.h one to one (tests check the symbol list
# against the header).
SIGNATURES = {
    "ctr_last_error": (c_char_p, []),
    "ctr_version": (c_int, []),
    "ctr_device_info": (c_int, [POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "ctr_enable_peer_access": (c_int, [c_int]),
    "ctr_peer_alloc": (c_int, [_I, POINTER(c_void_p)]),
    "ctr_peer_free": (c_int, [_P]),
    "ctr_ipc_export": (c_int, [_P, ctypes.c_char_p]),
    "ctr_ipc_import": (c_int, [ctypes.c_char_p, POINTER(c_void_p)]),
    "ctr_ipc_close": (c_int, [_P]),
    "ctr_vmm_granularity": (c_int, [POINTER(c_int64), POINTER(c_int64)]),
    "ctr_vmm_alloc": (c_int, [_I, _I, POINTER(c_void_p), POINTER(c_int), POINTER(c_int64)]),
    "ctr_vmm_import": (c_int, [c_int, _I, _I, POINTER(c_void_p)]),
    "ctr_vmm_free": (c_int, [_P]),
    "ctr_kernel_launches": (c_int64, []),
    "ctr_embed_fm2_fwd": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "ctr_embed_fm2_bwd": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P]),
    "ctr_embed_seq_fwd": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P]),
    "ctr_sigmoid_ce": (c_int, [_P, _P, _P, _I, _P, _P, _P]),
    "ctr_embed_scatter_add": (c_int, [_P, _P, _P, _P, _I, _I, _I, _P]),
    "ctr_embed_fm2_fwd_sharded": (c_int, [_P, _I, _P, _P, _I, _I, _I, _P, _P, _P]),
    "ctr_embed_fm2_lin_fwd": (c_int, [_P, _P, _P, c_int, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "ctr_embed_fm2_lin_bwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "ctr_embed_fm2_fwd_ids32": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P, _P, _P]),
    "ctr_embed_fm2_fwd_sharded_ids32": (c_int, [_P, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P]),
    "ctr_embed_fm2_lin_fwd_sharded": (c_int, [_P, _I, _P, _P, c_int, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    "ctr_embed_fm2_lin_bwd_push": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _I, _P, _P, _P]),
    "ctr_sharded_plan": (c_int, [_P, _P, c_int, _I, _I, _I, _I, _P, _P, _I, _P, _P, _P, _P]),
    "ctr_embed_fm2_bwd_push": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _I, _P, _P]),
    "ctr_sharded_grad_push": (c_int, [_P, _P, _I, _I, _I, _I, _I, _P, _I, _P]),
    "ctr_rows_scatter_add": (c_int, [_P, _I, _I, _P, _P, _P, _I, _P]),
    "ctr_adam_rows": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P, _P, _I, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                              ctypes.c_float, _P, _P]),
    "ctr_embed_bi_fwd": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "ctr_embed_bi_bwd": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P]),
    "ctr_embed_fwbi_fwd": (c_int, [_P, _P, _P, c_int, _I, _I, _I, _P, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    "ctr_fwbi_fwd": (c_int, [_P, _I, _I, _I, _P, _I, _P, _P, _P, _P, _P, _P]),
    "ctr_fwbi_bwd": (c_int, [_P, _P, _P, _I, _I, _I, _P, _I] + [_P] * 8),
    "ctr_fwfm_fwd": (c_int, [_P, _P, _I, _I, _I, _P, _P]),
    "ctr_fwfm_bwd": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "ctr_ffm_fwd": (c_int, [_P, _I, _I, _I, _P, _P]),
    "ctr_ffm_bwd": (c_int, [_P, _P, _I, _I, _I, _P, _P]),
    "ctr_afm_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P]),
    "ctr_afm_bwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P]),
    "ctr_bst_param_count": (_I, [_I, _I, _I]),
    "ctr_bst_transformer_fwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, c_int, _P, _P]),
    "ctr_bst_transformer_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, c_int, _P, _P, _P, _P, _P]),
    "ctr_adam_indexed_slices": (c_int, [_P, _P, _P, _I, _P, _I, _I, _P, _P, _I, _P, _P, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                        ctypes.c_float, _P, _P, _P]),
    "ctr_embed_fm2_bwd_adam": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _I, _P, _P, _P, ctypes.c_float, ctypes.c_float,
                                       ctypes.c_float, ctypes.c_float, _P, _P, _P]),
    "ctr_adam_rows_dedup": (c_int, [_P, _P, _P, _I, _I, _I, _P, _P, _P, _I, _I, _P, _P, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                    ctypes.c_float, _P, _P, _P]),
    "ctr_adam_dense_rest": (c_int, [_P, _P, _P, _I, _I, _I, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, _P, _P]),
    "ctr_first_order_fwd": (c_int, [_P, _P, _P, _I, _I, ctypes.c_float, _P, _P]),
    "ctr_crossed_indicator_fwd": (c_int, [_P, _P, _I, _I, _I, ctypes.c_uint64, _P, _P, _P, _P]),
    "ctr_crossed_indicator_bwd": (c_int, [_P, _P, _I, _I, _I, ctypes.c_uint64, _P, _P, _P, _P]),
    "ctr_ftrl_apply": (c_int, [_P, _P, _P, _P, _I, ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_float, _P]),
    "ctr_bag_lookup_fwd": (c_int, [_P, _I, _I, _P, _P, _I, _P, _I, _P]),
    "ctr_bag_lookup_bwd": (c_int, [_P, _I, _I, _I, _P, _P, _I, _P, _P]),
    "ctr_cross_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _P, _P]),
    "ctr_cross_bwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P]),
    "ctr_embed_cross_fwd": (c_int, [_P, _P, _P, c_int, _I, _I, _I, _P, _P, _I, _P, _P, _P]),
    "ctr_cin_fwd_workspace_bytes": (c_int64, [_I, _I, _I, _I, _I]),
    "ctr_cin_fwd": (c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, c_int, _P, _I, _P]),
    "ctr_cin_bwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _P]),
    "ctr_cin_bwd_workspace_bytes": (c_int64, [_I, _I, _I, _I, _I]),
    "ctr_din_attention_fwd": (c_int, [_P] * 9 + [_I, _I, _I, c_int, _P, _P, _P, _P]),
    "ctr_din_attention_bwd": (c_int, [_P] * 11 + [_I, _I, _I, c_int, _P, _P, _P, _P, _P]),
    "ctr_senet_fwd": (c_int, [_P, _P, _P, _I, _I, _I, _I, _P, _P]),
    "ctr_senet_bwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P]),
    "ctr_bilinear_fwd": (c_int, [_P, _P, _I, _I, _I, c_int, _P, _P]),
    "ctr_bilinear_bwd": (c_int, [_P, _P, _P, _I, _I, _I, c_int, _P, _P, _P]),
    "ctr_bilinear_set_rr": (c_int, [c_int]),
    "ctr_pnn_workspace_bytes": (c_int, [_I, _I, _I, c_int, POINTER(c_int64)]),
    "ctr_pnn_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, c_int, _P, _P, _I, _P]),
    "ctr_pnn_bwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, c_int, _P, _P, _P, _P, _P, _I, _P]),
    "ctr_dien_workspace_bytes": (c_int, [_I, _I, _I, _I, POINTER(c_int64)]),
    "ctr_dien_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, c_int, _P, _P, _P, _I, _P]),
    "ctr_dien_bwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, c_int, _P, _P, _P, _P, _I, _P]),
    "ctr_dien_aux_workspace_bytes": (c_int, [_I, _I, _I, _I, _I, POINTER(c_int64)]),
    "ctr_dien_aux_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P]),
    "ctr_dien_bwd_aux": (c_int, [_P] * 8 + [_I] * 5 + [c_int] + [_P] * 6 + [_I, _P]),
    "ctr_residual_unit_workspace_bytes": (c_int, [_I, _I, _I, POINTER(c_int64)]),
    "ctr_residual_unit_fwd": (c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _I, _P]),
    "ctr_residual_unit_bwd": (c_int, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _I, _P]),
    "ctr_mmoe_workspace_bytes": (c_int, [_I, _I, _I, _I, _I, POINTER(c_int64)]),
    "ctr_mmoe_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _I, _P]),
    "ctr_mmoe_bwd": (c_int, [_P] * 6 + [_I] * 5 + [_P] * 5 + [_I, _P]),
    "ctr_ple_workspace_bytes": (c_int, [_I, _I, _I, _I, _P, _I, _I, POINTER(c_int64)]),
    "ctr_ple_fwd": (c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _I, _I, _P, _P, _P, _I, _P]),
    "ctr_ple_bwd": (c_int, [_P] * 6 + [_I] * 4 + [_P, _I, _I] + [_P] * 5 + [_I, _P]),
    "ctr_autoint_workspace_bytes": (c_int, [_I, _I, _I, _I, _I, POINTER(c_int64)]),
    "ctr_autoint_fwd": (c_int, [_P] * 5 + [_I] * 5 + [_P, _P, _I, _P]),
    "ctr_autoint_bwd": (c_int, [_P] * 7 + [_I] * 5 + [_P] * 6 + [_I, _P]),
    "ctr_multitask_sigmoid_ce": (c_int, [_P, _P, _I, _I, c_int] + [_P] * 6),
    "ctr_multitask_gram_workspace_bytes": (c_int, [_I, _I, POINTER(c_int64)]),
    "ctr_multitask_gram": (c_int, [_P, _I, _I, _I, _P, _P, _I, _P]),
    "ctr_pcgrad_combine": (c_int, [_P, _I, _I, _I, _P, _P, _P, _P, _P]),
    "ctr_gradnorm_update": (c_int, [_P, _P, _P, _I, ctypes.c_float, ctypes.c_float, _P, _P, _P, _P]),
}


class CtrError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libctr_b200 error {code}: {msg}")
        self.code = code


class CtrInvalidArgument(CtrError, ValueError):
    """Maps the reference's Python-side ValueError / assert behaviour for bad arguments."""


_lib = None


def lib() -> ctypes.CDLL:
    """Load (once) and return the library; raises if it was never built -- no CPU fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m recalgorithm_b200.build` "
                "(or __graft_entry__.build()).  There is no CPU fallback.")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)      # AttributeError if the .so lacks a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc: int) -> None:
    if rc != CTR_OK:
        msg = lib().ctr_last_error().decode("utf-8", "replace")
        if rc in (CTR_ERR_INVALID_ARG, CTR_ERR_UNSUPPORTED):
            raise CtrInvalidArgument(rc, msg)
        raise CtrError(rc, msg)


def kernel_launches() -> int:
    return int(lib().ctr_kernel_launches())
