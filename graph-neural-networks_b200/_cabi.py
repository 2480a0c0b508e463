"""ctypes binding of include/b200gf.h (libb200gf.so, built by build.py with nvcc for sm_90a).

There is NO fallback: if the library is missing `load()` raises, and every LSIGF call raises with it.
"""
import ctypes
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200gf.so")

F32, F64 = 0, 1
DTYPE = {torch.float32: F32, torch.float64: F64}      # the dtypes the kernels run in, as the ABI's enum
FEATURE_MAJOR, NODE_MAJOR = 0, 1
HOP_FWD, HOP_BWD = 0, 1
ACT_NONE, ACT_RELU = 0, 1

_lib = None

c_i64 = ctypes.c_int64
c_int = ctypes.c_int
c_vp = ctypes.c_void_p
c_sz = ctypes.c_size_t
PP = ctypes.POINTER(ctypes.c_void_p)

_SIGNATURES = {
    "b200gf_strerror": (ctypes.c_char_p, [c_int]),
    "b200gf_version": (c_int, []),
    "b200gf_launch_count": (c_i64, [c_int]),
    "b200gf_plan_create": (c_int, [PP, c_int, c_i64, c_int, PP, PP, PP, c_int]),
    "b200gf_plan_create_ops": (c_int, [PP, c_int, c_i64, c_i64, c_int, PP, PP, PP, PP, PP, PP, c_int]),
    "b200gf_plan_create_device": (c_int, [PP, c_int, c_i64, c_int, PP, PP, PP, PP, PP, PP, c_int]),
    "b200gf_plan_destroy": (None, [c_vp]),
    "b200gf_plan_info": (c_i64, [c_vp, c_int]),
    "b200gf_plan_set_l2_bytes": (c_int, [c_vp, c_i64]),
    "b200gf_plan_set_hop_windows": (c_int, [c_vp, c_i64]),
    "b200gf_forward": (c_int, [c_vp, c_vp, c_int, c_i64, c_vp, c_vp, c_int, c_vp, c_int, c_i64, c_vp, c_sz,
                               c_int, c_int, c_int, c_int, c_vp]),
    "b200gf_forward_act": (c_int, [c_vp, c_vp, c_int, c_i64, c_vp, c_vp, c_int, c_vp, c_int, c_i64, c_vp, c_sz,
                                   c_int, c_int, c_int, c_int, c_int, c_vp]),
    "b200gf_relu_backward": (c_int, [c_int, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i64, c_int, c_vp]),
    "b200gf_maxpool_forward": (c_int, [c_int, c_vp, c_i64, c_i64, c_int, c_vp, c_i64, c_int, c_vp, c_i64, c_vp, c_vp]),
    "b200gf_maxpool_backward": (c_int, [c_int, c_vp, c_i64, c_vp, c_i64, c_int, c_vp, c_i64, c_i64, c_vp]),
    "b200gf_backward": (c_int, [c_vp, c_vp, c_int, c_i64, c_vp, c_int, c_i64, c_vp, c_vp, c_int, c_i64, c_vp, c_vp,
                                c_int, c_vp, c_sz, c_int, c_int, c_int, c_int, c_vp]),
    "b200gf_workspace_bytes": (c_sz, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int]),
    "b200gf_profile_hops": (c_int, [c_vp, c_int]),
    "b200gf_profile_read": (c_int, [c_vp, ctypes.POINTER(ctypes.c_float), c_int]),
    "b200gf_hop": (c_int, [c_vp, c_int, c_int, c_vp, c_i64, c_vp, c_i64, c_int, c_vp]),
    "b200gf_hop_scatter": (c_int, [c_vp, c_int, c_int, c_vp, c_i64, c_vp, c_i64, c_int, PP, c_int, c_i64, c_i64, c_i64,
                                   c_int, c_i64, c_vp]),
    "b200gf_scatter_rows": (c_int, [c_int, c_vp, c_i64, c_i64, c_int, PP, c_int, c_i64, c_i64, c_i64, c_int, c_i64, c_vp]),
    "b200gf_hop_bcast": (c_int, [c_vp, c_int, c_int, c_vp, c_i64, c_int, PP, c_int, c_vp, c_i64, c_i64, c_vp]),
    "b200gf_hop_grid": (c_int, [c_vp, c_int, c_int, c_vp, c_i64, c_int, PP, c_int, c_i64, c_i64, PP, c_int, c_i64, c_i64, c_i64,
                                c_int, c_i64, c_vp]),
    "b200gf_bcast_rows": (c_int, [c_int, c_vp, c_i64, c_i64, c_int, PP, c_int, c_vp, c_i64, c_i64, c_vp]),
    "b200gf_symm_alloc": (c_int, [PP, c_sz]),
    "b200gf_symm_free": (c_int, [c_vp]),
    "b200gf_symm_export": (c_int, [c_vp, c_vp]),
    "b200gf_symm_import": (c_int, [c_vp, PP]),
    "b200gf_symm_close": (c_int, [c_vp]),
    "b200gf_peer_signal": (c_int, [PP, c_int, c_int, c_vp, c_vp]),
    "b200gf_peer_wait": (c_int, [c_vp, c_int, c_vp, c_vp]),
    "b200gf_ev_forward": (c_int, [c_int, c_i64, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_int,
                                  c_vp, c_vp]),
    "b200gf_ev_backward": (c_int, [c_int, c_i64, c_int, c_int, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64,
                                   c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b200gf_egate_attention_forward": (c_int, [c_int, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b200gf_egate_attention_backward": (c_int, [c_int, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b200gf_attention_forward": (c_int, [c_int, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b200gf_attention_backward": (c_int, [c_int, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                          c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b200gf_gated_hop_forward": (c_int, [c_int, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp,
                                         c_i64, c_vp, c_i64, c_vp]),
    "b200gf_gated_hop_backward": (c_int, [c_int, c_i64, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                          c_i64, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i64, c_vp]),
    "b200gf_nv_pack_taps": (c_int, [c_int, c_vp, c_vp, c_int, c_int, c_int, c_int, c_i64, c_vp]),
    "b200gf_nv_forward": (c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_int, c_vp, c_i64, c_vp, c_sz,
                                  c_int, c_int, c_int, c_int, c_vp]),
    "b200gf_nv_backward": (c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp,
                                   c_int, c_vp, c_sz, c_int, c_int, c_int, c_int, c_vp]),
    "b200gf_nv_workspace_bytes": (c_sz, [c_vp, c_int, c_int, c_int, c_int, c_i64, c_int]),
    "b200gf_arma_forward": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_i64, c_vp, c_i64,
                                    c_vp, c_vp, c_sz, c_vp]),
    "b200gf_arma_backward": (c_int, [c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp, c_i64, c_vp, c_vp,
                                     c_i64, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b200gf_arma_workspace_bytes": (c_sz, [c_vp, c_int, c_int, c_int, c_int, c_int, c_int]),
    "b200gf_tap_contract":(c_int, [c_int, c_i64, c_int, c_int, c_int, c_int, PP, ctypes.POINTER(c_i64), c_vp, c_vp,
                                    c_int, c_vp, c_i64, c_int, c_vp, c_sz, c_vp]),
    "b200gf_tap_contract_scratch_bytes": (c_sz, [c_int, c_int, c_int]),
    "b200gf_tap_grad": (c_int, [c_int, c_i64, c_int, c_int, c_int, c_int, c_vp, c_i64, PP, ctypes.POINTER(c_i64),
                                c_vp, c_vp, c_sz, c_vp]),
    "b200gf_tap_grad_scratch_bytes": (c_sz, [c_int, c_i64, c_int, c_int, c_int, c_int]),
    "b200gf_to_node_major": (c_int, [c_int, c_vp, c_vp, c_i64, c_i64, c_int, c_vp]),
    "b200gf_to_feature_major": (c_int, [c_int, c_vp, c_i64, c_vp, c_i64, c_int, c_vp]),
    "b200gf_pack_taps": (c_int, [c_int, c_vp, c_vp, c_int, c_int, c_int, c_int, c_int, c_vp]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES.keys())


def load():
    """Returns the loaded library; raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "b200gf: CUDA extension %s is missing — build it with `python graph-neural-networks_b200/build.py` "
            "(there is no CPU fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def stream():
    """The current CUDA stream's handle: every entry point enqueues its launches there."""
    return torch.cuda.current_stream().cuda_stream


def check(rc):
    if rc != 0:
        raise RuntimeError(load().b200gf_strerror(int(rc)).decode())


def ptr_array(ptrs):
    arr = (ctypes.c_void_p * len(ptrs))(*[ctypes.c_void_p(int(p)) for p in ptrs])
    return arr


def i64_array(vals):
    return (ctypes.c_int64 * len(vals))(*[int(v) for v in vals])
