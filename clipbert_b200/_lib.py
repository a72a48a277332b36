"""ctypes binding of libclipbert_sm90.so (the C ABI declared in include/clipbert_b200.h).

The product path has no CPU or eager-PyTorch fallback: if the library is missing or fails to load,
every op raises. torch is used only for device memory, streams and torch.distributed.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libclipbert_sm90.so")

CB_GEMM_TN, CB_GEMM_WGRAD = 0, 1
ACT_NONE, ACT_RELU, ACT_GELU, ACT_TANH, ACT_GELU_STASH_GRAD = 0, 1, 2, 3, 4
AUX_NONE, AUX_RELU_MASK, AUX_GELU_GRAD, AUX_TANH_GRAD, AUX_MUL = 0, 1, 2, 3, 4
ROWMAP_NONE, ROWMAP_PAD, ROWMAP_UNPAD = 0, 1, 2


class GemmDesc(ctypes.Structure):
    _fields_ = [
        ("mode", ctypes.c_int32),
        ("m", ctypes.c_int32), ("n", ctypes.c_int32), ("k", ctypes.c_int32),
        ("a", ctypes.c_void_p), ("a_rows", ctypes.c_int64), ("a_ld", ctypes.c_int64),
        ("b", ctypes.c_void_p), ("b_rows", ctypes.c_int64), ("b_ld", ctypes.c_int64),
        ("ntaps", ctypes.c_int32), ("tap_w", ctypes.c_int32), ("tap_sign", ctypes.c_int32),
        ("split_k", ctypes.c_int32),
        ("scale", ctypes.c_void_p), ("shift", ctypes.c_void_p),
        ("residual", ctypes.c_void_p), ("res_ld", ctypes.c_int64),
        ("aux", ctypes.c_void_p), ("aux_ld", ctypes.c_int64), ("aux_mode", ctypes.c_int32),
        ("act", ctypes.c_int32),
        ("out", ctypes.c_void_p), ("out_ld", ctypes.c_int64), ("out_fp32", ctypes.c_int32),
        ("out2", ctypes.c_void_p), ("out2_ld", ctypes.c_int64),
        ("rowmap", ctypes.c_int32), ("map_h", ctypes.c_int32), ("map_w", ctypes.c_int32),
        ("dropout_p", ctypes.c_float), ("dropout_seed", ctypes.c_uint64),
        ("block_n", ctypes.c_int32), ("reserved", ctypes.c_int32),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_int64),
    ]


class NativeLibraryMissing(RuntimeError):
    pass


_lib = None


def lib():
    """Load (once) and return the shared library; raise loudly if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryMissing(
            "%s not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / eager fallback for the ClipBERT hot path)" % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    L.cb_last_error.restype = ctypes.c_char_p
    L.cb_version.restype = ctypes.c_int
    L.cb_sm_arch.restype = ctypes.c_int
    L.cb_launch_count.restype = ctypes.c_int64
    L.cb_gemm.argtypes = [ctypes.POINTER(GemmDesc), ctypes.c_void_p]
    L.cb_gemm.restype = ctypes.c_int
    L.cb_gemm_wgrad_group.argtypes = [ctypes.POINTER(GemmDesc), ctypes.c_int, ctypes.c_void_p]
    L.cb_gemm_wgrad_group.restype = ctypes.c_int
    L.cb_gemm_tile_width.argtypes = [ctypes.POINTER(GemmDesc)]
    L.cb_gemm_tile_width.restype = ctypes.c_int
    L.cb_gemm_workspace_bytes.argtypes = [ctypes.POINTER(GemmDesc)]
    L.cb_gemm_workspace_bytes.restype = ctypes.c_int64
    L.cb_gemm_wgrad_group_workspace_bytes.argtypes = [ctypes.POINTER(GemmDesc), ctypes.c_int]
    L.cb_gemm_wgrad_group_workspace_bytes.restype = ctypes.c_int64
    L.cb_set_deterministic.argtypes = [ctypes.c_int]
    L.cb_set_deterministic.restype = ctypes.c_int
    _lib = L
    return L


def check(rc, what="cb call"):
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, lib().cb_last_error().decode()))


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return None if t is None else t.data_ptr()
