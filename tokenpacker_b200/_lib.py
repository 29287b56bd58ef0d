"""ctypes binding of libtokenpacker_b200.so — the thin seam between the Python host code and the C-ABI CUDA library.

There is deliberately no fallback: if the shared library is missing the import fails loudly with the build command.
Signatures mirror include/tokenpacker_b200.h, include/tokenpacker_b200_hd_u8.h and include/tokenpacker_b200_input_grad.h one to one.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# TOKENPACKER_B200_LIB_OVERRIDE: load another BUILD of the same library (A/B experiments with -D variants); it must export
# every symbol of the header like the default one.  Unset in normal use.
LIB_PATH = os.environ.get("TOKENPACKER_B200_LIB_OVERRIDE") or os.path.join(_HERE, "libtokenpacker_b200.so")

TP_OK = 0
TP_ERR_INVALID_ARGUMENT = 1
TP_ERR_BAD_SCALE_FACTOR = 2
TP_ERR_WORKSPACE_TOO_SMALL = 3
TP_ERR_CUDA = 4
TP_ERR_UNSUPPORTED_DEVICE = 5
TP_ERR_BAD_PATCH_NUM = 6

WEIGHT_FIELDS = [
    # (struct field, reference state_dict key)            builder.py:59-83
    ("q_proj_w", "q_proj_1.weight"),
    ("k_proj_0_w", "k_proj_1.0.weight"), ("k_proj_0_b", "k_proj_1.0.bias"),
    ("k_proj_2_w", "k_proj_1.2.weight"), ("k_proj_2_b", "k_proj_1.2.bias"),
    ("v_proj_0_w", "v_proj_1.0.weight"), ("v_proj_0_b", "v_proj_1.0.bias"),
    ("v_proj_2_w", "v_proj_1.2.weight"), ("v_proj_2_b", "v_proj_1.2.bias"),
    ("ln_q_w", "ln_q_1.weight"), ("ln_q_b", "ln_q_1.bias"),
    ("ln_k_w", "ln_k_1.weight"), ("ln_k_b", "ln_k_1.bias"),
    ("ln_v_w", "ln_v_1.weight"), ("ln_v_b", "ln_v_1.bias"),
    ("in_proj_w", "clip_attn.in_proj_weight"), ("in_proj_b", "clip_attn.in_proj_bias"),
    ("out_proj_w", "clip_attn.out_proj.weight"), ("out_proj_b", "clip_attn.out_proj.bias"),
    ("mlp_0_w", "mlp.0.weight"), ("mlp_0_b", "mlp.0.bias"),
    ("mlp_2_w", "mlp.2.weight"), ("mlp_2_b", "mlp.2.bias"),
]


class TpWeights(C.Structure):
    _fields_ = [(name, C.c_void_p) for name, _ in WEIGHT_FIELDS]


class TpHdImage(C.Structure):
    """tp_hd_image: one row of the batched tiling plan."""
    _fields_ = [("image", C.c_void_p), ("h", C.c_int32), ("w", C.c_int32), ("hb", C.c_int32), ("wb", C.c_int32),
                ("h_r", C.c_int32), ("w_r", C.c_int32), ("h_t", C.c_int32), ("w_t", C.c_int32), ("crop0", C.c_int64),
                ("sy", C.c_float), ("sx", C.c_float), ("ty", C.c_float), ("tx", C.c_float)]


class TpHdU8Source(C.Structure):
    """tp_hd_u8_source (include/tokenpacker_b200_hd_u8.h): where one decoded 8-bit image lies (element strides of channel, row
    and column)."""
    _fields_ = [("pixels", C.c_void_p), ("stride_c", C.c_int64), ("stride_y", C.c_int64), ("stride_x", C.c_int64)]


# name -> (restype, argtypes); kept as data so tests can check the header and the binding agree
SIGNATURES = {
    "tp_strerror": (C.c_char_p, [C.c_int]),
    "tp_abi_version": (C.c_int, []),
    "tp_last_cuda_error": (C.c_char_p, []),
    "tp_launch_count": (C.c_uint64, []),
    "tp_packed_bytes": (C.c_size_t, [C.c_int]),
    "tp_pack_weights": (C.c_int, [C.POINTER(TpWeights), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int]),
    "tp_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int,
                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_forward_packed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                    C.c_void_p, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_forward_layers": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_forward_allgather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                       C.POINTER(C.c_void_p), C.c_int, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_forward_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, C.c_void_p]),
    "tp_train_saved_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int]),
    "tp_backward_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int]),
    "tp_pack_weights_train": (C.c_int, [C.POINTER(TpWeights), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_forward_train": (C.c_int, [C.POINTER(TpWeights), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                   C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_backward": (C.c_int, [C.POINTER(TpWeights), C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                              C.POINTER(TpWeights), C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_gemm_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                               C.c_int64, C.c_void_p, C.c_int, C.c_float, C.c_void_p]),
    "tp_gemm_tn_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                  C.c_float, C.c_void_p]),
    "tp_gemm_nn_bf16": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                  C.c_float, C.c_void_p]),
    "tp_hd_grid": (C.c_int, [C.c_int64, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tp_hd_fit": (C.c_int, [C.c_int64, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                            C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tp_hd_tile": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "tp_hd_tile_batch_plan": (C.c_int, [C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_void_p), C.c_int64, C.c_int,
                                        C.POINTER(TpHdImage), C.POINTER(C.c_int32), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                        C.POINTER(C.c_int64)]),
    "tp_hd_tile_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tp_hd_plan": (C.c_int, [C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int64, C.c_int, C.POINTER(C.c_int64),
                             C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                             C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "tp_hd_scatter_crops": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tp_gather_rows": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "tp_hd_fill_separators": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64,
                                        C.c_void_p, C.c_void_p]),
}

# the same for include/tokenpacker_b200_hd_u8.h (decoded 8-bit images into the batched HD front end)
HD_U8_SIGNATURES = {
    "tp_hd_preprocess_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
}

# the same for include/tokenpacker_b200_input_grad.h (gradients w.r.t. the CLIP features in the training path)
INPUT_GRAD_SIGNATURES = {
    "tp_backward_inputs": (C.c_int, [C.POINTER(TpWeights), C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                     C.c_void_p, C.POINTER(TpWeights), C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"tokenpacker_b200: {LIB_PATH} is missing. Build it with `make -C tokenpacker_b200/csrc` "
            "(or `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in {**SIGNATURES, **HD_U8_SIGNATURES, **INPUT_GRAD_SIGNATURES}.items():
        fn = getattr(lib, name)          # AttributeError here = ABI mismatch: fail loudly
        fn.restype = restype
        fn.argtypes = argtypes
    return lib


lib = _load()


class TokenPackerError(RuntimeError):
    def __init__(self, status: int, where: str):
        detail = lib.tp_last_cuda_error().decode() if status == TP_ERR_CUDA else ""
        super().__init__(f"{where}: {lib.tp_strerror(status).decode()}" + (f" [{detail}]" if detail else ""))
        self.status = status


def check(status: int, where: str):
    if status == TP_OK:
        return
    if status == TP_ERR_BAD_SCALE_FACTOR:
        raise ValueError(lib.tp_strerror(status).decode())      # same exception type and message as builder.py:51-52
    if status == TP_ERR_BAD_PATCH_NUM:
        raise NotImplementedError(lib.tp_strerror(status).decode())   # patch_divide.py:79-80
    raise TokenPackerError(status, where)
