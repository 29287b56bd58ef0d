"""ctypes binding of libtokenpacker_b200.so — the thin seam between the Python host code and the C-ABI CUDA library.

There is deliberately no fallback: if the shared library is missing the import fails loudly with the build command.
Signatures mirror include/tokenpacker_b200.h, include/tokenpacker_b200_hd_u8.h, include/tokenpacker_b200_clip_u8.h,
include/tokenpacker_b200_input_grad.h, include/tokenpacker_b200_layers.h, include/tokenpacker_b200_clip_tower.h,
include/tokenpacker_b200_clip_tower_f16.h, include/tokenpacker_b200_clip_tower_train.h, include/tokenpacker_b200_clip_tower_ckpt.h,
include/tokenpacker_b200_clip_tower_embed.h, include/tokenpacker_b200_clip_tower_crop_grad.h, include/tokenpacker_b200_clip_tower_interleaved.h,
include/tokenpacker_b200_jpeg.h and include/tokenpacker_b200_png.h one to one.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtokenpacker_b200.so")

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


class TpClipImage(C.Structure):
    """tp_clip_image (include/tokenpacker_b200_clip_u8.h): one row of the non-HD CLIP preprocessing plan."""
    _fields_ = [(n, C.c_int32) for n in ("h", "w", "canvas_h", "canvas_w", "pad_y", "pad_x", "resized_h", "resized_w", "top", "left",
                                         "ksize_x", "ksize_y")] + \
               [("coeff_x", C.c_int64), ("coeff_y", C.c_int64), ("row0", C.c_int32), ("rows", C.c_int32),
                ("workspace_offset", C.c_int64), ("workspace_row", C.c_int64)]


TP_CLIP_SQUARE = 0
TP_CLIP_PAD = 1


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

# the same for include/tokenpacker_b200_clip_u8.h (decoded 8-bit images into the non-HD CLIP input: pad / square)
CLIP_U8_SIGNATURES = {
    "tp_clip_preprocess_plan": (C.c_int, [C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int64, C.c_int, C.POINTER(TpClipImage),
                                          C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_size_t)]),
    "tp_clip_preprocess_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_size_t, C.c_void_p]),
}

# the same for include/tokenpacker_b200_input_grad.h (gradients w.r.t. the CLIP features in the training path)
INPUT_GRAD_SIGNATURES = {
    "tp_backward_inputs": (C.c_int, [C.POINTER(TpWeights), C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                     C.c_void_p, C.POINTER(TpWeights), C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
}

# the same for include/tokenpacker_b200_layers.h (training and packed HD output straight from the four CLIP hidden states)
LAYERS_SIGNATURES = {
    "tp_forward_train_layers": (C.c_int, [C.POINTER(TpWeights), C.c_void_p, C.POINTER(C.c_void_p), C.c_int64, C.c_int64, C.c_int, C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_backward_layers": (C.c_int, [C.POINTER(TpWeights), C.c_void_p, C.POINTER(C.c_void_p), C.c_int64, C.c_int64, C.c_int, C.c_int,
                                     C.c_void_p, C.c_void_p, C.POINTER(TpWeights), C.POINTER(C.c_void_p), C.c_int64, C.c_void_p,
                                     C.c_size_t, C.c_void_p]),
    "tp_forward_layers_packed": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                           C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
}

# the same for include/tokenpacker_b200_clip_tower.h (the frozen CLIP vision tower, forward only)
CLIP_TOWER_LAYERS = 23
CLIP_TOWER_LAYER_FIELDS = [
    # (struct field, parameter name inside encoder.layers.{i})
    ("ln1_w", "layer_norm1.weight"), ("ln1_b", "layer_norm1.bias"),
    ("q_w", "self_attn.q_proj.weight"), ("q_b", "self_attn.q_proj.bias"),
    ("k_w", "self_attn.k_proj.weight"), ("k_b", "self_attn.k_proj.bias"),
    ("v_w", "self_attn.v_proj.weight"), ("v_b", "self_attn.v_proj.bias"),
    ("o_w", "self_attn.out_proj.weight"), ("o_b", "self_attn.out_proj.bias"),
    ("ln2_w", "layer_norm2.weight"), ("ln2_b", "layer_norm2.bias"),
    ("fc1_w", "mlp.fc1.weight"), ("fc1_b", "mlp.fc1.bias"),
    ("fc2_w", "mlp.fc2.weight"), ("fc2_b", "mlp.fc2.bias"),
]
CLIP_TOWER_FIELDS = [
    ("patch_w", "embeddings.patch_embedding.weight"), ("class_emb", "embeddings.class_embedding"),
    ("pos_emb", "embeddings.position_embedding.weight"), ("pre_ln_w", "pre_layrnorm.weight"), ("pre_ln_b", "pre_layrnorm.bias"),
]


class TpClipTowerLayer(C.Structure):
    _fields_ = [(name, C.c_void_p) for name, _ in CLIP_TOWER_LAYER_FIELDS]


class TpClipTowerWeights(C.Structure):
    _fields_ = [(name, C.c_void_p) for name, _ in CLIP_TOWER_FIELDS] + [("layers", TpClipTowerLayer * CLIP_TOWER_LAYERS)]


CLIP_TOWER_SIGNATURES = {
    "tp_clip_tower_packed_bytes": (C.c_size_t, []),
    "tp_clip_tower_pack_weights": (C.c_int, [C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_clip_tower_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "tp_clip_tower_forward": (C.c_int, [C.c_void_p, C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int64, C.c_int64, C.POINTER(C.c_void_p),
                                        C.c_void_p, C.c_size_t, C.c_void_p]),
}

# the same for include/tokenpacker_b200_clip_tower_f16.h (the tower in fp16, as the evaluation and serving scripts run it)
TP_CLIP_CROPS_BF16 = 1
TP_CLIP_CROPS_F16 = 2
CLIP_TOWER_F16_SIGNATURES = {
    "tp_clip_tower_pack_weights_f16": (C.c_int, [C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_clip_tower_forward_f16": (C.c_int, [C.c_void_p, C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int, C.c_int64, C.c_int64,
                                            C.POINTER(C.c_void_p), C.c_void_p, C.c_size_t, C.c_void_p]),
}

# the same for include/tokenpacker_b200_clip_tower_interleaved.h (the four hidden states side by side in one [N, 577, 4096] buffer)
CLIP_TOWER_INTERLEAVED_SIGNATURES = {
    "tp_clip_tower_forward_interleaved": (C.c_int, [C.c_void_p, C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int64, C.c_int64, C.c_void_p,
                                                    C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_clip_tower_forward_interleaved_f16": (C.c_int, [C.c_void_p, C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int, C.c_int64, C.c_int64,
                                                        C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
}


# the same for include/tokenpacker_b200_clip_tower_train.h (training the last K layers of the tower)
class TpClipTowerLayerGrads(C.Structure):
    """tp_clip_tower_layer_grads: one gradient destination per parameter of a layer (None: not wanted)."""
    _fields_ = [(name, C.c_void_p) for name, _ in CLIP_TOWER_LAYER_FIELDS]


CLIP_TOWER_TRAIN_SIGNATURES = {
    "tp_clip_tower_train_saved_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "tp_clip_tower_train_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "tp_clip_tower_backward_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "tp_clip_tower_forward_train": (C.c_int, [C.c_void_p, C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                              C.POINTER(C.c_void_p), C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_clip_tower_backward": (C.c_int, [C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int64, C.c_int, C.POINTER(C.c_void_p),
                                         C.POINTER(TpClipTowerLayerGrads), C.c_void_p, C.c_size_t, C.c_void_p]),
}

# the same for include/tokenpacker_b200_clip_tower_ckpt.h (the trainable layers with gradient checkpointing)
CLIP_TOWER_CKPT_SIGNATURES = {
    "tp_clip_tower_ckpt_saved_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "tp_clip_tower_ckpt_backward_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "tp_clip_tower_forward_ckpt": (C.c_int, [C.c_void_p, C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                             C.POINTER(C.c_void_p), C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_clip_tower_backward_ckpt": (C.c_int, [C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int64, C.c_int, C.POINTER(C.c_void_p),
                                              C.POINTER(TpClipTowerLayerGrads), C.c_void_p, C.c_size_t, C.c_void_p]),
}


# the same for include/tokenpacker_b200_clip_tower_embed.h (the whole tower: 23 layers and the embedding stage below them)
class TpClipTowerEmbedGrads(C.Structure):
    """tp_clip_tower_embed_grads: one gradient destination per CLIP_TOWER_FIELDS parameter (None: not wanted)."""
    _fields_ = [(name, C.c_void_p) for name, _ in CLIP_TOWER_FIELDS]


CLIP_TOWER_EMBED_SIGNATURES = {
    "tp_clip_tower_embed_saved_bytes": (C.c_size_t, [C.c_int64]),
    "tp_clip_tower_forward_train_embed": (C.c_int, [C.c_void_p, C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                                    C.POINTER(C.c_void_p), C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                                    C.c_size_t, C.c_void_p]),
    "tp_clip_tower_backward_embed": (C.c_int, [C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_void_p, C.c_int64, C.c_int,
                                               C.POINTER(C.c_void_p), C.POINTER(TpClipTowerLayerGrads), C.POINTER(TpClipTowerEmbedGrads),
                                               C.c_void_p, C.c_size_t, C.c_void_p]),
}


# the same for include/tokenpacker_b200_clip_tower_crop_grad.h (gradients to the crops and through the HD tiling to the images)
TP_CROP_GRAD_BF16 = 0
TP_CROP_GRAD_F32 = 1


class TpHdImageGrad(C.Structure):
    """tp_hd_image_grad: where tp_hd_tile_batch_backward writes one image's gradient, and where its inverse-tap tables are."""
    _fields_ = [("d_image", C.c_void_p), ("row_taps", C.c_int64), ("col_taps", C.c_int64), ("thumb_row_taps", C.c_int64),
                ("thumb_col_taps", C.c_int64)]


CROP_GRAD_SIGNATURES = {
    "tp_clip_tower_backward_crops": (C.c_int, [C.POINTER(TpClipTowerWeights), C.c_void_p, C.c_void_p, C.c_int64, C.c_int,
                                               C.POINTER(C.c_void_p), C.POINTER(TpClipTowerLayerGrads), C.POINTER(TpClipTowerEmbedGrads),
                                               C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    "tp_hd_tile_batch_backward_plan": (C.c_int, [C.POINTER(TpHdImage), C.c_int64, C.POINTER(C.c_void_p), C.POINTER(TpHdImageGrad),
                                                 C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "tp_hd_tile_batch_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
}


# the same for include/tokenpacker_b200_jpeg.h (baseline JPEG files decoded on the GPU, bit for bit as PIL)
class TpJpegImage(C.Structure):
    """tp_jpeg_image: one row of the decode plan."""
    _fields_ = [(n, C.c_int32) for n in ("reason", "h", "w", "ncomp", "hs", "vs", "mcus_x", "mcus_y", "blocks_per_mcu", "restart",
                                         "n_segments")] + \
               [("comp_bx", C.c_int32 * 3), ("comp_by", C.c_int32 * 3), ("reserved", C.c_int32)] + \
               [(n, C.c_int64) for n in ("scan_offset", "scan_bytes", "unstuffed_offset", "seg_offset", "sub_offset", "sub_capacity",
                                         "coef_offset", "n_blocks", "block0", "plane_offset", "out_offset", "pixel0")]


class TpJpegHuff(C.Structure):
    _fields_ = [("lookup", C.c_uint16 * 512), ("maxcode", C.c_int32 * 18), ("valoff", C.c_int32 * 18), ("values", C.c_uint8 * 256)]


class TpJpegTables(C.Structure):
    _fields_ = [("dc", TpJpegHuff * 3), ("ac", TpJpegHuff * 3), ("quant", (C.c_uint16 * 64) * 3)]


class TpJpegTotals(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("staged_bytes", "output_bytes", "workspace_bytes", "blocks", "pixels")]


class TpJpegStatus(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("status", "sync_rounds", "subsequences", "reserved")]


TP_JPEG_SUPPORTED = 0
TP_JPEG_STATUS_OK, TP_JPEG_STATUS_ENTROPY, TP_JPEG_STATUS_RESTART = 0, 1, 2
JPEG_SIGNATURES = {
    "tp_jpeg_plan": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int64, C.POINTER(TpJpegImage), C.c_void_p, C.c_void_p,
                               C.POINTER(TpJpegTotals)]),
    "tp_jpeg_workspace_bytes": (C.c_size_t, [C.POINTER(TpJpegImage), C.c_int64]),
    "tp_jpeg_reason_string": (C.c_char_p, [C.c_int]),
    "tp_jpeg_decode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t,
                                       C.c_void_p, C.c_void_p]),
}


# the same for include/tokenpacker_b200_png.h (PNG files decoded on the GPU, byte for byte as PIL)
class TpPngImage(C.Structure):
    """tp_png_image: one row of the decode plan."""
    _fields_ = [(n, C.c_int32) for n in ("reason", "h", "w", "depth", "color_type", "channels", "row_bytes", "filter_bpp",
                                         "palette_entries", "window")] + \
               [(n, C.c_int64) for n in ("palette_offset", "stream_offset", "stream_bytes", "raw_bytes", "block_capacity", "mask_offset",
                                         "spec_offset", "block_offset", "raw_offset", "src_offset", "out_offset", "pixel0")]


class TpPngBlock(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("start_bit", "end_bit", "out_offset", "out_bytes", "flags")]


class TpPngTotals(C.Structure):
    _fields_ = [(n, C.c_int64) for n in ("staged_bytes", "output_bytes", "workspace_bytes", "max_raw_bytes", "pixels")]


class TpPngStatus(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("status", "blocks", "serial_blocks", "candidates")]


TP_PNG_SUPPORTED = 0
TP_PNG_PALETTE_BYTES = 768
TP_PNG_SPAN_BITS, TP_PNG_SLOTS, TP_PNG_MIN_BLOCK_BITS = 256, 4, 10
(TP_PNG_STATUS_OK, TP_PNG_STATUS_BLOCK_TYPE, TP_PNG_STATUS_CODE_LENGTHS, TP_PNG_STATUS_SYMBOL, TP_PNG_STATUS_DISTANCE,
 TP_PNG_STATUS_STORED, TP_PNG_STATUS_TRUNCATED, TP_PNG_STATUS_DATA_SIZE, TP_PNG_STATUS_ADLER, TP_PNG_STATUS_FILTER) = range(10)
PNG_SIGNATURES = {
    "tp_png_plan": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int64, C.POINTER(TpPngImage), C.c_void_p, C.c_void_p,
                              C.POINTER(TpPngTotals)]),
    "tp_png_workspace_bytes": (C.c_size_t, [C.POINTER(TpPngImage), C.c_int64]),
    "tp_png_reason_string": (C.c_char_p, [C.c_int]),
    "tp_png_decode_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_size_t,
                                      C.c_void_p, C.c_void_p]),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"tokenpacker_b200: {LIB_PATH} is missing. Build it with `make -C tokenpacker_b200/csrc` "
            "(or `python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in {**SIGNATURES, **HD_U8_SIGNATURES, **CLIP_U8_SIGNATURES, **INPUT_GRAD_SIGNATURES,
                                      **LAYERS_SIGNATURES, **CLIP_TOWER_SIGNATURES, **CLIP_TOWER_F16_SIGNATURES, **CLIP_TOWER_INTERLEAVED_SIGNATURES,
                                      **CLIP_TOWER_TRAIN_SIGNATURES, **CLIP_TOWER_CKPT_SIGNATURES,
                                      **CLIP_TOWER_EMBED_SIGNATURES, **CROP_GRAD_SIGNATURES, **JPEG_SIGNATURES, **PNG_SIGNATURES}.items():
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
