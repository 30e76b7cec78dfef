"""ctypes view of the clip.cpp C ABI (clip.h:8-113 in the reference).

The same `ClipLib` class drives either shared library, because the product keeps the reference's
22 exported symbols and struct layouts byte for byte:

  * `libclip_b200.so`        -- the H100-native product (this repository)
  * the unmodified reference built under oracle/ (path: oracle/ref_run.py REF_LIB) -- tests / bench use it as the checker

It mirrors the shape of the reference's own Python binding
(/root/reference/examples/python_bindings/clip_cpp/clip.py:36-208) but carries the `size` members of
clip_image_u8 / clip_image_f32 that the upstream binding forgot (clip.h:50-64).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np


class clip_text_hparams(C.Structure):
    _fields_ = [("n_vocab", C.c_int32), ("num_positions", C.c_int32), ("hidden_size", C.c_int32),
                ("n_intermediate", C.c_int32), ("projection_dim", C.c_int32), ("n_head", C.c_int32),
                ("n_layer", C.c_int32), ("eps", C.c_float)]


class clip_vision_hparams(C.Structure):
    _fields_ = [("image_size", C.c_int32), ("patch_size", C.c_int32), ("hidden_size", C.c_int32),
                ("n_intermediate", C.c_int32), ("projection_dim", C.c_int32), ("n_head", C.c_int32),
                ("n_layer", C.c_int32), ("eps", C.c_float)]


class clip_tokens(C.Structure):
    _fields_ = [("data", C.POINTER(C.c_int32)), ("size", C.c_size_t)]


class clip_image_u8(C.Structure):
    _fields_ = [("nx", C.c_int), ("ny", C.c_int), ("data", C.POINTER(C.c_uint8)), ("size", C.c_size_t)]


class clip_image_f32(C.Structure):
    _fields_ = [("nx", C.c_int), ("ny", C.c_int), ("data", C.POINTER(C.c_float)), ("size", C.c_size_t)]


class clip_image_u8_batch(C.Structure):
    _fields_ = [("data", C.POINTER(clip_image_u8)), ("size", C.c_size_t)]


class clip_image_f32_batch(C.Structure):
    _fields_ = [("data", C.POINTER(clip_image_f32)), ("size", C.c_size_t)]


REFERENCE_SYMBOLS = [
    "clip_model_load", "clip_free", "clip_get_text_hparams", "clip_get_vision_hparams", "clip_tokenize",
    "clip_image_u8_make", "clip_image_f32_make", "clip_image_u8_clean", "clip_image_f32_clean",
    "clip_image_u8_free", "clip_image_f32_free", "clip_image_load_from_file", "clip_image_preprocess",
    "clip_text_encode", "clip_image_encode", "clip_image_batch_preprocess", "clip_image_batch_encode",
    "clip_compare_text_and_image", "clip_similarity_score", "softmax_with_sorting",
    "clip_zero_shot_label_image", "clip_model_quantize",
]

# additive entry points of this library (include/clip_b200.h); absent from the reference library
EXTENSION_SYMBOLS = [
    "clip_text_batch_encode", "clip_b200_image_encode_device", "clip_b200_text_encode_device",
    "clip_b200_zero_shot_batch", "clip_b200_device_malloc", "clip_b200_device_free",
    "clip_b200_host_malloc", "clip_b200_host_free", "clip_b200_memcpy_h2d", "clip_b200_memcpy_d2h",
    "clip_b200_synchronize", "clip_b200_last_error", "clip_b200_kernel_launches",
    "clip_b200_last_device_ms", "clip_b200_version", "clip_b200_set_micro_batch",
    "clip_b200_debug_gemm", "clip_b200_debug_gemm_scaled", "clip_b200_debug_attention", "clip_b200_debug_attention_hd", "clip_b200_image_batch_encode_u8",
    "clip_b200_image_batch_preprocess_device", "clip_b200_get_stream", "clip_b200_kernel_ms",
    "clip_b200_debug_repack_roundtrip", "clip_b200_debug_tokenize", "clip_b200_debug_preprocess",
    "clip_b200_mark", "clip_b200_mark_elapsed_ms",
    # scoring + multi-GPU (round 2)
    "clip_b200_topk_search", "clip_b200_rows_to_16bit", "clip_b200_topk_search_16", "clip_b200_rows_to_int8", "clip_b200_topk_search_i8",
    "clip_b200_rows_to_binary", "clip_b200_topk_search_b1", "clip_b200_topk_rescore",
    "clip_b200_zero_shot_images", "clip_b200_dist_unique_id", "clip_b200_dist_init_with_id",
    "clip_b200_dist_init", "clip_b200_dist_rank", "clip_b200_dist_world", "clip_b200_device_count", "clip_b200_nccl_version", "clip_b200_cuda_device_count",
    "clip_b200_dist_barrier", "clip_b200_dist_max_f64", "clip_b200_dist_all_gather", "clip_b200_image_encode_device_all",
    "clip_b200_text_encode_device_all", "clip_b200_image_batch_encode_all", "clip_b200_text_batch_encode_all",
    "clip_b200_debug_rendezvous", "clip_b200_debug_shard_bounds",
    # row-kernel test hooks
    "clip_b200_debug_layernorm", "clip_b200_debug_assemble_preln", "clip_b200_debug_im2col", "clip_b200_debug_text_embed",
    "clip_b200_debug_gather_rows", "clip_b200_debug_l2norm", "clip_b200_debug_fill_last",
    # per-token hidden states
    "clip_b200_image_tokens", "clip_b200_image_tokens_device", "clip_b200_text_tokens", "clip_b200_text_tokens_device",
    "clip_b200_debug_token_rows",
    # any patch-multiple image size (interpolated position table)
    "clip_b200_image_encode_device_hw", "clip_b200_image_tokens_device_hw", "clip_b200_image_batch_encode_hw", "clip_b200_image_tokens_hw",
    "clip_b200_debug_im2col_hw", "clip_b200_debug_pos_resample",
    # several layers' token rows from one forward pass
    "clip_b200_image_tokens_layers", "clip_b200_image_tokens_layers_device", "clip_b200_text_tokens_layers",
    "clip_b200_text_tokens_layers_device",
    # attention probabilities (TOKENS_ATTENTION entries)
    "clip_b200_debug_attention_probs",
    # head_dim 104 (ViT-bigG/14): the loader's QKV row padding
    "clip_b200_debug_pad_qkv",
    # images of different sizes in one call (variable-length attention)
    "clip_b200_image_batch_encode_mixed", "clip_b200_image_encode_device_mixed", "clip_b200_image_tokens_mixed",
    "clip_b200_image_tokens_device_mixed", "clip_b200_debug_attention_mixed",
    # token sequences of different lengths in one call (causal variable-length attention)
    "clip_b200_text_batch_encode_packed", "clip_b200_text_encode_device_packed", "clip_b200_text_tokens_packed",
    "clip_b200_text_tokens_device_packed", "clip_b200_debug_attention_mixed_causal",
    # inverted-file index over 16-bit databases
    "clip_b200_ivf_train_16", "clip_b200_ivf_build_16", "clip_b200_ivf_search_16",
    "clip_b200_ivfpq_train_16", "clip_b200_ivfpq_encode_16", "clip_b200_ivfpq_build", "clip_b200_ivfpq_search_16",
]

# include/clip_b200.h: output types and flags of the *_tokens entry points
OUT_F32, OUT_F16, OUT_BF16 = 0, 1, 2
OUT_DTYPES = {OUT_F32: np.float32, OUT_F16: np.float16, OUT_BF16: np.uint16}      # bf16 comes back as its raw 16-bit pattern
TOKENS_POST_LN, TOKENS_PROJECT, TOKENS_NORMALIZE, TOKENS_NO_CLS = 1, 2, 4, 8
TOKENS_ATTENTION, TOKENS_ATTENTION_CLS = 32, 64      # bit 16 stays unassigned


def slab_offsets(nbytes, flags):
    """byte offsets of the slabs of a *_tokens_layers output: slab j follows slab j - 1, except that the slab after an ATTENTION
    slab starts at the next multiple of 16 bytes.  nbytes[j]: slab j's size, flags[j]: its flags."""
    offs, o = [], 0
    for b, f in zip(nbytes, flags):
        offs.append(o)
        o += b
        if f & TOKENS_ATTENTION:
            o = (o + 15) // 16 * 16
    return offs

HERE = os.path.dirname(os.path.abspath(__file__))
PRODUCT_LIB = os.environ.get("CLIP_B200_LIB") or os.path.join(HERE, "libclip_b200.so")     # CLIP_B200_LIB: experiment builds only


class ClipLib:
    """Thin, explicit ctypes wrapper. `path` picks the implementation."""

    def __init__(self, path: str = PRODUCT_LIB):
        if not os.path.exists(path):
            raise FileNotFoundError(
                "%s not built -- run `python -c 'import __graft_entry__ as g; g.build()'`" % path)
        self.path = path
        self.lib = L = C.CDLL(path, mode=os.RTLD_LOCAL | os.RTLD_NOW)
        self.is_product = hasattr(L, "clip_b200_version")
        vp, ip, fp = C.c_void_p, C.c_int, C.POINTER(C.c_float)
        L.clip_model_load.restype = vp
        L.clip_model_load.argtypes = [C.c_char_p, ip]
        L.clip_free.argtypes = [vp]
        L.clip_free.restype = None
        L.clip_get_text_hparams.restype = C.POINTER(clip_text_hparams)
        L.clip_get_text_hparams.argtypes = [vp]
        L.clip_get_vision_hparams.restype = C.POINTER(clip_vision_hparams)
        L.clip_get_vision_hparams.argtypes = [vp]
        L.clip_tokenize.restype = C.c_bool
        L.clip_tokenize.argtypes = [vp, C.c_char_p, C.POINTER(clip_tokens)]
        L.clip_image_preprocess.restype = C.c_bool
        L.clip_image_preprocess.argtypes = [vp, C.POINTER(clip_image_u8), C.POINTER(clip_image_f32)]
        L.clip_image_batch_preprocess.restype = None
        L.clip_image_batch_preprocess.argtypes = [vp, ip, C.POINTER(clip_image_u8_batch),
                                                  C.POINTER(clip_image_f32_batch)]
        L.clip_image_f32_clean.argtypes = [C.POINTER(clip_image_f32)]
        L.clip_image_f32_clean.restype = None
        L.clip_text_encode.restype = C.c_bool
        L.clip_text_encode.argtypes = [vp, ip, C.POINTER(clip_tokens), fp, C.c_bool]
        L.clip_image_encode.restype = C.c_bool
        L.clip_image_encode.argtypes = [vp, ip, C.POINTER(clip_image_f32), fp, C.c_bool]
        L.clip_image_batch_encode.restype = C.c_bool
        L.clip_image_batch_encode.argtypes = [vp, ip, C.POINTER(clip_image_f32_batch), fp, C.c_bool]
        L.clip_compare_text_and_image.restype = C.c_bool
        L.clip_compare_text_and_image.argtypes = [vp, ip, C.c_char_p, C.POINTER(clip_image_u8), fp]
        L.clip_similarity_score.restype = C.c_float
        L.clip_similarity_score.argtypes = [fp, fp, ip]
        L.softmax_with_sorting.restype = C.c_bool
        L.softmax_with_sorting.argtypes = [fp, ip, fp, C.POINTER(C.c_int)]
        L.clip_zero_shot_label_image.restype = C.c_bool
        L.clip_zero_shot_label_image.argtypes = [vp, ip, C.POINTER(clip_image_u8), C.POINTER(C.c_char_p),
                                                 C.c_size_t, fp, C.POINTER(C.c_int)]
        L.clip_model_quantize.restype = C.c_bool
        L.clip_model_quantize.argtypes = [C.c_char_p, C.c_char_p, ip]
        if self.is_product:
            L.clip_b200_version.restype = C.c_char_p
            L.clip_b200_last_error.restype = C.c_char_p
            L.clip_text_batch_encode.restype = C.c_bool
            L.clip_text_batch_encode.argtypes = [vp, ip, C.POINTER(clip_tokens), C.c_size_t, fp, C.c_bool]
            L.clip_b200_image_encode_device.restype = C.c_bool
            L.clip_b200_image_encode_device.argtypes = [vp, vp, C.c_size_t, vp, C.c_bool]
            L.clip_b200_text_encode_device.restype = C.c_bool
            L.clip_b200_text_encode_device.argtypes = [vp, vp, vp, C.c_size_t, ip, vp, C.c_bool]
            L.clip_b200_zero_shot_batch.restype = C.c_bool
            L.clip_b200_zero_shot_batch.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, fp, C.POINTER(C.c_int), ip]
            L.clip_b200_device_malloc.restype = vp
            L.clip_b200_device_malloc.argtypes = [vp, C.c_size_t]
            L.clip_b200_device_free.argtypes = [vp, vp]
            L.clip_b200_device_free.restype = None
            L.clip_b200_host_malloc.restype = vp
            L.clip_b200_host_malloc.argtypes = [C.c_size_t]
            L.clip_b200_host_free.argtypes = [vp]
            L.clip_b200_host_free.restype = None
            L.clip_b200_memcpy_h2d.restype = C.c_bool
            L.clip_b200_memcpy_h2d.argtypes = [vp, vp, vp, C.c_size_t]
            L.clip_b200_memcpy_d2h.restype = C.c_bool
            L.clip_b200_memcpy_d2h.argtypes = [vp, vp, vp, C.c_size_t]
            L.clip_b200_synchronize.restype = C.c_bool
            L.clip_b200_synchronize.argtypes = [vp]
            L.clip_b200_kernel_launches.restype = C.c_uint64
            L.clip_b200_kernel_launches.argtypes = [vp]
            L.clip_b200_last_device_ms.restype = C.c_float
            L.clip_b200_last_device_ms.argtypes = [vp]
            L.clip_b200_set_micro_batch.restype = None
            L.clip_b200_set_micro_batch.argtypes = [vp, ip, ip]
            L.clip_b200_get_stream.restype = vp
            L.clip_b200_get_stream.argtypes = [vp]
            L.clip_b200_kernel_ms.restype = C.c_float
            L.clip_b200_kernel_ms.argtypes = [vp, ip, C.POINTER(C.c_uint64)]
            L.clip_b200_mark.restype = C.c_bool
            L.clip_b200_mark.argtypes = [vp, ip]
            L.clip_b200_mark_elapsed_ms.restype = C.c_float
            L.clip_b200_mark_elapsed_ms.argtypes = [vp, ip, ip]
            L.clip_b200_debug_repack_roundtrip.restype = C.c_int
            L.clip_b200_debug_repack_roundtrip.argtypes = [ip, vp, ip, ip]
            L.clip_b200_debug_tokenize.restype = C.c_int
            L.clip_b200_debug_tokenize.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(C.c_int32), ip]
            L.clip_b200_debug_preprocess.restype = C.c_int
            L.clip_b200_debug_preprocess.argtypes = [C.POINTER(C.c_uint8), ip, ip, ip, fp, fp, fp]
            L.clip_b200_image_batch_encode_u8.restype = C.c_bool
            L.clip_b200_image_batch_encode_u8.argtypes = [vp, C.POINTER(clip_image_u8_batch), fp, C.c_bool]
            L.clip_b200_image_batch_preprocess_device.restype = C.c_bool
            L.clip_b200_image_batch_preprocess_device.argtypes = [vp, C.POINTER(clip_image_u8_batch), C.POINTER(clip_image_f32_batch)]
            L.clip_b200_debug_attention.restype = C.c_int
            L.clip_b200_debug_attention.argtypes = [ip, ip, ip, ip, ip, ip, fp, fp, C.POINTER(C.c_float)]
            L.clip_b200_debug_attention_hd.restype = C.c_int
            L.clip_b200_debug_attention_hd.argtypes = [ip, ip, ip, ip, ip, ip, ip, fp, fp, C.POINTER(C.c_float)]
            L.clip_b200_debug_attention_mixed.restype = C.c_int
            L.clip_b200_debug_attention_mixed.argtypes = [ip, ip, C.POINTER(C.c_int), ip, ip, fp, fp]
            L.clip_b200_debug_attention_mixed_causal.restype = C.c_int
            L.clip_b200_debug_attention_mixed_causal.argtypes = [ip, ip, C.POINTER(C.c_int), ip, ip, fp, fp]
            L.clip_b200_debug_attention_probs.restype = C.c_int
            L.clip_b200_debug_attention_probs.argtypes = [ip, ip, ip, ip, ip, ip, ip, ip, fp, vp]
            L.clip_b200_debug_gemm.restype = C.c_int
            L.clip_b200_debug_gemm.argtypes = [ip, ip, ip, ip, ip, ip, ip, fp, vp, fp, fp, fp, C.POINTER(C.c_float)]
            L.clip_b200_debug_gemm_scaled.restype = C.c_int
            L.clip_b200_debug_gemm_scaled.argtypes = [ip, ip, ip, ip, ip, ip, ip, C.c_float, fp, vp, fp, fp, fp, C.POINTER(C.c_float)]
            i32p = C.POINTER(C.c_int32)
            for f, args in (("clip_b200_debug_layernorm", [ip, ip, C.c_size_t, C.c_float, fp, fp, fp, fp, ip, fp, fp]),
                            ("clip_b200_debug_assemble_preln", [fp, fp, fp, ip, ip, ip, C.c_float, fp, fp, fp]),
                            ("clip_b200_debug_im2col", [fp, ip, ip, ip, ip, fp]),
                            ("clip_b200_debug_text_embed", [i32p, fp, fp, ip, ip, ip, ip, fp]),
                            ("clip_b200_debug_gather_rows", [fp, ip, ip, ip, ip, i32p, fp, ip, fp]),
                            ("clip_b200_debug_l2norm", [fp, ip, ip, ip, fp]),
                            ("clip_b200_debug_fill_last", [i32p, ip, ip, i32p]),
                            ("clip_b200_debug_token_rows", [ip, ip, ip, C.c_size_t, ip, C.c_float, fp, fp, fp, ip, vp]),
                            ("clip_b200_debug_im2col_hw", [fp, ip, ip, ip, ip, ip, fp]),
                            ("clip_b200_debug_pos_resample", [fp, ip, ip, ip, ip, fp])):
                getattr(L, f).restype = C.c_int
                getattr(L, f).argtypes = args
            L.clip_b200_image_tokens.restype = C.c_bool
            L.clip_b200_image_tokens.argtypes = [vp, C.POINTER(clip_image_f32_batch), ip, ip, ip, vp]
            L.clip_b200_image_tokens_device.restype = C.c_bool
            L.clip_b200_image_tokens_device.argtypes = [vp, vp, C.c_size_t, ip, ip, ip, vp]
            L.clip_b200_text_tokens.restype = C.c_bool
            L.clip_b200_text_tokens.argtypes = [vp, i32p, C.c_size_t, ip, ip, ip, ip, vp]
            L.clip_b200_text_tokens_device.restype = C.c_bool
            L.clip_b200_text_tokens_device.argtypes = [vp, vp, C.c_size_t, ip, ip, ip, ip, vp]
            L.clip_b200_image_encode_device_hw.restype = C.c_bool
            L.clip_b200_image_encode_device_hw.argtypes = [vp, vp, C.c_size_t, ip, ip, vp, C.c_bool]
            L.clip_b200_image_tokens_device_hw.restype = C.c_bool
            L.clip_b200_image_tokens_device_hw.argtypes = [vp, vp, C.c_size_t, ip, ip, ip, ip, ip, vp]
            L.clip_b200_image_batch_encode_hw.restype = C.c_bool
            L.clip_b200_image_batch_encode_hw.argtypes = [vp, C.POINTER(clip_image_f32_batch), fp, C.c_bool]
            L.clip_b200_image_tokens_hw.restype = C.c_bool
            L.clip_b200_image_tokens_hw.argtypes = [vp, C.POINTER(clip_image_f32_batch), ip, ip, ip, vp]
            intp = C.POINTER(C.c_int)
            L.clip_b200_image_batch_encode_mixed.restype = C.c_bool
            L.clip_b200_image_batch_encode_mixed.argtypes = [vp, C.POINTER(clip_image_f32_batch), fp, C.c_bool]
            L.clip_b200_image_encode_device_mixed.restype = C.c_bool
            L.clip_b200_image_encode_device_mixed.argtypes = [vp, vp, C.c_size_t, intp, intp, vp, C.c_bool]
            L.clip_b200_image_tokens_mixed.restype = C.c_bool
            L.clip_b200_image_tokens_mixed.argtypes = [vp, C.POINTER(clip_image_f32_batch), ip, ip, ip, vp]
            L.clip_b200_image_tokens_device_mixed.restype = C.c_bool
            L.clip_b200_image_tokens_device_mixed.argtypes = [vp, vp, C.c_size_t, intp, intp, ip, ip, ip, vp]
            L.clip_b200_text_batch_encode_packed.restype = C.c_bool
            L.clip_b200_text_batch_encode_packed.argtypes = [vp, C.POINTER(clip_tokens), C.c_size_t, fp, C.c_bool]
            L.clip_b200_text_encode_device_packed.restype = C.c_bool
            L.clip_b200_text_encode_device_packed.argtypes = [vp, vp, C.c_size_t, intp, vp, C.c_bool]
            L.clip_b200_text_tokens_packed.restype = C.c_bool
            L.clip_b200_text_tokens_packed.argtypes = [vp, C.POINTER(C.c_int32), C.c_size_t, intp, ip, ip, ip, vp]
            L.clip_b200_text_tokens_device_packed.restype = C.c_bool
            L.clip_b200_text_tokens_device_packed.argtypes = [vp, vp, C.c_size_t, intp, ip, ip, ip, vp]
            L.clip_b200_image_tokens_layers.restype = C.c_bool
            L.clip_b200_image_tokens_layers.argtypes = [vp, C.POINTER(clip_image_f32_batch), intp, intp, ip, ip, vp]
            L.clip_b200_image_tokens_layers_device.restype = C.c_bool
            L.clip_b200_image_tokens_layers_device.argtypes = [vp, vp, C.c_size_t, ip, ip, intp, intp, ip, ip, vp]
            L.clip_b200_text_tokens_layers.restype = C.c_bool
            L.clip_b200_text_tokens_layers.argtypes = [vp, i32p, C.c_size_t, ip, intp, intp, ip, ip, vp]
            L.clip_b200_text_tokens_layers_device.restype = C.c_bool
            L.clip_b200_text_tokens_layers_device.argtypes = [vp, vp, C.c_size_t, ip, intp, intp, ip, ip, vp]
            ipp = C.POINTER(C.c_int)
            L.clip_b200_topk_search.restype = C.c_bool
            L.clip_b200_topk_search.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, ip, fp, ipp]
            L.clip_b200_rows_to_16bit.restype = C.c_bool
            L.clip_b200_rows_to_16bit.argtypes = [vp, vp, C.c_size_t, ip, ip, vp]
            L.clip_b200_topk_search_16.restype = C.c_bool
            L.clip_b200_topk_search_16.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, ip, ip, ip, fp, ipp]
            L.clip_b200_rows_to_int8.restype = C.c_bool
            L.clip_b200_rows_to_int8.argtypes = [vp, vp, C.c_size_t, ip, vp, vp]
            L.clip_b200_topk_search_i8.restype = C.c_bool
            L.clip_b200_topk_search_i8.argtypes = [vp, vp, vp, C.c_size_t, vp, vp, C.c_size_t, ip, ip, fp, ipp]
            L.clip_b200_rows_to_binary.restype = C.c_bool
            L.clip_b200_rows_to_binary.argtypes = [vp, vp, C.c_size_t, ip, vp, vp]
            L.clip_b200_topk_search_b1.restype = C.c_bool
            L.clip_b200_topk_search_b1.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, ip, ip, fp, ipp]
            L.clip_b200_topk_rescore.restype = C.c_bool
            L.clip_b200_topk_rescore.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, ip, ip, ipp, ip, ip, fp, ipp]
            L.clip_b200_ivf_train_16.restype = C.c_bool
            L.clip_b200_ivf_train_16.argtypes = [vp, vp, C.c_size_t, ip, ip, ip, ip, vp]
            L.clip_b200_ivf_build_16.restype = C.c_bool
            L.clip_b200_ivf_build_16.argtypes = [vp, vp, C.c_size_t, ip, ip, vp, ip, vp, vp, vp]
            L.clip_b200_ivf_search_16.restype = C.c_bool
            L.clip_b200_ivf_search_16.argtypes = [vp, vp, C.c_size_t, ip, ip, vp, ip, vp, vp, vp, C.c_size_t, ip, ip, fp, ipp]
            L.clip_b200_ivfpq_train_16.restype = C.c_bool
            L.clip_b200_ivfpq_train_16.argtypes = [vp, vp, C.c_size_t, ip, ip, vp, ip, ip, ip, vp]
            L.clip_b200_ivfpq_encode_16.restype = C.c_bool
            L.clip_b200_ivfpq_encode_16.argtypes = [vp, vp, C.c_size_t, ip, ip, vp, ip, vp, ip, vp, vp]
            L.clip_b200_ivfpq_build.restype = C.c_bool
            L.clip_b200_ivfpq_build.argtypes = [vp, vp, vp, C.c_size_t, ip, ip, vp, vp, vp]
            L.clip_b200_ivfpq_search_16.restype = C.c_bool
            L.clip_b200_ivfpq_search_16.argtypes = [vp, vp, C.c_size_t, ip, ip, vp, ip, vp, ip, vp, vp, vp, C.c_size_t, ip, ip, fp, ipp]
            L.clip_b200_zero_shot_images.restype = C.c_bool
            L.clip_b200_zero_shot_images.argtypes = [vp, ip, C.POINTER(clip_image_f32_batch), C.POINTER(clip_tokens), C.c_size_t,
                                                     C.c_bool, ip, fp, ipp]
            L.clip_b200_dist_unique_id.restype = C.c_bool
            L.clip_b200_dist_unique_id.argtypes = [vp]
            L.clip_b200_dist_init_with_id.restype = C.c_bool
            L.clip_b200_dist_init_with_id.argtypes = [vp, ip, ip, vp]
            L.clip_b200_dist_init.restype = C.c_bool
            L.clip_b200_dist_init.argtypes = [vp, ip, ip, C.c_char_p]
            for f in ("clip_b200_dist_rank", "clip_b200_dist_world", "clip_b200_device_count"):
                getattr(L, f).restype = C.c_int
                getattr(L, f).argtypes = [vp]
            L.clip_b200_nccl_version.restype = C.c_int
            L.clip_b200_nccl_version.argtypes = []
            L.clip_b200_cuda_device_count.restype = C.c_int
            L.clip_b200_cuda_device_count.argtypes = []
            L.clip_b200_debug_pad_qkv.restype = C.c_int
            L.clip_b200_debug_pad_qkv.argtypes = [ip, ip, ip, ip, ip, vp, vp]
            L.clip_b200_debug_rendezvous.restype = C.c_int
            L.clip_b200_debug_rendezvous.argtypes = [ip, ip, C.c_char_p, vp]
            L.clip_b200_debug_shard_bounds.restype = None
            L.clip_b200_debug_shard_bounds.argtypes = [C.c_size_t, ip, ip, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
            L.clip_b200_dist_barrier.restype = C.c_bool
            L.clip_b200_dist_barrier.argtypes = [vp]
            L.clip_b200_dist_max_f64.restype = C.c_bool
            L.clip_b200_dist_max_f64.argtypes = [vp, C.POINTER(C.c_double), ip]
            L.clip_b200_dist_all_gather.restype = C.c_bool
            L.clip_b200_dist_all_gather.argtypes = [vp, vp, vp, C.c_size_t]
            L.clip_b200_image_encode_device_all.restype = C.c_bool
            L.clip_b200_image_encode_device_all.argtypes = [vp, vp, C.c_size_t, vp, C.c_bool]
            L.clip_b200_text_encode_device_all.restype = C.c_bool
            L.clip_b200_text_encode_device_all.argtypes = [vp, vp, vp, C.c_size_t, ip, vp, C.c_bool]
            L.clip_b200_image_batch_encode_all.restype = C.c_bool
            L.clip_b200_image_batch_encode_all.argtypes = [vp, ip, C.POINTER(clip_image_f32_batch), fp, C.c_bool]
            L.clip_b200_text_batch_encode_all.restype = C.c_bool
            L.clip_b200_text_batch_encode_all.argtypes = [vp, ip, C.POINTER(clip_tokens), C.c_size_t, fp, C.c_bool]

    # ---- model -----------------------------------------------------------------------------------
    def load(self, path: str, verbosity: int = 0):
        ctx = self.lib.clip_model_load(path.encode(), verbosity)
        if not ctx:
            raise RuntimeError("clip_model_load(%s) failed: %s" % (path, self.last_error()))
        return ctx

    def free(self, ctx):
        self.lib.clip_free(ctx)

    def last_error(self) -> str:
        if self.is_product:
            return self.lib.clip_b200_last_error().decode()
        return ""

    def vision_hparams(self, ctx) -> clip_vision_hparams:
        return self.lib.clip_get_vision_hparams(ctx).contents

    def text_hparams(self, ctx) -> clip_text_hparams:
        return self.lib.clip_get_text_hparams(ctx).contents

    def quantize(self, src: str, dst: str, itype: int) -> bool:
        return bool(self.lib.clip_model_quantize(src.encode(), dst.encode(), itype))

    # ---- encoders (host buffers; the reference-facing calls) ---------------------------------------
    @staticmethod
    def make_image_batch(images: np.ndarray):
        """images: [n, H, W, 3] float32 C-contiguous (H = W = image_size for the native calls) -> (batch struct, keep-alive tuple)."""
        assert images.dtype == np.float32 and images.flags["C_CONTIGUOUS"] and images.ndim == 4
        n, hgt, wid = images.shape[:3]
        arr = (clip_image_f32 * n)()
        per = hgt * wid * 3
        base = images.ctypes.data
        for i in range(n):
            arr[i].nx = wid
            arr[i].ny = hgt
            arr[i].size = per
            arr[i].data = C.cast(base + i * per * 4, C.POINTER(C.c_float))
        batch = clip_image_f32_batch(arr, n)
        return batch, (arr, images)

    def image_batch_encode(self, ctx, images: np.ndarray, normalize=True, n_threads=4) -> np.ndarray:
        d = self.vision_hparams(ctx).projection_dim
        batch, keep = self.make_image_batch(images)
        out = np.empty((images.shape[0], d), np.float32)
        ok = self.lib.clip_image_batch_encode(ctx, n_threads, C.byref(batch),
                                              out.ctypes.data_as(C.POINTER(C.c_float)), normalize)
        if not ok:
            raise RuntimeError("clip_image_batch_encode failed: " + self.last_error())
        return out

    def image_encode(self, ctx, image: np.ndarray, normalize=True, n_threads=4) -> np.ndarray:
        assert image.dtype == np.float32 and image.ndim == 3 and image.flags["C_CONTIGUOUS"]
        d = self.vision_hparams(ctx).projection_dim
        s = image.shape[0]
        img = clip_image_f32(s, s, image.ctypes.data_as(C.POINTER(C.c_float)), s * s * 3)
        out = np.empty((d,), np.float32)
        ok = self.lib.clip_image_encode(ctx, n_threads, C.byref(img), out.ctypes.data_as(C.POINTER(C.c_float)),
                                        normalize)
        if not ok:
            raise RuntimeError("clip_image_encode failed: " + self.last_error())
        return out

    def text_encode(self, ctx, ids: np.ndarray, normalize=True, n_threads=4) -> np.ndarray:
        ids = np.ascontiguousarray(ids, np.int32)
        d = self.text_hparams(ctx).projection_dim
        tk = clip_tokens(ids.ctypes.data_as(C.POINTER(C.c_int32)), ids.size)
        out = np.empty((d,), np.float32)
        ok = self.lib.clip_text_encode(ctx, n_threads, C.byref(tk), out.ctypes.data_as(C.POINTER(C.c_float)),
                                       normalize)
        if not ok:
            raise RuntimeError("clip_text_encode failed: " + self.last_error())
        return out

    def text_batch_encode(self, ctx, seqs, normalize=True, n_threads=4) -> np.ndarray:
        """seqs: list of int32 arrays (ragged).  Product-only extension (include/clip_b200.h)."""
        seqs = [np.ascontiguousarray(s, np.int32) for s in seqs]
        d = self.text_hparams(ctx).projection_dim
        arr = (clip_tokens * len(seqs))()
        for i, s in enumerate(seqs):
            arr[i].data = s.ctypes.data_as(C.POINTER(C.c_int32))
            arr[i].size = s.size
        out = np.empty((len(seqs), d), np.float32)
        ok = self.lib.clip_text_batch_encode(ctx, n_threads, arr, len(seqs),
                                             out.ctypes.data_as(C.POINTER(C.c_float)), normalize)
        if not ok:
            raise RuntimeError("clip_text_batch_encode failed: " + self.last_error())
        return out

    # ---- per-token hidden states (include/clip_b200.h) ------------------------------------------------------------------------
    def token_shape(self, ctx, vision: bool, n: int, rows: int, flags: int):
        """shape of a *_tokens output: [n, rows (T, T - 1 with NO_CLS, or seq_len), hidden_size or projection_dim]; with ATTENTION
        [n, n_head, rows or 1 (ATTENTION_CLS), rows]"""
        hp = self.vision_hparams(ctx) if vision else self.text_hparams(ctx)
        if flags & TOKENS_ATTENTION:
            return (n, hp.n_head, 1 if flags & TOKENS_ATTENTION_CLS else rows, rows)
        width = hp.projection_dim if flags & TOKENS_PROJECT else hp.hidden_size
        return (n, rows - (1 if flags & TOKENS_NO_CLS else 0), width)

    def image_tokens(self, ctx, images: np.ndarray, layer: int = -1, flags: int = 0, out_type: int = OUT_F32) -> np.ndarray:
        """images [n, S, S, 3] float32 -> rows of every image after `layer`: [n, T or T - 1, width] of OUT_DTYPES[out_type]"""
        batch, keep = self.make_image_batch(images)
        hp = self.vision_hparams(ctx)
        T = (hp.image_size // hp.patch_size) ** 2 + 1
        out = np.empty(self.token_shape(ctx, True, images.shape[0], T, flags), OUT_DTYPES.get(out_type, np.float32))
        if not self.lib.clip_b200_image_tokens(ctx, C.byref(batch), layer, flags, out_type, out.ctypes.data):
            raise RuntimeError("clip_b200_image_tokens failed: " + self.last_error())
        return out

    # ---- any patch-multiple image size (include/clip_b200.h: *_hw) --------------------------------------------------------------
    def image_batch_encode_hw(self, ctx, images: np.ndarray, normalize=True) -> np.ndarray:
        """images [n, H, W, 3] float32, H and W multiples of patch_size -> [n, projection_dim] (position table resampled to the grid)"""
        batch, keep = self.make_image_batch(images)
        out = np.empty((images.shape[0], self.vision_hparams(ctx).projection_dim), np.float32)
        if not self.lib.clip_b200_image_batch_encode_hw(ctx, C.byref(batch), out.ctypes.data_as(C.POINTER(C.c_float)), normalize):
            raise RuntimeError("clip_b200_image_batch_encode_hw failed: " + self.last_error())
        return out

    def image_tokens_hw(self, ctx, images: np.ndarray, layer: int = -1, flags: int = 0, out_type: int = OUT_F32) -> np.ndarray:
        """images [n, H, W, 3] float32 -> [n, T or T - 1, width], T = (H / P) * (W / P) + 1, patch rows in row-major grid order"""
        batch, keep = self.make_image_batch(images)
        P = self.vision_hparams(ctx).patch_size
        T = (images.shape[1] // P) * (images.shape[2] // P) + 1
        out = np.empty(self.token_shape(ctx, True, images.shape[0], T, flags), OUT_DTYPES.get(out_type, np.float32))
        if not self.lib.clip_b200_image_tokens_hw(ctx, C.byref(batch), layer, flags, out_type, out.ctypes.data):
            raise RuntimeError("clip_b200_image_tokens_hw failed: " + self.last_error())
        return out

    # ---- images of different sizes in one call (include/clip_b200.h: *_mixed) -------------------------------------------------
    @staticmethod
    def make_mixed_batch(images):
        """images: a list of [H_i, W_i, 3] float32 C-contiguous arrays -> (batch struct, keep-alive tuple)"""
        arr = (clip_image_f32 * len(images))()
        for i, im in enumerate(images):
            assert im.dtype == np.float32 and im.flags["C_CONTIGUOUS"] and im.ndim == 3
            arr[i].ny, arr[i].nx, arr[i].size = im.shape[0], im.shape[1], im.size
            arr[i].data = C.cast(im.ctypes.data, C.POINTER(C.c_float))
        return clip_image_f32_batch(arr, len(images)), (arr, images)

    def mixed_token_rows(self, ctx, sizes, flags: int) -> list:
        """rows per image of a *_tokens_mixed call: (H / P) * (W / P) + 1, less one with NO_CLS"""
        P = self.vision_hparams(ctx).patch_size
        return [(h // P) * (w // P) + 1 - (1 if flags & TOKENS_NO_CLS else 0) for h, w in sizes]

    def image_batch_encode_mixed(self, ctx, images, normalize=True) -> np.ndarray:
        """images: a list of [H_i, W_i, 3] float32 arrays, each its own patch-multiple size -> [n, projection_dim]"""
        batch, keep = self.make_mixed_batch(images)
        out = np.empty((len(images), self.vision_hparams(ctx).projection_dim), np.float32)
        if not self.lib.clip_b200_image_batch_encode_mixed(ctx, C.byref(batch), out.ctypes.data_as(C.POINTER(C.c_float)), normalize):
            raise RuntimeError("clip_b200_image_batch_encode_mixed failed: " + self.last_error())
        return out

    def image_tokens_mixed(self, ctx, images, layer: int = -1, flags: int = 0, out_type: int = OUT_F32) -> list:
        """images: a list of [H_i, W_i, 3] float32 arrays -> a list of [T_i or T_i - 1, width] arrays (views of one ragged buffer)"""
        batch, keep = self.make_mixed_batch(images)
        hp = self.vision_hparams(ctx)
        width = hp.projection_dim if flags & TOKENS_PROJECT else hp.hidden_size
        rows = self.mixed_token_rows(ctx, [im.shape[:2] for im in images], flags)
        flat = np.empty((sum(rows), width), OUT_DTYPES.get(out_type, np.float32))
        if not self.lib.clip_b200_image_tokens_mixed(ctx, C.byref(batch), layer, flags, out_type, flat.ctypes.data):
            raise RuntimeError("clip_b200_image_tokens_mixed failed: " + self.last_error())
        return np.split(flat, np.cumsum(rows)[:-1])

    # ---- token sequences of different lengths in one call (include/clip_b200.h: text *_packed) ----------------------------------
    def text_batch_encode_packed(self, ctx, seqs, normalize=True) -> np.ndarray:
        """seqs: a list of id lists / int32 arrays, each at its own length -> [n, projection_dim], packed with no padding"""
        seqs = [np.ascontiguousarray(s, np.int32) for s in seqs]
        arr = (clip_tokens * max(len(seqs), 1))()
        for i, s in enumerate(seqs):
            arr[i].data = s.ctypes.data_as(C.POINTER(C.c_int32))
            arr[i].size = s.size
        out = np.empty((len(seqs), self.text_hparams(ctx).projection_dim), np.float32)
        if not self.lib.clip_b200_text_batch_encode_packed(ctx, arr, len(seqs), out.ctypes.data_as(C.POINTER(C.c_float)), normalize):
            raise RuntimeError("clip_b200_text_batch_encode_packed failed: " + self.last_error())
        return out

    def text_tokens_packed(self, ctx, seqs, layer: int = -1, flags: int = 0, out_type: int = OUT_F32) -> list:
        """seqs: a list of id lists / int32 arrays -> a list of [len_i, width] arrays (views of one ragged buffer)"""
        seqs = [np.ascontiguousarray(s, np.int32) for s in seqs]
        lens = np.array([s.size for s in seqs], np.int32)
        ids = np.concatenate(seqs) if seqs else np.zeros(1, np.int32)
        hp = self.text_hparams(ctx)
        width = hp.projection_dim if flags & TOKENS_PROJECT else hp.hidden_size
        flat = np.empty((int(lens.sum()), width), OUT_DTYPES.get(out_type, np.float32))
        if not self.lib.clip_b200_text_tokens_packed(ctx, ids.ctypes.data_as(C.POINTER(C.c_int32)), len(seqs),
                                                     lens.ctypes.data_as(C.POINTER(C.c_int)), layer, flags, out_type, flat.ctypes.data):
            raise RuntimeError("clip_b200_text_tokens_packed failed: " + self.last_error())
        return np.split(flat, np.cumsum(lens)[:-1]) if seqs else []

    def text_tokens(self, ctx, ids: np.ndarray, layer: int = -1, flags: int = 0, out_type: int = OUT_F32) -> np.ndarray:
        """ids [n, seq_len] int32, padded by the caller -> [n, seq_len, width] of OUT_DTYPES[out_type]"""
        ids = np.ascontiguousarray(ids, np.int32)
        out = np.empty(self.token_shape(ctx, False, ids.shape[0], ids.shape[1], flags), OUT_DTYPES.get(out_type, np.float32))
        if not self.lib.clip_b200_text_tokens(ctx, ids.ctypes.data_as(C.POINTER(C.c_int32)), ids.shape[0], ids.shape[1], layer, flags,
                                              out_type, out.ctypes.data):
            raise RuntimeError("clip_b200_text_tokens failed: " + self.last_error())
        return out

    # ---- several layers from one forward pass (include/clip_b200.h: *_tokens_layers) ----------------------------------------------
    def _layers_call(self, ctx, vision, n, rows, layers, flags, out_type, out, call, name):
        """run call(c_layers, c_flags, n_layers, out) and return the per-entry views of the layer-major output, each shaped as the
        single-layer wrapper shapes its result.  flags None is passed as NULL (0 for every entry).  `out`: a flat buffer of the
        output dtype to write into (for example pinned memory), or None for a new numpy array."""
        layers = [int(l) for l in layers]
        k = max(len(layers), 1)
        c_layers = (C.c_int * k)(*layers)
        fl = [0] * len(layers) if flags is None else [int(f) for f in flags]
        c_flags = None if flags is None else (C.c_int * max(len(fl), 1))(*fl)
        shapes = [self.token_shape(ctx, vision, n, rows, f) for f in fl[:len(layers)]]
        sizes = [int(np.prod(s)) for s in shapes]
        dtype = np.dtype(OUT_DTYPES.get(out_type, np.float32))
        offs = [b // dtype.itemsize for b in slab_offsets([z * dtype.itemsize for z in sizes], fl)]
        total = offs[-1] + sizes[-1] if sizes else 0
        if out is None:
            out = np.empty(total, dtype)
        assert out.flags["C_CONTIGUOUS"] and out.size >= total
        if not call(c_layers, c_flags, len(layers), out):
            raise RuntimeError(name + " failed: " + self.last_error())
        flat = out.reshape(-1)
        return [flat[o:o + z].reshape(s) for o, z, s in zip(offs, sizes, shapes)]

    def _via_device(self, ctx, inp, out, fn):
        """upload inp, fn(d_in, d_out) into a device buffer of out.nbytes, download into out"""
        d_in = self.lib.clip_b200_device_malloc(ctx, max(inp.nbytes, 1))
        d_out = self.lib.clip_b200_device_malloc(ctx, max(out.nbytes, 1))
        try:
            if not (d_in and d_out and self.lib.clip_b200_memcpy_h2d(ctx, d_in, inp.ctypes.data, inp.nbytes)):
                return False
            if not fn(d_in, d_out):
                return False
            return self.lib.clip_b200_memcpy_d2h(ctx, out.ctypes.data, d_out, out.nbytes)
        finally:
            self.lib.clip_b200_device_free(ctx, d_in)
            self.lib.clip_b200_device_free(ctx, d_out)

    def image_tokens_layers(self, ctx, images: np.ndarray, layers, flags=None, out_type: int = OUT_F32, out=None):
        """images [n, H, W, 3] float32 -> one [n, T or T - 1, width] array per entry (layers[j], flags[j]), from one forward pass"""
        batch, keep = self.make_image_batch(images)
        P = self.vision_hparams(ctx).patch_size
        T = (images.shape[1] // P) * (images.shape[2] // P) + 1
        return self._layers_call(ctx, True, images.shape[0], T, layers, flags, out_type, out,
                                 lambda ls, fs, k, o: self.lib.clip_b200_image_tokens_layers(ctx, C.byref(batch), ls, fs, k, out_type, o.ctypes.data),
                                 "clip_b200_image_tokens_layers")

    def image_tokens_layers_device(self, ctx, images: np.ndarray, layers, flags=None, out_type: int = OUT_F32):
        """image_tokens_layers through the device form: images uploaded, the slabs written on the GPU and downloaded"""
        images = np.ascontiguousarray(images, np.float32)
        n, H, W = images.shape[:3]
        P = self.vision_hparams(ctx).patch_size
        return self._layers_call(ctx, True, n, (H // P) * (W // P) + 1, layers, flags, out_type, None,
                                 lambda ls, fs, k, o: self._via_device(ctx, images, o, lambda di, do: self.lib.clip_b200_image_tokens_layers_device(
                                     ctx, di, n, H, W, ls, fs, k, out_type, do)),
                                 "clip_b200_image_tokens_layers_device")

    def text_tokens_layers(self, ctx, ids: np.ndarray, layers, flags=None, out_type: int = OUT_F32, out=None):
        """ids [n, seq_len] int32, padded by the caller -> one [n, seq_len, width] array per entry, from one forward pass"""
        ids = np.ascontiguousarray(ids, np.int32)
        return self._layers_call(ctx, False, ids.shape[0], ids.shape[1], layers, flags, out_type, out,
                                 lambda ls, fs, k, o: self.lib.clip_b200_text_tokens_layers(
                                     ctx, ids.ctypes.data_as(C.POINTER(C.c_int32)), ids.shape[0], ids.shape[1], ls, fs, k, out_type, o.ctypes.data),
                                 "clip_b200_text_tokens_layers")

    def text_tokens_layers_device(self, ctx, ids: np.ndarray, layers, flags=None, out_type: int = OUT_F32):
        """text_tokens_layers through the device form"""
        ids = np.ascontiguousarray(ids, np.int32)
        n, S = ids.shape
        return self._layers_call(ctx, False, n, S, layers, flags, out_type, None,
                                 lambda ls, fs, k, o: self._via_device(ctx, ids, o, lambda di, do: self.lib.clip_b200_text_tokens_layers_device(
                                     ctx, di, n, S, ls, fs, k, out_type, do)),
                                 "clip_b200_text_tokens_layers_device")

    @staticmethod
    def make_token_array(seqs):
        seqs = [np.ascontiguousarray(s, np.int32) for s in seqs]
        arr = (clip_tokens * max(len(seqs), 1))()
        for i, s in enumerate(seqs):
            arr[i].data = s.ctypes.data_as(C.POINTER(C.c_int32))
            arr[i].size = s.size
        return arr, seqs

    def zero_shot_images(self, ctx, images: np.ndarray, label_seqs, top_k: int, normalize=False, n_threads=4):
        """extension: batch form of clip_zero_shot_label_image -> (scores [n, k], indices [n, k]); labels are token arrays.
        In ranks mode `label_seqs` is this rank's shard and the result ranks ALL ranks' labels (index = rank * len + j)."""
        batch, keep = self.make_image_batch(images)
        arr, keep2 = self.make_token_array(label_seqs)
        n_all = len(label_seqs) * max(1, self.lib.clip_b200_dist_world(ctx))
        k = n_all if top_k <= 0 or top_k > n_all else top_k
        scores = np.empty((images.shape[0], k), np.float32)
        idx = np.empty((images.shape[0], k), np.int32)
        ok = self.lib.clip_b200_zero_shot_images(ctx, n_threads, C.byref(batch), arr, len(label_seqs), normalize, k,
                                                 scores.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int)))
        if not ok:
            raise RuntimeError("clip_b200_zero_shot_images failed: " + self.last_error())
        return scores, idx

    def compare_text_and_image(self, ctx, text: str, img_u8: np.ndarray, n_threads=4) -> float:
        img_u8 = np.ascontiguousarray(img_u8, np.uint8)
        src = clip_image_u8(img_u8.shape[1], img_u8.shape[0], img_u8.ctypes.data_as(C.POINTER(C.c_uint8)), img_u8.size)
        score = C.c_float(0)
        if not self.lib.clip_compare_text_and_image(ctx, n_threads, text.encode(), C.byref(src), C.byref(score)):
            raise RuntimeError("clip_compare_text_and_image failed: " + self.last_error())
        return float(score.value)

    def zero_shot_label_image(self, ctx, img_u8: np.ndarray, labels, n_threads=4):
        img_u8 = np.ascontiguousarray(img_u8, np.uint8)
        src = clip_image_u8(img_u8.shape[1], img_u8.shape[0], img_u8.ctypes.data_as(C.POINTER(C.c_uint8)), img_u8.size)
        arr = (C.c_char_p * len(labels))(*[l.encode() for l in labels])
        scores = np.empty(len(labels), np.float32)
        idx = np.empty(len(labels), np.int32)
        if not self.lib.clip_zero_shot_label_image(ctx, n_threads, C.byref(src), arr, len(labels),
                                                   scores.ctypes.data_as(C.POINTER(C.c_float)), idx.ctypes.data_as(C.POINTER(C.c_int))):
            raise RuntimeError("clip_zero_shot_label_image failed: " + self.last_error())
        return scores, idx

    def tokenize(self, ctx, text: str) -> np.ndarray:
        tk = clip_tokens()
        if not self.lib.clip_tokenize(ctx, text.encode(), C.byref(tk)):
            raise RuntimeError("clip_tokenize failed")
        return np.ctypeslib.as_array(tk.data, shape=(tk.size,)).copy()

    def _u8_batch(self, images):
        """list of [ny, nx, 3] uint8 arrays -> (clip_image_u8_batch, keep-alive objects)"""
        arrs = [np.ascontiguousarray(im, np.uint8) for im in images]
        items = (clip_image_u8 * len(arrs))()
        for i, a in enumerate(arrs):
            items[i] = clip_image_u8(a.shape[1], a.shape[0], a.ctypes.data_as(C.POINTER(C.c_uint8)), a.size)
        return clip_image_u8_batch(items, len(arrs)), (arrs, items)

    def image_batch_encode_u8(self, ctx, images, normalize=True) -> np.ndarray:
        """extension (N1): raw u8 images of any size -> embeddings; resize / crop / normalise run on the GPU"""
        batch, keep = self._u8_batch(images)
        d = self.vision_hparams(ctx).projection_dim
        out = np.empty((len(images), d), np.float32)
        if not self.lib.clip_b200_image_batch_encode_u8(ctx, C.byref(batch), out.ctypes.data_as(C.POINTER(C.c_float)), normalize):
            raise RuntimeError("clip_b200_image_batch_encode_u8 failed: " + self.last_error())
        return out

    def preprocess_device(self, ctx, images) -> np.ndarray:
        """extension (N1): GPU preprocess alone -> [n, S, S, 3] float32"""
        batch, keep = self._u8_batch(images)
        res = (clip_image_f32 * len(images))()
        outb = clip_image_f32_batch(res, len(images))
        if not self.lib.clip_b200_image_batch_preprocess_device(ctx, C.byref(batch), C.byref(outb)):
            raise RuntimeError("clip_b200_image_batch_preprocess_device failed: " + self.last_error())
        s = res[0].nx
        out = np.stack([np.ctypeslib.as_array(res[i].data, shape=(s, s, 3)).copy() for i in range(len(images))])
        for i in range(len(images)):
            self.lib.clip_image_f32_clean(C.byref(res[i]))
        return out

    def batch_preprocess(self, ctx, images, n_threads: int = 4) -> np.ndarray:
        """clip_image_batch_preprocess (clip.h:95-96): the reference's batch call -> [n, S, S, 3] float32.  Host threads by default,
        the GPU when CLIP_B200_PREPROCESS=device is set in the environment."""
        batch, keep = self._u8_batch(images)
        res = (clip_image_f32 * len(images))()
        outb = clip_image_f32_batch(res, len(images))
        self.lib.clip_image_batch_preprocess(ctx, n_threads, C.byref(batch), C.byref(outb))
        if any(not res[i].data for i in range(len(images))):
            raise RuntimeError("clip_image_batch_preprocess failed: " + self.last_error())
        s = res[0].nx
        out = np.stack([np.ctypeslib.as_array(res[i].data, shape=(s, s, 3)).copy() for i in range(len(images))])
        for i in range(len(images)):
            self.lib.clip_image_f32_clean(C.byref(res[i]))
        return out

    def preprocess(self, ctx, img_u8: np.ndarray) -> np.ndarray:
        """img_u8: [ny, nx, 3] uint8 -> [S, S, 3] float32 (clip.cpp:797-927 semantics)."""
        img_u8 = np.ascontiguousarray(img_u8, np.uint8)
        ny, nx = img_u8.shape[:2]
        src = clip_image_u8(nx, ny, img_u8.ctypes.data_as(C.POINTER(C.c_uint8)), img_u8.size)
        dst = clip_image_f32()
        if not self.lib.clip_image_preprocess(ctx, C.byref(src), C.byref(dst)):
            raise RuntimeError("clip_image_preprocess failed")
        s = dst.nx
        out = np.ctypeslib.as_array(dst.data, shape=(s, s, 3)).copy()
        self.lib.clip_image_f32_clean(C.byref(dst))
        return out
