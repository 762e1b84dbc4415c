"""ctypes binding of libape_b200.so (the C-ABI declared in include/ape_b200.h).

The library is built in-tree by `make` / `__graft_entry__.build()`; there is no CPU
fallback: if it is missing, importing this module raises."""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libape_b200.so")

APE_DTYPE_F32, APE_DTYPE_F16, APE_DTYPE_BF16, APE_DTYPE_E4M3 = 0, 1, 2, 3
_DTYPE_CODE = {torch.float32: APE_DTYPE_F32, torch.float16: APE_DTYPE_F16, torch.bfloat16: APE_DTYPE_BF16,
               torch.float8_e4m3fn: APE_DTYPE_E4M3}

# APE_B200_CONTAINER_ONLY=1: import the package for its parameter containers / configs only (bench.py's CPU reference arm
# builds the reference-named state_dict this way) WITHOUT mapping the native library; every kernel entry point then raises.
CONTAINER_ONLY = os.environ.get("APE_B200_CONTAINER_ONLY") == "1"


class _NotLoaded:
    def __getattr__(self, name):
        raise RuntimeError(f"libape_b200.so is not loaded (APE_B200_CONTAINER_ONLY=1): `{name}` is unavailable; "
                           "ape_b200 has no CPU / PyTorch fallback")


if CONTAINER_ONLY:
    lib = _NotLoaded()
elif not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} not found: build it with `make` (or `python -c 'import __graft_entry__ as g; g.build()'`). "
        "ape_b200 has no CPU / PyTorch fallback."
    )
else:
    lib = ctypes.CDLL(LIB_PATH)

_vp, _i, _i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64


def _declare(lib):

    lib.ape_abi_version.restype = _i
    lib.ape_abi_version.argtypes = []
    lib.ape_last_error.restype = ctypes.c_char_p
    lib.ape_last_error.argtypes = []
    lib.ape_launch_count.restype = ctypes.c_uint64
    lib.ape_launch_count.argtypes = []
    lib.ape_msda_fwd.restype = _i
    lib.ape_msda_fwd.argtypes = [_vp] * 6 + [_i] * 8 + [_vp]
    lib.ape_msda_fwd_variant.restype = _i
    lib.ape_msda_fwd_variant.argtypes = [_vp] * 6 + [_i] * 9 + [_vp]
    lib.ape_msda_fused_fwd.restype = _i
    lib.ape_msda_fused_fwd.argtypes = [_vp, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _i, _vp] + [_i] * 9 + [_vp]

    lib.ape_msda_bwd.restype = _i
    lib.ape_msda_bwd.argtypes = [_vp] * 9 + [_i] * 8 + [_vp]
    lib.ape_msda_pair_values.restype = _i
    lib.ape_msda_pair_values.argtypes = [_vp, _i64, _vp, _vp, _i, _i, _i, _i, _i, _vp]
    lib.ape_msda_pair_supported.restype = _i
    lib.ape_msda_pair_supported.argtypes = [_vp, _i, _i, _i, _i, _i]
    lib.ape_msda_pair_fused_fwd.restype = _i
    lib.ape_msda_pair_fused_fwd.argtypes = [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _i, _vp] + [_i] * 12 + [_vp]
    lib.ape_gemm_tn.restype = _i
    lib.ape_gemm_tn.argtypes = [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i64] + [_i] * 7 + [_vp]

    lib.ape_gemm_tn_ex.restype = _i
    lib.ape_gemm_tn_ex.argtypes = [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i64] + [_i] * 8 + [_vp]
    lib.ape_gemm_tn_fused.restype = _i
    lib.ape_gemm_tn_fused.argtypes = [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _vp, _i64] + [_i] * 8 + [_vp, _i, _vp, ctypes.c_float, ctypes.c_float, _vp, _i, _vp]
    lib.ape_gemm_tn_e4m3.restype = _i
    lib.ape_gemm_tn_e4m3.argtypes = [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _i, _i, _vp, _i, _vp]
    lib.ape_conv3x3_nhwc.restype = _i
    lib.ape_conv3x3_nhwc.argtypes = [_vp, _vp, _vp, _vp] + [_i] * 7 + [_vp]
    lib.ape_gemm_set_trace.restype = None
    lib.ape_gemm_set_trace.argtypes = [_vp]
    lib.ape_ffn_fused.restype = _i
    lib.ape_ffn_fused.argtypes = [_vp, _i64, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64] + [_i] * 5 + [_vp]
    lib.ape_gemm_tn_rope.restype = _i
    lib.ape_gemm_tn_rope.argtypes = [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _vp]

    lib.ape_layernorm.restype = _i
    lib.ape_layernorm.argtypes = [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _i, _i, ctypes.c_float, _i, _i, _vp]
    lib.ape_layernorm_e4m3.restype = _i
    lib.ape_layernorm_e4m3.argtypes = [_vp, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _i, _i, ctypes.c_float, _i, _vp]
    lib.ape_layernorm_ex.restype = _i
    lib.ape_layernorm_ex.argtypes = [_vp, _i64, _vp, _i64, _vp, _vp, ctypes.c_float, _vp, _vp, ctypes.c_float, _vp, _i64, _i,
                                     _vp, _i64, _vp, _i64, _i, _i, _i, _i, _vp]
    lib.ape_groupnorm_workspace_bytes.restype = _i64
    lib.ape_groupnorm_workspace_bytes.argtypes = [_i, _i, _i]
    lib.ape_groupnorm_nhwc.restype = _i
    lib.ape_groupnorm_nhwc.argtypes = [_vp, _i64, _vp, _i64, _i64, _vp, _vp, _vp, _i, _i, _i, _i, ctypes.c_float, _i, _i, _vp]
    lib.ape_rope_qk.restype = _i
    lib.ape_rope_qk.argtypes = [_vp, _i64, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]

    lib.ape_text_embed_packed.restype = _i
    lib.ape_text_embed_packed.argtypes = [_vp] * 5 + [_i] * 4 + [_vp]
    lib.ape_rows_gather.restype = _i
    lib.ape_rows_gather.argtypes = [_vp, _i64, _vp, _vp, _i64, _i, _i, _vp]

    lib.ape_attn_fwd.restype = _i
    lib.ape_attn_fwd.argtypes = [_vp, _i64, _vp, _i64, _i, _i, _i, _i, ctypes.c_float, _i, _vp]
    lib.ape_attn_fwd_ex.restype = _i
    lib.ape_attn_fwd_ex.argtypes = [_vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, ctypes.c_float, _i, _vp, _i, _i, _i64, _vp]
    lib.ape_attn_fwd_mapped.restype = _i
    lib.ape_attn_fwd_mapped.argtypes = [_vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, ctypes.c_float, _i, _vp, _i, _i, _i64, _vp, _vp]
    lib.ape_attn_fwd_seg.restype = _i
    lib.ape_attn_fwd_seg.argtypes = [_vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, ctypes.c_float, _i, _vp, _i, _i, _i64, _vp, _vp]
    lib.ape_attn_variant.restype = _i
    lib.ape_attn_variant.argtypes = [_i]
    lib.ape_attn_cross_fwd.restype = _i
    lib.ape_attn_cross_fwd.argtypes = [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _i, ctypes.c_float, _i, _vp]
    lib.ape_vlf_pool_workspace_bytes.restype = _i64
    lib.ape_vlf_pool_workspace_bytes.argtypes = [_i, _i, _i, _i]
    lib.ape_vlf_pool.restype = _i
    lib.ape_vlf_pool.argtypes = [_vp, _vp, _vp, _vp, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(_i)] + [_i] * 6 + [_vp]
    lib.ape_nms_workspace_bytes.restype = _i64
    lib.ape_nms_workspace_bytes.argtypes = [_i]
    lib.ape_nms_sorted.restype = _i
    lib.ape_nms_sorted.argtypes = [_vp, _i, ctypes.c_float, _vp, _vp, _vp, _vp]
    lib.ape_nms_sorted_dev.restype = _i
    lib.ape_nms_sorted_dev.argtypes = [_vp, _i, _vp, ctypes.c_float, _vp, _vp, _vp, _vp]
    lib.ape_nms_classwise_workspace_bytes.restype = _i64
    lib.ape_nms_classwise_workspace_bytes.argtypes = [_i]
    lib.ape_nms_classwise.restype = _i
    lib.ape_nms_classwise.argtypes = [_vp, _vp, _i64, _vp, _i, _i, ctypes.c_float, ctypes.c_float, _vp, _vp, _vp]
    lib.ape_ref_update.restype = _i
    lib.ape_ref_update.argtypes = [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, ctypes.c_float, _vp]
    lib.ape_gemv_f32.restype = _i
    lib.ape_gemv_f32.argtypes = [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]
    lib.ape_mask_crop_workspace_bytes.restype = _i64
    lib.ape_mask_crop_workspace_bytes.argtypes = [_i, _i, _i]
    lib.ape_mask_crop.restype = _i
    lib.ape_mask_crop.argtypes = [_vp] * 5 + [_i] * 7 + [_vp]
    lib.ape_mask_paste.restype = _i
    lib.ape_mask_paste.argtypes = [_vp, _vp, _vp, _i, _i, _i, _i, ctypes.c_float, _vp]
    lib.ape_mask_paste_rle.restype = _i
    lib.ape_mask_paste_rle.argtypes = [_vp, _vp, _i, _i, _i, _i, ctypes.c_float, _vp, _vp, _vp, _vp]
    lib.ape_rle_to_string.restype = _i
    lib.ape_rle_to_string.argtypes = [_vp, _i, _vp]
    lib.ape_mask_pack_workspace_bytes.restype = _i64
    lib.ape_mask_pack_workspace_bytes.argtypes = [_i] * 6
    lib.ape_mask_pack.restype = _i
    lib.ape_mask_pack.argtypes = [_vp] * 5 + [_i] * 10 + [_vp]
    lib.ape_resample_ksize.restype = _i
    lib.ape_resample_ksize.argtypes = [_i, _i]
    lib.ape_resample_coeffs_u8.restype = _i
    lib.ape_resample_coeffs_u8.argtypes = [_i, _i, _vp, _vp]
    lib.ape_resample_u8.restype = _i
    lib.ape_resample_u8.argtypes = [_vp, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _i, _vp, _vp, _i] + [_i] * 6 + [_vp]
    lib.ape_semseg_resample.restype = _i
    lib.ape_semseg_resample.argtypes = [_vp, _vp, _vp, _i64] + [_i] * 13 + [_vp]
    lib.ape_semseg_keys_init.restype = _i
    lib.ape_semseg_keys_init.argtypes = [_vp, _i64, ctypes.c_float, _i, _vp]
    lib.ape_gemm_tn_argmax.restype = _i
    lib.ape_gemm_tn_argmax.argtypes = [_vp, _i64, _vp, _i64, _vp, _i, _i, _i, _i, _i, _vp]
    lib.ape_semseg_keys_decode.restype = _i
    lib.ape_semseg_keys_decode.argtypes = [_vp, _i64, _vp, _vp, _vp]
    lib.ape_label_rle_workspace_bytes.restype = _i64
    lib.ape_label_rle_workspace_bytes.argtypes = [_i, _i, _i64]
    lib.ape_label_rle_out_bytes.restype = _i64
    lib.ape_label_rle_out_bytes.argtypes = [_i, _i]
    lib.ape_label_rle_sizes.restype = _i
    lib.ape_label_rle_sizes.argtypes = [_vp, _i, _i, _vp, _vp, _vp]
    lib.ape_label_rle.restype = _i
    lib.ape_label_rle.argtypes = [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp]
    lib.ape_label_rle_pack_workspace_bytes.restype = _i64
    lib.ape_label_rle_pack_workspace_bytes.argtypes = [_i, _i, _i]
    lib.ape_label_rle_pack.restype = _i
    lib.ape_label_rle_pack.argtypes = [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]
    lib.ape_panoptic_winners.restype = _i
    lib.ape_panoptic_winners.argtypes = [_vp] * 5 + [_i] * 9 + [ctypes.c_float, _i, _vp]
    lib.ape_panoptic_pack_workspace_bytes.restype = _i64
    lib.ape_panoptic_pack_workspace_bytes.argtypes = [_i, _i]
    lib.ape_panoptic_pack.restype = _i
    lib.ape_panoptic_pack.argtypes = [_vp] * 3 + [_i] * 4 + [ctypes.c_double, _i, _i, _vp, _vp, _i, _vp]
    lib.ape_pad_geometry.restype = _i
    lib.ape_pad_geometry.argtypes = [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _i] + [ctypes.c_float] * 3 + [_i, _vp, _vp, _i] + [_vp] * 6
    lib.ape_zero_masked_rows.restype = _i
    lib.ape_zero_masked_rows.argtypes = [_vp, _i64, _vp, _i64, _i, _i, _vp]
    lib.ape_mask_pack_dev.restype = _i
    lib.ape_mask_pack_dev.argtypes = [_vp, _vp, _vp, _i, _vp, _vp] + [_i] * 10 + [_vp]
    lib.ape_semseg_keys_init_dev.restype = _i
    lib.ape_semseg_keys_init_dev.argtypes = [_vp, _vp, _i, ctypes.c_float, _i, _i64, _i, _vp, _vp]
    lib.ape_semseg_resample_dev.restype = _i
    lib.ape_semseg_resample_dev.argtypes = [_vp, _vp, _vp, _i64] + [_i] * 5 + [_vp, _i, _i64, _i, _i, _i, _vp]
    lib.ape_gemm_tn_argmax_dev.restype = _i
    lib.ape_gemm_tn_argmax_dev.argtypes = [_vp, _i64, _vp, _i64, _vp, _i, _vp, _i, _i, _i, _i, _vp]
    lib.ape_semseg_keys_decode_dev.restype = _i
    lib.ape_semseg_keys_decode_dev.argtypes = [_vp, _vp, _i, _vp, _vp, _vp]
    lib.ape_label_rle_pack_dev.restype = _i
    lib.ape_label_rle_pack_dev.argtypes = [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp]
    lib.ape_panoptic_winners_dev.restype = _i
    lib.ape_panoptic_winners_dev.argtypes = [_vp] * 5 + [_i] * 5 + [_vp, _i, ctypes.c_float, _i, _vp]
    lib.ape_panoptic_pack_dev.restype = _i
    lib.ape_panoptic_pack_dev.argtypes = [_vp] * 3 + [_i] * 4 + [ctypes.c_double, _vp, _i, _vp, _vp, _i, _vp]



if not CONTAINER_ONLY:
    _declare(lib)

# every symbol include/ape_b200.h declares (tests check the .so exports exactly these)
EXPORTS = (
    "ape_abi_version",
    "ape_last_error",
    "ape_launch_count",
    "ape_msda_fwd",
    "ape_msda_fwd_variant",
    "ape_msda_fused_fwd",
    "ape_msda_bwd",
    "ape_msda_pair_values",
    "ape_msda_pair_supported",
    "ape_msda_pair_fused_fwd",
    "ape_gemm_tn",
    "ape_gemm_tn_ex",
    "ape_gemm_tn_fused",
    "ape_gemm_tn_e4m3",
    "ape_conv3x3_nhwc",
    "ape_gemm_tn_rope",
    "ape_ffn_fused",
    "ape_gemm_set_trace",
    "ape_layernorm",
    "ape_layernorm_e4m3",
    "ape_layernorm_ex",
    "ape_rope_qk",
    "ape_text_embed_packed",
    "ape_rows_gather",
    "ape_attn_fwd",
    "ape_attn_fwd_ex",
    "ape_attn_fwd_mapped",
    "ape_attn_fwd_seg",
    "ape_attn_variant",
    "ape_attn_cross_fwd",
    "ape_groupnorm_workspace_bytes",
    "ape_groupnorm_nhwc",
    "ape_vlf_pool_workspace_bytes",
    "ape_vlf_pool",
    "ape_nms_workspace_bytes",
    "ape_nms_sorted",
    "ape_nms_sorted_dev",
    "ape_nms_classwise_workspace_bytes",
    "ape_nms_classwise",
    "ape_ref_update",
    "ape_gemv_f32",
    "ape_mask_crop_workspace_bytes",
    "ape_mask_crop",
    "ape_mask_paste",
    "ape_mask_paste_rle",
    "ape_rle_to_string",
    "ape_mask_pack_workspace_bytes",
    "ape_mask_pack",
    "ape_resample_ksize",
    "ape_resample_coeffs_u8",
    "ape_resample_u8",
    "ape_semseg_resample",
    "ape_semseg_keys_init",
    "ape_gemm_tn_argmax",
    "ape_semseg_keys_decode",
    "ape_label_rle_workspace_bytes",
    "ape_label_rle_out_bytes",
    "ape_label_rle_sizes",
    "ape_label_rle",
    "ape_label_rle_pack_workspace_bytes",
    "ape_label_rle_pack",
    "ape_panoptic_winners",
    "ape_panoptic_pack_workspace_bytes",
    "ape_panoptic_pack",
    "ape_pad_geometry",
    "ape_zero_masked_rows",
    "ape_mask_pack_dev",
    "ape_semseg_keys_init_dev",
    "ape_semseg_resample_dev",
    "ape_gemm_tn_argmax_dev",
    "ape_semseg_keys_decode_dev",
    "ape_label_rle_pack_dev",
    "ape_panoptic_winners_dev",
    "ape_panoptic_pack_dev",
)


def dtype_code(dt: torch.dtype) -> int:
    try:
        return _DTYPE_CODE[dt]
    except KeyError:
        raise RuntimeError(f"ape_b200: unsupported dtype {dt} (float32 / float16 / bfloat16 / float8_e4m3fn only)") from None


def check(status: int, what: str) -> None:
    """Convert a non-zero C-ABI status into RuntimeError (the reference only printf's launch
    errors, ms_deform_im2col_cuda.cuh:948-952; we raise)."""
    if status != 0:
        msg = lib.ape_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed (status {status}): {msg}")


def current_stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def launch_count() -> int:
    return int(lib.ape_launch_count())
