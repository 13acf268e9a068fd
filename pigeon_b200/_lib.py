"""ctypes binding of libpigeon_b200.so (the C ABI declared in include/pigeon_b200.h).

There is deliberately no fallback: if the shared object is missing or a call fails, a
`PigeonB200Error` is raised — nothing here ever routes to PyTorch/CPU arithmetic.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Optional

from . import _build

c_void_p, c_int32, c_int64, c_size_t, c_float, c_double = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t, C.c_float, C.c_double


class PigeonB200Error(RuntimeError):
    pass


class VitConfig(C.Structure):
    _fields_ = [("image_size", c_int32), ("patch_size", c_int32), ("hidden", c_int32), ("heads", c_int32),
                ("intermediate", c_int32), ("layers", c_int32), ("ln_eps", c_float), ("patch_k_pad", c_int32)]


class Image(C.Structure):
    _fields_ = [("data", c_void_p), ("height", c_int32), ("width", c_int32), ("row_stride", c_int64)]


class VitLayer(C.Structure):
    _fields_ = [(n, c_void_p) for n in ("ln1_g", "ln1_b", "w_qkv", "b_qkv", "w_o", "b_o", "ln2_g", "ln2_b",
                                        "w_fc1", "b_fc1", "w_fc2", "b_fc2", "w_qkv_ln", "b_qkv_ln", "cs_qkv",
                                        "w_fc1_ln", "b_fc1_ln", "cs_fc1")]


class VitSavedLayer(C.Structure):
    _fields_ = [(n, c_void_p) for n in ("x0", "xn1", "qkv", "lse2", "ao", "x1", "xn2", "u", "h")]


class VitSaved(C.Structure):
    _fields_ = [("im2col", c_void_p), ("e", c_void_p), ("x_out", c_void_p), ("layers_host", C.POINTER(VitSavedLayer))]


class VitLayerBwd(C.Structure):
    _fields_ = [(n, c_void_p) for n in ("w_qkv_t", "w_o_t", "w_fc1_t", "w_fc2_t", "d_ln1_g", "d_ln1_b", "d_w_qkv",
                                        "d_b_qkv", "d_w_o", "d_b_o", "d_ln2_g", "d_ln2_b", "d_w_fc1", "d_b_fc1",
                                        "d_w_fc2", "d_b_fc2")]


class VitGrads(C.Structure):
    _fields_ = [("d_patch_w", c_void_p), ("d_class_emb", c_void_p), ("d_pos_emb", c_void_p), ("d_pre_ln_g", c_void_p),
                ("d_pre_ln_b", c_void_p), ("layers_host", C.POINTER(VitLayerBwd)),
                ("layer_done_events", C.POINTER(c_void_p))]


class VitWeights(C.Structure):
    _fields_ = [("patch_w", c_void_p), ("class_emb", c_void_p), ("pos_emb", c_void_p), ("pre_ln_g", c_void_p),
                ("pre_ln_b", c_void_p), ("layers_host", C.POINTER(VitLayer))]


class TextConfig(C.Structure):
    _fields_ = [("vocab", c_int32), ("max_positions", c_int32), ("hidden", c_int32), ("heads", c_int32),
                ("intermediate", c_int32), ("layers", c_int32), ("ln_eps", c_float)]


class TextWeights(C.Structure):
    _fields_ = [("token_emb", c_void_p), ("pos_emb", c_void_p), ("layers_host", C.POINTER(VitLayer)),
                ("final_ln_g", c_void_p), ("final_ln_b", c_void_p)]


class TextSaved(C.Structure):
    _fields_ = [("x_final", c_void_p), ("layers_host", C.POINTER(VitSavedLayer))]


class TextGrads(C.Structure):
    _fields_ = [("d_token_emb", c_void_p), ("d_pos_emb", c_void_p), ("d_final_ln_g", c_void_p), ("d_final_ln_b", c_void_p),
                ("layers_host", C.POINTER(VitLayerBwd))]


class RefinerBank(C.Structure):
    _fields_ = [("num_cells", c_int32), ("dim", c_int32), ("cell_off", c_void_p), ("proto_emb", c_void_p),
                ("proto_lnglat", c_void_p), ("proto_count", c_void_p), ("member_off", c_void_p),
                ("member_idx", c_void_p), ("data_emb", c_void_p), ("data_lnglat", c_void_p), ("proto_sqnorm", c_void_p), ("num_protos", c_int64), ("live_cells", c_int32)]


class PgCountries(C.Structure):
    _fields_ = [("verts", c_void_p), ("ring_off", c_void_p), ("part_ring_off", c_void_p), ("geom_part_off", c_void_p),
                ("num_verts", c_int64), ("num_rings", c_int64), ("num_parts", c_int64), ("num_geoms", c_int64),
                ("index", c_void_p), ("index_bytes", c_size_t), ("entries", c_void_p), ("num_entries", c_int64)]


class JpegInfo(C.Structure):
    _fields_ = [("status", c_int32), ("sof", c_int32), ("precision", c_int32), ("height", c_int32), ("width", c_int32),
                ("components", c_int32), ("component_id", c_int32 * 3), ("h_samp", c_int32 * 3), ("v_samp", c_int32 * 3),
                ("quant_table", c_int32 * 3), ("dc_table", c_int32 * 3), ("ac_table", c_int32 * 3),
                ("restart_interval", c_int32), ("num_segments", c_int32), ("table_mask", c_int32),
                ("scan_offset", c_int64), ("scan_bytes", c_int64), ("qt", (C.c_uint16 * 64) * 4),
                ("dc_bits", (C.c_uint8 * 16) * 4), ("ac_bits", (C.c_uint8 * 16) * 4), ("dc_vals", (C.c_uint8 * 256) * 4),
                ("ac_vals", (C.c_uint8 * 256) * 4)]


class JpegScan(C.Structure):
    _fields_ = [("components", c_int32), ("component", c_int32 * 3), ("ss", c_int32), ("se", c_int32), ("ah", c_int32),
                ("al", c_int32), ("restart_interval", c_int32), ("num_segments", c_int32), ("level", c_int32)]


class PngInfo(C.Structure):
    _fields_ = [("status", c_int32), ("width", c_int32), ("height", c_int32), ("bit_depth", c_int32),
                ("color_type", c_int32), ("channels", c_int32), ("bpp", c_int32), ("palette_entries", c_int32),
                ("idat_chunks", c_int32), ("row_bytes", c_int64), ("idat_offset", c_int64), ("zlib_bytes", c_int64),
                ("palette", (C.c_uint8 * 3) * 256)]


class GemmProblem(C.Structure):
    _fields_ = [("M", c_int32), ("N", c_int32), ("K", c_int32), ("a", c_void_p), ("lda", c_int32), ("w", c_void_p),
                ("ldw", c_int32), ("out", c_void_p), ("ldo", c_int32), ("bias", c_void_p), ("epilogue", c_int32),
                ("rowmap_div", c_int32), ("rowmap_mul", c_int32), ("rowmap_add", c_int32), ("operand_bf16", c_int32),
                ("resid", c_void_p), ("aux", c_void_p), ("mn_major", c_int32), ("stats", c_void_p), ("colsum", c_void_p),
                ("ln_eps", c_float)]


# name -> (restype, argtypes); must list every symbol declared in include/pigeon_b200.h
SIGNATURES = {
    "pg_abi_version": (c_int32, []),
    "pg_last_error": (C.c_char_p, []),
    "pg_device_sm_count": (c_int32, []),
    "pg_vit_create": (c_int32, [C.POINTER(VitConfig), C.POINTER(VitWeights), C.POINTER(c_void_p)]),
    "pg_vit_destroy": (None, [c_void_p]),
    "pg_vit_workspace_bytes": (c_size_t, [c_void_p, c_int32]),
    "pg_vit_forward": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "pg_vit_forward_cls": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p, c_void_p, c_void_p,
                                     c_void_p]),
    "pg_text_create": (c_int32, [C.POINTER(TextConfig), C.POINTER(TextWeights), C.POINTER(c_void_p)]),
    "pg_text_destroy": (None, [c_void_p]),
    "pg_text_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "pg_text_forward": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_size_t, c_void_p, c_void_p,
                                  c_void_p]),
    "pg_clip_project_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "pg_clip_project": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_float, c_void_p, c_int32, c_void_p,
                                  c_size_t, c_void_p, c_void_p]),
    "pg_clip_logits": (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_int32, c_float, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p]),
    "pg_vit_forward_train": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, C.POINTER(VitSaved), c_void_p, c_void_p]),
    "pg_vit_backward_workspace_bytes": (c_size_t, [c_void_p, c_int32]),
    "pg_vit_backward": (c_int32, [c_void_p, C.POINTER(VitSaved), c_void_p, c_int32, C.POINTER(VitGrads), c_void_p, c_size_t,
                                  c_void_p]),
    "pg_vit_backward_cls": (c_int32, [c_void_p, C.POINTER(VitSaved), c_void_p, c_int32, C.POINTER(VitGrads), c_void_p,
                                      c_size_t, c_void_p]),
    "pg_text_forward_train": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, C.POINTER(TextSaved), c_void_p,
                                        c_void_p]),
    "pg_text_backward_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "pg_text_backward": (c_int32, [c_void_p, C.POINTER(TextSaved), c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                                   C.POINTER(TextGrads), c_void_p, c_size_t, c_void_p]),
    "pg_clip_loss_grad_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "pg_clip_loss_grad": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_double, c_void_p, c_size_t, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pg_attention_f16_masked_lse": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                                              c_void_p]),
    "pg_attention_backward_masked": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_int32,
                                               c_int32, c_int32, c_void_p, c_size_t, c_void_p]),
    "pg_layernorm_f32": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_float, c_void_p]),
    "pg_gemm_ex": (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_int32,
                             c_int32, c_int32, c_int32, c_void_p]),
    "pg_gemm_tn": (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                             c_void_p]),
    "pg_gemm_problem_run": (c_int32, [C.POINTER(GemmProblem), c_void_p]),
    "pg_attention_f16_lse": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p]),
    "pg_attention_backward_workspace_bytes": (c_size_t, [c_int32, c_int32, c_int32]),
    "pg_attention_backward": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                        c_void_p, c_size_t, c_void_p]),
    "pg_layernorm_backward": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_int64,
                                        c_int32, c_float, c_void_p]),
    "pg_dgelu_bf16": (c_int32, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "pg_transpose_to_bf16": (c_int32, [c_void_p, c_int32, c_int64, c_void_p, c_int64, c_int64, c_int32, c_void_p]),
    "pg_head_pack_weight": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_void_p]),
    "pg_head_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "pg_head_forward": (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_int32, c_int32,
                                  c_void_p, c_size_t, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p]),
    "pg_head_loss": (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_double,
                               c_void_p, c_void_p, c_void_p]),
    "pg_preprocess_workspace_bytes": (c_size_t, [c_void_p, c_int32, c_int32]),
    "pg_preprocess_clip": (c_int32, [c_void_p, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p, c_int32,
                                     c_void_p]),
    "pg_jpeg_parse": (c_int32, [c_void_p, c_int64, C.POINTER(JpegInfo)]),
    "pg_jpeg_parse_multiscan": (c_int32, [c_void_p, c_int64, C.POINTER(JpegInfo)]),
    "pg_jpeg_scans": (c_int32, [c_void_p, c_int64, C.POINTER(JpegScan), c_int32]),
    "pg_jpeg_workspace_bytes": (c_size_t, [C.POINTER(JpegInfo), c_int32, c_int64]),
    "pg_jpeg_decode": (c_int32, [c_void_p, c_void_p, C.POINTER(JpegInfo), c_int32, c_void_p, c_void_p, c_size_t, c_void_p,
                                 c_void_p]),
    "pg_jpeg_set_schedule": (c_int32, [c_int32, c_int32]),
    "pg_jpeg_entropy_host": (c_int64, [c_void_p, c_void_p, C.POINTER(JpegInfo), c_int32, c_int32, c_void_p, c_void_p,
                                       c_void_p]),
    "pg_png_parse": (c_int32, [c_void_p, c_int64, C.POINTER(PngInfo)]),
    "pg_png_workspace_bytes": (c_size_t, [C.POINTER(PngInfo), c_int32, c_int64]),
    "pg_png_decode": (c_int32, [c_void_p, c_void_p, C.POINTER(PngInfo), c_int32, c_void_p, c_void_p, c_size_t, c_void_p,
                                c_void_p]),
    "pg_png_decode_host": (c_int64, [c_void_p, c_void_p, C.POINTER(PngInfo), c_int32, c_void_p, c_void_p]),
    "pg_head_loss_grad": (c_int32, [c_void_p, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_double,
                                    c_double, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pg_head_backward": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p, c_void_p,
                                   c_void_p, c_void_p]),
    "pg_adamw_step": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_double, c_double, c_double, c_double,
                                c_double, c_int64, c_double, c_void_p]),
    "pg_grad_norm_clip_workspace_bytes": (c_size_t, [c_int64]),
    "pg_grad_norm_clip": (c_int32, [c_void_p, c_int64, c_double, c_double, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "pg_adamw_hf_step": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_double, c_double, c_double, c_double,
                                   c_double, c_int64, c_double, c_void_p, c_void_p]),
    "pg_optics_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "pg_optics_xi": (c_int32, [c_void_p, c_int64, c_void_p, c_int32, c_int64, c_int32, c_double, c_void_p, c_size_t,
                               c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pg_country_index_bytes": (c_size_t, [c_int64, c_int64, c_int64]),
    "pg_country_index_build": (c_int32, [C.POINTER(PgCountries), c_void_p, c_void_p]),
    "pg_country_index_fill": (c_int32, [C.POINTER(PgCountries), c_void_p]),
    "pg_country_locate": (c_int32, [C.POINTER(PgCountries), c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                                    c_void_p]),
    "pg_geo_metrics_workspace_bytes": (c_size_t, [c_int64]),
    "pg_geo_metrics": (c_int32, [c_void_p, c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int32, c_void_p,
                                 c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "pg_refiner_workspace_bytes": (c_size_t, [c_int64, c_int32, c_int32, c_int32]),
    "pg_refiner_forward": (c_int32, [C.POINTER(RefinerBank), c_void_p, c_int64, c_int32, c_void_p, c_void_p, c_void_p,
                                     c_int32, c_int32, c_float, c_double, c_void_p, c_size_t, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pg_refiner_set_schedule": (c_int32, [c_int32]),
    "pg_head_set_fused": (c_int32, [c_int32]),
    "pg_gemm_set_schedule": (c_int32, [c_int32]),
    "pg_refiner_bank_sqnorm": (c_int32, [c_void_p, c_int64, c_int32, c_void_p, c_void_p]),
    "pg_refiner_scan": (c_int32, [C.POINTER(RefinerBank), c_void_p, c_int64, c_int32, c_void_p, c_int32, c_int32, c_void_p,
                                  c_size_t, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pg_refiner_finalize": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int64, c_int32,
                                      c_float, c_double, c_void_p, c_void_p, c_void_p, c_void_p]),
    "pg_bank_build": (c_int32, [c_void_p, c_int64, c_int32, c_int32, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "pg_profile_begin": (None, []),
    "pg_profile_end": (c_int32, []),
    "pg_profile_read": (None, [C.POINTER(C.c_char_p), C.POINTER(c_float), C.POINTER(c_int32), c_int32]),
    "pg_nccl_unique_id": (c_int32, [c_void_p]),
    "pg_nccl_comm_create": (c_int32, [c_void_p, c_int32, c_int32, C.POINTER(c_void_p)]),
    "pg_nccl_comm_destroy": (None, [c_void_p]),
    "pg_allgather_embeddings": (c_int32, [c_void_p, c_void_p, c_void_p, C.c_size_t, c_void_p]),
    "pg_gemm_f16": (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_int32, c_int32,
                              c_int32, c_int32, c_void_p]),
    "pg_layernorm_f16": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_float, c_void_p]),
    "pg_attention_f16": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_void_p]),
    "pg_attention_f16_masked": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "pg_attention_f16_variant": (c_int32, [c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32,
                                           c_void_p]),
}

ABI_VERSION = 4   # == PG_ABI_VERSION in include/pigeon_b200.h; bumped whenever a signature or struct changes

EPI_F16_BIAS, EPI_F16_BIAS_QGELU, EPI_F32_BIAS_RESID, EPI_F32_BIAS = 0, 1, 2, 3
EPI_F32_ROWMAP, EPI_BF16_DGELU, EPI_F16_BIAS_QGELU_SAVE, EPI_F32_BIAS_RESID_STATS, EPI_F16_LN_BIAS, EPI_F16_LN_BIAS_QGELU = \
    4, 5, 6, 7, 8, 9

_lib: Optional[C.CDLL] = None


def lib_path() -> Path:
    return _build.LIB_PATH


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load (building first if needed) the shared object and type every entry point."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if build_if_missing:
        # build() is content-hash idempotent: it returns at once when the binary matches the sources and rebuilds a stale
        # one (the .so is git-ignored, so a pull can leave an old binary beside new sources).  Without nvcc an existing,
        # hash-matching binary is used as it is; a stale or missing one is an error, never a silent mismatch.
        try:
            _build.build()
        except RuntimeError as e:
            if not path.exists() or not _build.is_current():
                raise PigeonB200Error(f"{path} is missing or older than its sources and cannot be rebuilt: {e}") from e
    elif not path.exists():
        raise PigeonB200Error(f"{path} is missing: run `python -m pigeon_b200._build` (needs nvcc)")
    try:
        lib = C.CDLL(str(path))
    except OSError as e:  # pragma: no cover - environment problem
        raise PigeonB200Error(f"cannot load {path}: {e}") from e
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise PigeonB200Error(f"{path} does not export {name}; rebuild with `python -m pigeon_b200._build --force`") from e
        fn.restype = res
        fn.argtypes = args
    if lib.pg_abi_version() != ABI_VERSION:
        raise PigeonB200Error(f"ABI version mismatch: library {lib.pg_abi_version()} != binding {ABI_VERSION}")
    _lib = lib
    return lib


def check(status: int, what: str) -> None:
    if status != 0:
        msg = load().pg_last_error()
        raise PigeonB200Error(f"{what} failed: {msg.decode() if msg else 'unknown error'}")


def ptr(t) -> Optional[int]:
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def current_stream_ptr() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
