"""ctypes binding of include/b200clip.h.  The library is required: no fallback of any kind."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "lib", "libb200clip.so")


class B200Error(RuntimeError):
    """Raised when a b200clip C-ABI call returns a negative status."""


def library_path():
    return _LIB_PATH


def _load():
    if not os.path.exists(_LIB_PATH):
        raise ImportError(
            "b200clip CUDA library missing: %s — build it with `python clip-retrieval_b200/build.py` "
            "(or __graft_entry__.build()); there is no CPU fallback." % _LIB_PATH
        )
    return C.CDLL(_LIB_PATH)


lib = _load()


class SynthSpecC(C.Structure):
    _fields_ = [
        ("seed", C.c_uint64),
        ("clustered", C.c_int32),
        ("centroid_seed", C.c_uint64),
        ("nlist", C.c_int32),
        ("cw", C.c_int32),
        ("nw", C.c_int32),
    ]


class TowerConfigC(C.Structure):
    _fields_ = [("width", C.c_int32), ("layers", C.c_int32), ("heads", C.c_int32), ("mlp", C.c_int32)]


class ClipConfigC(C.Structure):
    _fields_ = [
        ("embed_dim", C.c_int32),
        ("image_size", C.c_int32),
        ("patch", C.c_int32),
        ("vision", TowerConfigC),
        ("context_length", C.c_int32),
        ("vocab_size", C.c_int32),
        ("text", TowerConfigC),
        ("quick_gelu", C.c_int32),
        ("max_batch", C.c_int32),
    ]


class ResNetConfigC(C.Structure):
    _fields_ = [("layers", C.c_int32 * 4), ("width", C.c_int32), ("heads", C.c_int32)]


class ConvNeXtConfigC(C.Structure):
    _fields_ = [("depths", C.c_int32 * 4), ("dims", C.c_int32 * 4), ("head_mlp", C.c_int32), ("eps", C.c_float)]


class TextEncoderConfigC(C.Structure):
    _fields_ = [
        ("layers", C.c_int32),
        ("width", C.c_int32),
        ("heads", C.c_int32),
        ("ffn", C.c_int32),
        ("vocab_size", C.c_int32),
        ("max_positions", C.c_int32),
        ("type_vocab_size", C.c_int32),
        ("position_offset", C.c_int32),
        ("layer_norm_eps", C.c_float),
        ("out_dim", C.c_int32),
        ("proj_bias", C.c_int32),
        ("max_batch", C.c_int32),
        ("max_tokens", C.c_int32),
    ]


class TensorViewC(C.Structure):
    _fields_ = [
        ("name", C.c_char_p),
        ("data", C.c_void_p),
        ("dtype", C.c_int32),
        ("ndim", C.c_int32),
        ("shape", C.c_int64 * 4),
    ]


class GemmEpilogueC(C.Structure):
    _fields_ = [
        ("bias", C.c_void_p),
        ("residual", C.c_void_p),
        ("res_ld", C.c_int64),
        ("res_row_mod", C.c_int32),
        ("res_row_off", C.c_int32),
        ("out_ld", C.c_int64),
        ("out_group", C.c_int32),
        ("act", C.c_int32),
        ("reserved0", C.c_void_p),
        ("reserved1", C.c_void_p),
        ("reserved2", C.c_int32),
        ("reserved3", C.c_void_p),
    ]


_vp, _i, _i64, _fp =C.c_void_p, C.c_int, C.c_int64, C.POINTER(C.c_float)

# name -> (restype, argtypes).  Kept in one table so tests can check every symbol of the header.
PROTOTYPES = {
    "b200_last_error": (C.c_char_p, []),
    "b200_version": (C.c_char_p, []),
    "b200_launch_count": (_i64, []),
    "b200_synth_rows_f16": (_i, [_vp, _i64, _i, _i64, C.POINTER(SynthSpecC), _vp]),
    "b200_synth_rows_f32": (_i, [_vp, _i64, _i, _i64, C.POINTER(SynthSpecC), _vp]),
    "b200_index_create_flat": (_i, [_i, _i, C.POINTER(_vp)]),
    "b200_index_create_ivfflat": (_i, [_i, _i, _vp, _i, C.POINTER(_vp)]),
    "b200_index_create_ivfpq": (_i, [_i, _i, _i, _i, _vp, _vp, _i, C.POINTER(_vp)]),
    "b200_index_add_codes": (_i, [_vp, _vp, _i64, _i, _vp]),
    "b200_index_set_pretransform": (_i, [_vp, _i, _vp, _vp]),
    "b200_index_pq_m": (_i, [_vp]),
    "b200_index_set_host_lists": (_i, [_vp, _i, _vp, _vp, _vp]),
    "b200_index_set_stream_arena": (_i, [_vp, C.c_size_t]),
    "b200_index_last_stream_stats": (_i, [_vp, _vp]),
    "b200_ids_map_device": (_i, [_vp, _i64, _vp, _i64, _vp, _i, _vp]),
    "b200_index_encode_device": (_i, [_vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "b200_pq_train_f32": (_i, [_vp, _i64, _i, _i, _i, C.c_uint64, _vp, _vp, _i]),
    "b200_opq_train_f32": (_i, [_vp, _i64, _i, _i, _i, _i, _i, _i, C.c_uint64, _vp, _vp, _vp, _i]),
    "b200_rows_pretransform_device": (_i, [_vp, _i64, _i, _vp, _vp, _i, _vp, _i, _i, _vp]),
    "b200_opq_cross_f32_device": (_i, [_vp, _i64, _i, _vp, _vp, _i, _i, _vp, _i, _vp]),
    "b200_opq_polar_f32_device": (_i, [_vp, _i, _i, _vp, _i, _vp]),
    "b200_index_get_quantizer": (_i, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "b200_index_copy_rows": (_i, [_vp, _i64, _i64, _vp, _vp]),
    "b200_index_destroy": (_i, [_vp]),
    "b200_index_reserve": (_i, [_vp, _i64]),
    "b200_index_add_f16": (_i, [_vp, _vp, _i64, _i]),
    "b200_index_add_f32": (_i, [_vp, _vp, _i64, _i]),
    "b200_index_add_assigned_f16": (_i, [_vp, _vp, _i64, _i, _vp]),
    "b200_index_add_synthetic": (_i, [_vp, _i64, _i64, C.POINTER(SynthSpecC)]),
    "b200_index_finalize": (_i, [_vp]),
    "b200_index_ntotal": (_i64, [_vp]),
    "b200_index_d": (_i, [_vp]),
    "b200_index_nlist": (_i, [_vp]),
    "b200_index_set_id_base": (_i, [_vp, _i64]),
    "b200_index_set_nprobe": (_i, [_vp, _i]),
    "b200_index_get_nprobe": (_i, [_vp]),
    "b200_index_set_tensor_scan": (_i, [_vp, _i]),
    "b200_index_ivf_lists": (_i, [_vp, _vp, _vp]),
    "b200_index_search": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    "b200_index_search_device": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "b200_index_range_search": (_i, [_vp, _vp, C.c_float, _i64, _vp, _vp, C.POINTER(_i64)]),
    "b200_index_reconstruct_device": (_i, [_vp, _vp, _i64, _vp, _vp]),
    "b200_topk_merge_device": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _i, _vp]),
    "b200_index_last_scan_ms": (_i, [_vp, C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "b200_topk_merge_packed_device": (_i, [_vp, _i, C.c_size_t, _i, _i, _vp, _vp, _i, _vp]),
    "b200_sharded_create": (_i, [C.POINTER(_vp), _i, C.POINTER(_vp)]),
    "b200_sharded_destroy": (_i, [_vp]),
    "b200_sharded_peer_mode": (_i, [_vp]),
    "b200_sharded_search": (_i, [_vp, C.POINTER(_vp), _vp, _i, _i, _vp, _vp]),
    "b200_nccl_comm_init_all": (_i, [_i, C.POINTER(C.c_int), C.POINTER(_vp)]),
    "b200_nccl_comm_destroy": (_i, [_vp]),
    "b200_clip_create": (_i, [C.POINTER(ClipConfigC), _i, C.POINTER(_vp)]),
    "b200_clip_create_resnet": (_i, [C.POINTER(ClipConfigC), C.POINTER(ResNetConfigC), _i, C.POINTER(_vp)]),
    "b200_clip_create_siglip": (_i, [C.POINTER(ClipConfigC), _i, C.POINTER(_vp)]),
    "b200_clip_create_convnext": (_i, [C.POINTER(ClipConfigC), C.POINTER(ConvNeXtConfigC), _i, C.POINTER(_vp)]),
    "b200_clip_destroy": (_i, [_vp]),
    "b200_clip_load_weights": (_i, [_vp, C.POINTER(TensorViewC), _i]),
    "b200_clip_encode_image_device": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp]),
    "b200_clip_encode_text_device": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp]),
    "b200_clip_encode_image": (_i, [_vp, _vp, _i, _vp, _i, _i]),
    "b200_clip_encode_text": (_i, [_vp, _vp, _i, _vp, _i, _i]),
    "b200_clip_last_timing": (_i, [_vp, C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "b200_clip_set_profiling": (_i, [_vp, _i]),
    "b200_layernorm_bf16_device": (_i, [_vp, _vp, _vp, _vp, _i64, _i, _i, _vp]),
    "b200_attention_bf16_device": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200_vision_front_bf16_device": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _vp, _i, _vp]),
    "b200_text_embed_bf16_device": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200_token_argmax_device": (_i, [_vp, _i, _i, _vp, _i, _vp]),
    "b200_pool_ln_proj_device": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp]),
    "b200_gemm_bf16_device": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200_gemm_bf16_ex_device": (_i, [_vp, _vp, _vp, _i, _i, _i, C.POINTER(GemmEpilogueC), _i, _i, _i, _vp]),
    "b200_conv_bf16_device": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _i, _vp, C.POINTER(GemmEpilogueC), _i, _i, _vp]),
    "b200_stem_gather_device": (_i, [_vp, _i, _i, _vp, _i, _vp]),
    "b200_avgpool_bf16_device": (_i, [_vp, _i, _i, _i, _i, _i, _vp, _i, _vp]),
    "b200_attnpool_tokens_device": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp]),
    "b200_latent_pool_attention_device": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _i, _vp]),
    "b200_pool_last_ln_proj_bias_device": (_i, [_vp, _i, _i, _i, _vp, _vp, C.c_float, _vp, _vp, _i, _vp, _vp, _i, _i, _i,
                                                _vp]),
    "b200_dwconv7_ln_bf16_device": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, C.c_float, _vp, _i, _vp]),
    "b200_ln_s2d_bf16_device": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, C.c_float, _vp, _i, _vp]),
    "b200_convnext_head_device": (_i, [_vp, _i, _i, _i, _vp, _vp, C.c_float, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _vp,
                                       _i, _i, _i, _vp]),
    "b200_index_last_hi_only_fallbacks": (_i, [_vp]),
    "b200_index_last_scan_plan": (_i, [_vp, _vp]),
    "b200_kmeans_train_f16": (_i, [_vp, _i64, _i, _i, _i, C.c_uint64, _i, _vp, _vp, _i]),
    "b200_dedup_device": (_i, [_vp, _i, _i, C.c_float, _vp, _vp, _vp, C.c_size_t, _i, _vp]),
    "b200_prompt_argmax_device": (_i, [_vp, _i, _i, _vp, _i, _i, _vp, _i, _vp]),
    "b200_preproc_create": (_i, [_i, C.POINTER(C.c_float), C.POINTER(C.c_float), _i, C.POINTER(_vp)]),
    "b200_preproc_create_mode": (_i, [_i, C.POINTER(C.c_float), C.POINTER(C.c_float), _i, _i, C.POINTER(_vp)]),
    "b200_preproc_destroy": (_i, [_vp]),
    "b200_preproc_run": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _vp]),
    "b200_jpeg_create": (_i, [_i, C.POINTER(_vp)]),
    "b200_jpeg_destroy": (_i, [_vp]),
    "b200_jpeg_info": (_i, [_vp, _vp, _vp, _i, _vp, _vp]),
    "b200_jpeg_decode": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp]),
    "b200_mlp_create": (_i, [_i, _vp, _vp, _i, C.POINTER(_vp)]),
    "b200_mlp_destroy": (_i, [_vp]),
    "b200_mlp_load_layer": (_i, [_vp, _i, _vp, _vp]),
    "b200_mlp_forward_device": (_i, [_vp, _vp, _i, _vp, _vp]),
    "b200_text_encoder_create": (_i, [C.POINTER(TextEncoderConfigC), _i, C.POINTER(_vp)]),
    "b200_text_encoder_create_mlp": (_i, [C.POINTER(TextEncoderConfigC), _i, _i, C.POINTER(_vp)]),
    "b200_text_encoder_destroy": (_i, [_vp]),
    "b200_text_encoder_load_weights": (_i, [_vp, C.POINTER(TensorViewC), _i]),
    "b200_text_encoder_encode_device": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _i, _vp]),
    "b200_text_encoder_encode": (_i, [_vp, _vp, _vp, _i, _i, _vp, _i, _i]),
    "b200_text_encoder_last_timing": (_i, [_vp, C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "b200_text_encoder_set_profiling": (_i, [_vp, _i]),
    "b200_layernorm_eps_bf16_device": (_i, [_vp, _vp, _vp, _vp, _i64, _i, C.c_float, _i, _vp]),
    "b200_attention_len_bf16_device": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200_text_lengths_device": (_i, [_vp, _i, _i, _i64, _vp, _vp]),
    "b200_mean_mlp_head_device": (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "b200_mean_proj_head_device": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp]),
    "b200_encoder_embed_bf16_device": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp, C.c_float, _vp, _i, _i, _i, _i, _i, _vp]),
}

for _name, (_res, _args) in PROTOTYPES.items():
    _fn = getattr(lib, _name)  # AttributeError here = the library is stale; rebuild
    _fn.restype = _res
    _fn.argtypes = _args


def check(status, what=""):
    if status != 0:
        msg = lib.b200_last_error()
        raise B200Error("%s failed (status %d): %s" % (what or "b200clip call", status, (msg or b"").decode()))


def launch_count():
    return int(lib.b200_launch_count())
