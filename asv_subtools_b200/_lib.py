"""ctypes binding of libxvb200.so (C ABI: include/xvb200.h).  No fallback: if the shared library
is missing or a call fails, an exception is raised."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# XVB_LIB names another build of the same library (tools/tile_timeline.py loads the timeline build through it)
LIB_PATH = os.environ.get("XVB_LIB") or os.path.join(_HERE, "libxvb200.so")

RELU, BN, SIGMOID, TANH, SWISH = 1, 2, 4, 8, 16
POOL_ATTENTION, POOL_XI_POSTMEAN, POOL_XI_POSTDIST = 1, 2, 3   # xvb_extractor_set_attention_pooling kinds
ACT_NONE, ACT_RELU, ACT_SWISH, ACT_TANH = 0, 1, 2, 3


class TdnnArgs(C.Structure):
    """xvb_tdnn_args_t (include/xvb200.h)."""
    _fields_ = [("x_hi", C.c_void_p), ("x_lo", C.c_void_p), ("ldx", C.c_int64),
                ("x2_hi", C.c_void_p), ("x2_lo", C.c_void_p), ("ldx2", C.c_int64),
                ("w_hi", C.c_void_p), ("w_lo", C.c_void_p),
                ("bias", C.c_void_p), ("bn_scale", C.c_void_p), ("bn_shift", C.c_void_p),
                ("row_bias", C.c_void_p), ("utt_bias", C.c_void_p), ("ld_utt_bias", C.c_int64),
                ("flags", C.c_int), ("context_host", C.POINTER(C.c_int)), ("ntaps", C.c_int),
                ("y_hi", C.c_void_p), ("y_lo", C.c_void_p), ("ldy", C.c_int64),
                ("y_f32", C.c_void_p), ("ldyf", C.c_int64),
                ("B", C.c_int), ("T", C.c_int), ("Cin", C.c_int), ("Cout", C.c_int),
                ("pool_partial", C.c_void_p), ("x_batch_stride", C.c_int64), ("groups", C.c_int),
                ("lengths", C.c_void_p)]
MAX_TAPS = 16


class Conv2dArgs(C.Structure):
    """xvb_conv2d_args_t (include/xvb200.h)."""
    _fields_ = [("x_hi", C.c_void_p), ("x_lo", C.c_void_p), ("w_hi", C.c_void_p), ("w_lo", C.c_void_p),
                ("B", C.c_int), ("T", C.c_int), ("F", C.c_int), ("Cin", C.c_int), ("Cout", C.c_int),
                ("ksize", C.c_int), ("stride", C.c_int),
                ("scale", C.c_void_p), ("shift", C.c_void_p), ("res_hi", C.c_void_p), ("res_lo", C.c_void_p),
                ("relu", C.c_int), ("y_hi", C.c_void_p), ("y_lo", C.c_void_p), ("y_f32", C.c_void_p),
                ("scale2", C.c_void_p), ("shift2", C.c_void_p), ("y2_hi", C.c_void_p), ("y2_lo", C.c_void_p),
                ("stride_t", C.c_int), ("lengths", C.c_void_p)]


class LayerNormArgs(C.Structure):
    """xvb_layer_norm_args_t (include/xvb200.h)."""
    _fields_ = [("rows", C.c_int64), ("C", C.c_int), ("eps", C.c_float),
                ("x", C.c_void_p), ("ldx", C.c_int64),
                ("delta", C.c_void_p), ("ld_delta", C.c_int64), ("delta_scale", C.c_float),
                ("table", C.c_void_p), ("table_rows", C.c_int),
                ("x_out", C.c_void_p), ("ld_x_out", C.c_int64),
                ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("second", C.c_int),
                ("gamma2", C.c_void_p), ("beta2", C.c_void_p),
                ("act", C.c_int),
                ("y_hi", C.c_void_p), ("y_lo", C.c_void_p), ("ldy", C.c_int64),
                ("y_f32", C.c_void_p), ("ldyf", C.c_int64)]


class ConformerConfig(C.Structure):
    """xvb_conformer_config_t (include/xvb200.h)."""
    _fields_ = [(n, C.c_int) for n in ("feat_dim", "subsampling", "D", "H", "linear_units", "blocks", "conv_kernel", "pos",
                                       "rotary_value", "softmax_plus", "act", "cm_norm", "out_dim", "out_norm",
                                       "pool_hidden", "fc1", "position")]


class CamPPConfig(C.Structure):
    """xvb_campp_config_t (include/xvb200.h)."""
    _fields_ = [(n, C.c_int) for n in ("feat_dim", "embd_dim", "init_channels", "growth_rate", "bn_size")]


class RepVGGConfig(C.Structure):
    """xvb_repvgg_config_t (include/xvb200.h)."""
    _fields_ = [("feat_dim", C.c_int), ("ksize", C.c_int), ("num_blocks", C.c_int * 4), ("strides", C.c_int * 5),
                ("widths", C.c_int * 5), ("pooling_eps", C.c_float)]


class XvbError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "asv_subtools_b200: native library {} not found -- build it with "
            "`python -c 'import __graft_entry__ as g; g.build()'` (make -C asv_subtools_b200/csrc). "
            "There is no Python/CPU fallback.".format(LIB_PATH))
    return C.CDLL(LIB_PATH)


lib = _load()

_p = C.c_void_p
_i = C.c_int
_i64 = C.c_int64
_f = C.c_float
_ip = C.POINTER(C.c_int)

# name -> (restype, argtypes); every symbol declared in include/xvb200.h must appear here
SIGNATURES = {
    "xvb_version": (_i, []),
    "xvb_last_error": (C.c_char_p, []),
    "xvb_device_check": (_i, []),
    "xvb_split_f32": (_i, [_p, _i64, _i, _i64, _p, _p, _i64, _p]),
    "xvb_packed_weight_elems": (_i64, [_i, _i, _i]),
    "xvb_pack_tdnn_weight": (_i, [_p, _i, _i, _i, _i, _ip, _i, _p, _p, _p]),
    "xvb_tdnn_affine": (_i, [_p, _p, _i64, _p, _p, _p, _p, _p, _i, _ip, _i, _p, _p, _i64, _p, _i64, _i, _i, _i, _i, _p]),
    "xvb_tdnn_affine_simt": (_i, [_p, _i64, _p, _i, _i, _p, _p, _p, _i, _ip, _i, _p, _i64, _i, _i, _i, _i, _p]),
    "xvb_stats_pool": (_i, [_p, _i64, _i, _i, _i, _f, _p, _p, _p, _i64, _p]),
    "xvb_stats_pool_ex": (_i, [_p, _i64, _i, _i, _i, _f, _i, _p, _p, _p, _i64, _p]),
    "xvb_tdnn_affine_ex": (_i, [_p, _p]),
    "xvb_split_frames": (_i, [_p, _i, _i, _i, _p, _p, _i64, _i, _i, _p]),
    "xvb_split_frames_lengths": (_i, [_p, _i, _i, _i, _p, _p, _i64, _i, _i, _p, _p]),
    "xvb_pool_partial_blocks": (_i, [_i, _i, _ip]),
    "xvb_pool_finalize": (_i, [_p, _i, _i, _i, _i, _i, _f, _i, _p, _p, _p, _i64, _p]),
    "xvb_stats_pool_lengths": (_i, [_p, _i64, _i, _i, _i, _f, _i, _p, _p, _p, _p, _i64, _p]),
    "xvb_extractor_set_fused_pooling": (_i, [_p, _i]),
    "xvb_plane_mean": (_i, [_p, _p, _i64, _i, _i, _i, _p, _p, _p, _i64, _p]),
    "xvb_plane_mean_lengths": (_i, [_p, _p, _i64, _i, _i, _i, _p, _i, _p, _p, _p, _i64, _p]),
    "xvb_res2net_block": (_i, [_p, _p, _i64, _p, _p, _p, _p, _p, _i, _i, _p, _p, _i64, _i, _i, _p]),
    "xvb_res2net_block_ex": (_i, [_p, _p, _i64, _p, _p, _p, _p, _p, _i, _i, _p, _p, _i64, _i, _i, _i, _p]),
    "xvb_copy_rows": (_i, [_p, _i64, _p, _i64, _i64, _i64, _p]),
    "xvb_se_apply": (_i, [_p, _p, _i64, _p, _p, _i64, _p, _p, _p, _i64, _p, _p, _i64, _i, _i, _i, _p]),
    "xvb_attn_stats_pool": (_i, [_p, _i64, _p, _i64, _i, _i, _i, _f, _p, _p, _p, _i64, _p]),
    "xvb_attn_stats_pool_lengths": (_i, [_p, _i64, _p, _i64, _i, _i, _i, _f, _p, _p, _p, _p, _i64, _p]),
    "xvb_vad_energy": (_i, [_p, _p, _i, _i, _f, _f, _i, _f, _p, _p, _p]),
    "xvb_cmn": (_i, [_p, _p, _i, _i, _i, _p, _p]),
    "xvb_select_frames": (_i, [_p, _p, _p, _p, _i, _i, _p, _p]),
    "xvb_center_length_norm": (_i, [_p, _p, _p, _i64, _i, _p]),
    "xvb_column_mean": (_i, [_p, _i64, _i, _p, _p]),
    "xvb_cosine_trials": (_i, [_p, _p, _i, _p, _p, _i64, _p, _p]),
    "xvb_speaker_mean": (_i, [_p, _i, _p, _p, _i, _p, _p]),
    "xvb_ipc_alloc": (_i, [_p, C.c_size_t]),
    "xvb_ipc_free": (_i, [_p]),
    "xvb_ipc_export": (_i, [_p, _p]),
    "xvb_ipc_open": (_i, [_p, _p]),
    "xvb_ipc_close": (_i, [_p]),
    "xvb_scatter_rows": (_i, [_p, _i64, _i, _p, _i, _i64, _i64, _p]),
    "xvb_extractor_set_gather": (_i, [_p, _p, _i, _i64, _i64]),
    "xvb_ecapa_set_gather": (_i, [_p, _p, _i, _i64, _i64]),
    "xvb_lde_pool": (_i, [_p, _i64, _i, _i, _i, _p, _i, _p, _p, _p, _p, _p, _i64, _p]),
    "xvb_small_affine": (_i, [_p, _i64, _p, _i, _i, _i, _p, _p, _p, _i, _p, _i64, _p, _p, _i64, _p]),
    "xvb_attn_head_stats_pool": (_i, [_p, _i64, _i, _p, _i64, _i, _i, _i, _i, _i, _f, _i, _p, _p, _p, _i64, _p]),
    "xvb_attn_head_stats_pool_prior": (_i, [_p, _i64, _i, _p, _i64, _i, _i, _i, _i, _i, _f, _i, _p, _p, _i, _p, _p, _p, _i64, _p]),
    "xvb_attn_head_stats_pool_lengths": (_i, [_p, _i64, _i, _p, _i64, _i, _i, _i, _i, _i, _f, _i, _p, _p, _i, _p, _p, _p, _p,
                                              _i64, _p]),
    "xvb_attn_head_stats_pool_mq": (_i, [_p, _i64, _i, _p, _i64, _i, _i, _i, _i, _i, _i, _i, _f, _i, _p, _p, _p, _i64, _p]),
    "xvb_tdnn_grouped_fits": (_i, [_i, _i, _i]),
    "xvb_topn_mean_std": (_i, [_p, _i64, _i64, _i, _i, _p, _p, _p]),
    "xvb_topn_mean_std_ddof": (_i, [_p, _i64, _i64, _i, _i, _i, _p, _p, _p]),
    "xvb_snorm_trials": (_i, [_p, _p, _p, _i64, _p, _p, _p, _p, _p, _p]),
    "xvb_bilinear_trials": (_i, [_p, _p, _i, _p, _p, _i64, _p, _p, _p, _p]),
    "xvb_project": (_i, [_p, _i64, _i, _p, _i, _p, _p]),
    "xvb_cosine_matrix": (_i, [_p, _i64, _p, _i64, _i, _p, _i64, _p]),
    "xvb_plda_terms": (_i, [_p, _i64, _i, _p, _p, _p, _p]),
    "xvb_plda_matrix": (_i, [_p, _i64, _p, _i64, _i, _p, _p, _p, _p, _i64, _p]),
    "xvb_topn_indices": (_i, [_p, _i64, _i64, _i, _i, _p, _p]),
    "xvb_snorm_cross_trials": (_i, [_p, _p, _p, _i64, _p, _i64, _p, _i64, _p, _p, _i, _p, _p]),
    "xvb_matmul_nt": (_i, [_p, _i64, _p, _i64, _i, _p, _p, _p, _i64, _p]),
    "xvb_center_rows_transposed": (_i, [_p, _p, _p, _p, _i64, _i, _p, _i64, _p]),
    "xvb_plda_em_rows": (_i, [_p, _p, _p, _p, _i, _i, _p, _p, _i64, _p]),
    "xvb_plda_normalize_rows": (_i, [_p, _p, _p, _i64, _i, _i, _p]),
    "xvb_plda_llr_operands": (_i, [_p, _p, _p, _i64, _i, _i, _p, _p, _p]),
    "xvb_trial_histogram": (_i, [_p, _i64, _p, _p, _i64, _p, _i, _p, _p, _i, _i, _i, _f, _f, _i, _p, _p]),
    "xvb_topk_merge": (_i, [_p, _i64, _i64, _i64, _i64, _i, _p, _p, _p, _p]),
    "xvb_retrieve_topk_slab_bytes": (_i64, [_i64, _i64]),
    "xvb_retrieve_topk": (_i, [_p, _i64, _p, _i64, _i, _p, _p, _i, _p, _i64, _p, _p, _p]),
    "xvb_conv2d": (_i, [_p, _p]),
    "xvb_conv2d_head": (_i, [_p, _i, _i, _i, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "xvb_conv2d_taps": (_i, [_p, _ip, _i, _p]),
    "xvb_conv2d_head_lengths": (_i, [_p, _i, _i, _i, _p, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "xvb_conv2d_head_k": (_i, [_p, _i, _i, _i, _p, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "xvb_conv2d_valid": (_i, [_p, _p]),
    "xvb_subsample_head": (_i, [_p, _i, _i, _i, _p, _p, _i, _p, _p, _p]),
    "xvb_subsample_head_stride": (_i, [_p, _i, _i, _i, _p, _p, _i, _i, _p, _p, _p]),
    "xvb_subsample_head_lengths": (_i, [_p, _i, _i, _i, _p, _p, _p, _i, _i, _p, _p, _p]),
    "xvb_layer_norm": (_i, [_p, _p]),
    "xvb_rope_attention": (_i, [_p, _i64, _i, _i, _i, _i, _p, _i, _f, _p, _p, _i64, _p]),
    "xvb_rope_attention_lengths": (_i, [_p, _i64, _i, _i, _i, _i, _p, _i, _p, _p, _i, _p, _p, _i64, _p]),
    "xvb_conv_module": (_i, [_p, _i64, _i, _i, _i, _p, _p, _i, _p, _p, _i, _f, _i, _p, _p, _i64, _p]),
    "xvb_bn_relu_planes": (_i, [_p, _p, _i64, _i64, _i, _p, _p, _p, _p, _i64, _p]),
    "xvb_cam_gate": (_i, [_p, _p, _i64, _i, _i, _i, _i, _p, _p, _i, _p, _p, _i, _p, _p]),
    "xvb_cam_gate_lengths": (_i, [_p, _p, _i64, _i, _i, _i, _i, _p, _p, _i, _p, _p, _i, _p, _p, _p]),
    "xvb_seg_gate_apply": (_i, [_p, _p, _i64, _p, _p, _i64, _p, _i, _p, _p, _i64, _i, _i, _i, _p]),
    "xvb_se_residual": (_i, [_p, _p, _p, _p, _p, _i, _i64, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p]),
    "xvb_se_residual_lengths": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p]),
    "xvb_extractor_create": (_i, [C.POINTER(_p), _i]),
    "xvb_extractor_add_frame_layer": (_i, [_p, _i, _ip, _i, _p, _p, _p, _p, _i]),
    "xvb_extractor_add_segment_layer": (_i, [_p, _i, _p, _p, _p, _p, _i]),
    "xvb_extractor_set_attention_pooling": (_i, [_p, _i, _i, _i, _i, _p, _p]),
    "xvb_extractor_add_attention_layer": (_i, [_p, _i, _ip, _i, _p, _p, _p, _p, _i]),
    "xvb_extractor_finalize": (_i, [_p, _f]),
    "xvb_extractor_embed_dim": (_i, [_p]),
    "xvb_extractor_extract": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_extractor_extract_lengths": (_i, [_p, _p, _p, _i, _i, _p, _p]),
    "xvb_extractor_extract_host": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_extractor_submit_host": (_i, [_p, _p, _i, _i, _p, _i, _p]),
    "xvb_extractor_wait": (_i, [_p, _i]),
    "xvb_extractor_extract_shard": (_i, [_p, _p, C.c_int64, _i, _i, _p, _p]),
    "xvb_extractor_extract_shard_host": (_i, [_p, _p, C.c_int64, _i, _i, _p, _p]),
    "xvb_extractor_set_profiling": (_i, [_p, _i]),
    "xvb_extractor_kernel_times": (_i, [_p, C.POINTER(C.c_float), _i]),
    "xvb_extractor_last_launches": (_i, [_p]),
    "xvb_extractor_debug_f32": (_p, [_p, _i]),
    "xvb_extractor_destroy": (None, [_p]),
    "xvb_fbank_default_opts": (None, [_p]),
    "xvb_fbank_create": (_i, [C.POINTER(_p), _p]),
    "xvb_fbank_dim": (_i, [_p]),
    "xvb_fbank_num_frames": (_i64, [_p, _i64]),
    "xvb_fbank_compute": (_i, [_p, _p, _p, _p, _i, _i64, _p, _p]),
    "xvb_fbank_destroy": (None, [_p]),
    "xvb_ecapa_create": (_i, [C.POINTER(_p), _i, _i, _i, _i, _i]),
    "xvb_ecapa_set_mqmha": (_i, [_p, _i, _i, _i, _i, _i, _i, _i]),
    "xvb_ecapa_set_chained": (_i, [_p, _i]),
    "xvb_ecapa_set_attention": (_i, [_p, _i, _f]),
    "xvb_ecapa_set_layer": (_i, [_p, C.c_char_p, _i, _i, _ip, _i, _p, _p, _p, _p, _i]),
    "xvb_ecapa_finalize": (_i, [_p]),
    "xvb_ecapa_embed_dim": (_i, [_p]),
    "xvb_ecapa_feat_dim": (_i, [_p]),
    "xvb_ecapa_extract": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_ecapa_extract_host": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_ecapa_extract_shard": (_i, [_p, _p, C.c_int64, _i, _i, _p, _p]),
    "xvb_ecapa_extract_shard_host": (_i, [_p, _p, C.c_int64, _i, _i, _p, _p]),
    "xvb_ecapa_last_launches": (_i, [_p]),
    "xvb_ecapa_save": (_i, [_p, C.c_char_p]),
    "xvb_ecapa_load": (_i, [C.POINTER(_p), C.c_char_p]),
    "xvb_ecapa_destroy": (None, [_p]),
    "xvb_resnet_create": (_i, [C.POINTER(_p), _i, _ip, _ip, _i, _f]),
    "xvb_resnet_set_layer": (_i, [_p, C.c_char_p, _i, _i, _i, _p, _p, _p, _p, _i]),
    "xvb_resnet_finalize": (_i, [_p]),
    "xvb_resnet_feat_dim": (_i, [_p]),
    "xvb_resnet_embed_dim": (_i, [_p]),
    "xvb_resnet_last_launches": (_i, [_p]),
    "xvb_resnet_extract": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_resnet_extract_lengths": (_i, [_p, _p, _p, _i, _i, _p, _p]),
    "xvb_resnet_extract_host": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_resnet_extract_shard": (_i, [_p, _p, C.c_int64, _i, _i, _p, _p]),
    "xvb_resnet_extract_shard_host": (_i, [_p, _p, C.c_int64, _i, _i, _p, _p]),
    "xvb_resnet_save": (_i, [_p, C.c_char_p]),
    "xvb_resnet_load": (_i, [C.POINTER(_p), C.c_char_p]),
    "xvb_resnet_destroy": (None, [_p]),
    "xvb_repvgg_create": (_i, [C.POINTER(_p), _p]),
    "xvb_repvgg_set_layer": (_i, [_p, C.c_char_p, _i, _i, _i, _p, _p, _p, _p, _i]),
    "xvb_repvgg_finalize": (_i, [_p]),
    "xvb_repvgg_feat_dim": (_i, [_p]),
    "xvb_repvgg_embed_dim": (_i, [_p]),
    "xvb_repvgg_last_launches": (_i, [_p]),
    "xvb_repvgg_extract": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_repvgg_save": (_i, [_p, C.c_char_p]),
    "xvb_repvgg_load": (_i, [C.POINTER(_p), C.c_char_p]),
    "xvb_repvgg_destroy": (None, [_p]),
    "xvb_conv2d_kept_taps": (_i, [_p, _i, _i, _i, _ip, _i]),
    "xvb_conformer_create": (_i, [C.POINTER(_p), _p]),
    "xvb_conformer_set_layer": (_i, [_p, C.c_char_p, _i, _i, _p, _p, _p, _p, _i]),
    "xvb_conformer_finalize": (_i, [_p]),
    "xvb_conformer_feat_dim": (_i, [_p]),
    "xvb_conformer_embed_dim": (_i, [_p]),
    "xvb_conformer_last_launches": (_i, [_p]),
    "xvb_conformer_extract": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_conformer_extract_lengths": (_i, [_p, _p, _p, _i, _i, _p, _p]),
    "xvb_conformer_save": (_i, [_p, C.c_char_p]),
    "xvb_conformer_load": (_i, [C.POINTER(_p), C.c_char_p]),
    "xvb_conformer_destroy": (None, [_p]),
    "xvb_campp_create": (_i, [C.POINTER(_p), _p]),
    "xvb_campp_set_layer": (_i, [_p, C.c_char_p, _i, _i, _p, _p, _p, _p, _i]),
    "xvb_campp_finalize": (_i, [_p]),
    "xvb_campp_feat_dim": (_i, [_p]),
    "xvb_campp_embed_dim": (_i, [_p]),
    "xvb_campp_last_launches": (_i, [_p]),
    "xvb_campp_extract": (_i, [_p, _p, _i, _i, _p, _p]),
    "xvb_campp_extract_lengths": (_i, [_p, _p, _p, _i, _i, _p, _p]),
    "xvb_campp_save": (_i, [_p, C.c_char_p]),
    "xvb_campp_load": (_i, [C.POINTER(_p), C.c_char_p]),
    "xvb_campp_destroy": (None, [_p]),
    "xvb_campp_chunk_sizes": (_i, [_i, _i, _ip, _i]),
    "xvb_extractor_load": (_i, [C.POINTER(_p), C.c_char_p]),
    "xvb_extractor_save": (_i, [_p, C.c_char_p]),
    "xvb_extractor_feat_dim": (_i, [C.c_char_p]),
    "xvb_ark_reader_open": (_i, [C.POINTER(_p), C.c_char_p]),
    "xvb_ark_reader_next": (_i, [_p, C.POINTER(C.c_char_p), _ip, _ip, C.POINTER(C.POINTER(C.c_float))]),
    "xvb_ark_reader_close": (None, [_p]),
    "xvb_ark_writer_open": (_i, [C.POINTER(_p), C.c_char_p]),
    "xvb_ark_writer_put_vector": (_i, [_p, C.c_char_p, _p, _i]),
    "xvb_ark_writer_close": (_i, [_p]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)  # AttributeError here == the .so does not export what the header declares
    _fn.restype = _res
    _fn.argtypes = _args


class FbankOpts(C.Structure):
    """xvb_fbank_opts_t"""
    _fields_ = [(n, C.c_float) for n in ("sample_frequency", "frame_length_ms", "frame_shift_ms", "preemphasis_coefficient",
                                         "low_freq", "high_freq", "energy_floor", "cepstral_lifter", "blackman_coeff")] + \
               [(n, C.c_int) for n in ("num_mel_bins", "num_ceps", "use_energy", "raw_energy", "remove_dc_offset",
                                       "use_log_fbank", "use_power", "htk_compat", "window_type")]


def last_error():
    return lib.xvb_last_error().decode("utf-8", "replace")


def check(rc, what=""):
    if rc != 0:
        raise XvbError("{} failed (rc={}): {}".format(what or "libxvb200 call", rc, last_error()))


def int_array(values):
    arr = (C.c_int * len(values))(*[int(v) for v in values])
    return arr
