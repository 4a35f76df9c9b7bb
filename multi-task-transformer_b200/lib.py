"""ctypes binding of libmtt_sm90.so (the C ABI declared in include/mtt_b200.h).

There is no fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmtt_sm90.so")

ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2
METER_CONFUSION, METER_SALIENCY, METER_NORMALS, METER_DEPTH, METER_EDGE = 0, 1, 2, 3, 4


class GemmDesc(C.Structure):
    _fields_ = [
        ("a_hi", C.c_void_p), ("a_lo", C.c_void_p), ("lda", C.c_int64),
        ("b_hi", C.c_void_p), ("b_lo", C.c_void_p), ("ldb", C.c_int64),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("nsplit", C.c_int32), ("mode", C.c_int32),
        ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("ksize", C.c_int32), ("dil", C.c_int32),
        ("bias", C.c_void_p), ("act", C.c_int32),
        ("residual", C.c_void_p), ("ldr", C.c_int64), ("res_row_mod", C.c_int32),
        ("out_f32", C.c_void_p), ("ldo_f32", C.c_int64),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("ldo_bf", C.c_int64),
        ("in_group", C.c_int32), ("out_group", C.c_int32), ("out_offset", C.c_int32),
        ("a_group_rows", C.c_int32), ("a_group_stride", C.c_int64),
        ("out_row_stride", C.c_int32),
        ("sk_ws", C.c_void_p), ("sk_ws_bytes", C.c_int64),
    ]


class AttnDesc(C.Structure):
    _fields_ = [
        ("qkv_hi", C.c_void_p), ("qkv_lo", C.c_void_p),
        ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
        ("prompt_logits", C.c_void_p),
        ("B", C.c_int32), ("N", C.c_int32), ("H", C.c_int32), ("T", C.c_int32),
        ("nsplit", C.c_int32), ("scale", C.c_float),
    ]


class Shape(C.Structure):
    _fields_ = [("rows", C.c_int32), ("C", C.c_int32), ("hidden", C.c_int32), ("nsplit", C.c_int32),
                ("B", C.c_int32), ("N", C.c_int32), ("H", C.c_int32), ("T", C.c_int32)]


class Weight(C.Structure):
    _fields_ = [("hi", C.c_void_p), ("lo", C.c_void_p), ("ld", C.c_int64)]


class GatedTask(C.Structure):
    _fields_ = [("w_spa", Weight), ("b_spa", C.c_void_p), ("w_chan", Weight), ("b_chan", C.c_void_p),
                ("cat_hi", C.c_void_p), ("cat_lo", C.c_void_p)]


OP_LN_QKV, OP_ATTN_FWD, OP_PROJ_RESIDUAL, OP_LN_MLP_RESIDUAL, OP_CHAN_PROMPT_LOGITS = 1, 2, 3, 4, 5
OP_GATED_CONV1X1, OP_CONV3X3_BN_ACT, OP_BILINEAR_UP, OP_INVPT_ATTN, OP_LAYERNORM = 6, 7, 8, 9, 10


class ProfileRec(C.Structure):
    _fields_ = [("kind", C.c_int32), ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("ms", C.c_float),
                ("flops", C.c_double)]


class BilinearSrc(C.Structure):
    _fields_ = [("in_", C.c_void_p), ("ld_in", C.c_int64), ("h", C.c_int32), ("w", C.c_int32),
                ("batch_rows", C.c_int64), ("row_offset", C.c_int64)]


AUG_MAX_TASKS, AUG_CANDIDATES = 7, 11
AUG_TASK_KIND = {"semseg": 0, "human_parts": 1, "sal": 2, "edge": 3, "normals": 4, "depth": 5}


class AugmentSample(C.Structure):
    _fields_ = [("off", C.c_int64 * (1 + AUG_MAX_TASKS)),
                ("lin_y", C.c_double), ("lin_x", C.c_double), ("nn_y", C.c_double), ("nn_x", C.c_double),
                ("h", C.c_int32), ("w", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
                ("scaled", C.c_int32), ("depth_scale", C.c_float),
                ("ncand", C.c_int32), ("cand", C.c_int32 * (2 * AUG_CANDIDATES)),
                ("flip", C.c_int32),
                ("bright_on", C.c_int32), ("f_mode", C.c_int32), ("contrast_on", C.c_int32), ("sat_on", C.c_int32),
                ("hue_on", C.c_int32),
                ("beta", C.c_float), ("alpha", C.c_float), ("sat_alpha", C.c_float), ("hue_delta", C.c_int32)]


class AugmentDesc(C.Structure):
    _fields_ = [("samples", C.c_void_p), ("data", C.c_void_p),
                ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("train", C.c_int32),
                ("crop_h", C.c_int32), ("crop_w", C.c_int32), ("ntasks", C.c_int32),
                ("task_kind", C.c_int32 * AUG_MAX_TASKS), ("task_out", C.c_void_p * AUG_MAX_TASKS),
                ("image_out", C.c_void_p), ("mean", C.c_float * 3), ("std", C.c_float * 3),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


RENDER_MAX_TASKS, RENDER_MAX_IMAGES = 8, 96
RENDER_SRC_LOGITS, RENDER_SRC_CLASS, RENDER_SRC_MAP = 0, 1, 2
RENDER_U8, RENDER_CLASS, RENDER_PALETTE_BGR, RENDER_NORMALS_BGR, RENDER_JET = 0, 1, 2, 3, 4


class RenderDesc(C.Structure):
    _fields_ = [("src_kind", C.c_int32), ("src", C.c_void_p),
                ("B", C.c_int32), ("C", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
                ("out_h", C.c_int32), ("out_w", C.c_int32), ("postproc", C.c_int32), ("encode", C.c_int32),
                ("table", C.c_void_p), ("table_len", C.c_int32),
                ("crop", C.POINTER(C.c_int32)), ("offset", C.POINTER(C.c_int64)), ("out_size", C.POINTER(C.c_int32)),
                ("out", C.c_void_p), ("out_bytes", C.c_int64),
                ("label", C.c_void_p), ("label_numel", C.c_int64), ("ignore_index", C.c_float),
                ("flags", C.c_void_p)]


# name -> (restype, argtypes); every symbol include/mtt_b200.h declares
_i64, _i32, _f32, _vp = C.c_int64, C.c_int32, C.c_float, C.c_void_p
SYMBOLS = {
    "mtt_version": (C.c_int, []),
    "mtt_last_error": (C.c_char_p, []),
    "mtt_device_check": (C.c_int, []),
    "mtt_launch_count": (C.c_int64, []),
    "mtt_launch_count_reset": (None, []),
    "mtt_profile_begin": (C.c_int, []),
    "mtt_profile_end": (C.c_int, [C.POINTER(ProfileRec), _i32, C.POINTER(C.c_int32)]),
    "mtt_split_f32": (C.c_int, [_vp, _i64, _vp, _vp, _i64, _i64, _i32, _i32, _vp]),
    "mtt_layernorm": (C.c_int, [_vp, _i64, _vp, _vp, _f32, _vp, _i64, _vp, _vp, _i64, _i64, _i32, _vp]),
    "mtt_gemm": (C.c_int, [C.POINTER(GemmDesc), _vp]),
    "mtt_gemm_grouped": (C.c_int, [C.POINTER(GemmDesc), _i32, _vp]),
    "mtt_sum_partials": (C.c_int, [_vp, _i32, _i64, _i32, _i64, _vp, _vp, _i64, _vp]),
    "mtt_set_gemm_variant": (None, [C.c_int]),
    "mtt_gemm_streamk_bytes": (C.c_size_t, []),
    "mtt_set_gemm_streamk": (None, [C.c_int]),
    "mtt_debug_streamk_schedule": (C.c_int, [_i32, _i32, _i32, _i32, C.POINTER(C.c_int32), _i32]),
    "mtt_attention": (C.c_int, [C.POINTER(AttnDesc), _vp]),
    "mtt_set_attention_variant": (None, [C.c_int]),
    "mtt_set_attention_trace": (None, [C.c_void_p]),
    "mtt_im2col_patch": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_broadcast_rows": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i64, _i64, _vp]),
    "mtt_chan_logits": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp]),
    "mtt_gate_split": (C.c_int, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32,
                                 _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i64, _i64, _vp]),
    "mtt_ctr_weights": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mtt_ctr_mix": (C.c_int, [_vp, _vp, _vp, _i32, _i64, _i32, _i64, _i32, _i32, _vp]),
    "mtt_bilinear": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _vp, _i64, _vp,
                               _i32, _i64, _i64, _i64, _i64, _vp]),
    "mtt_preprocess_image": (C.c_int, [_vp, _i32, _i32, _i32, _i32, C.POINTER(C.c_float), C.POINTER(C.c_float), _vp,
                                       _i32, _i32, _vp]),
    "mtt_bilinear_postproc": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "mtt_augment_workspace_bytes": (C.c_size_t, [_i32]),
    "mtt_augment": (C.c_int, [C.POINTER(AugmentDesc), _vp]),
    "mtt_cityscapes_targets": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "mtt_render_workspace_bytes": (C.c_size_t, [_i32, _i32]),
    "mtt_render": (C.c_int, [C.POINTER(RenderDesc), _i32, _vp, _vp]),
    "mtt_render_jet_bgr": (C.POINTER(C.c_uint8), []),
    "mtt_bilinear_sum3": (C.c_int,[C.POINTER(BilinearSrc), _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_split_rows": (C.c_int, [_vp, _i64, _i64, _i64, _i64, _vp, _vp, _i64, _i64, _i32, _vp]),
    "mtt_layernorm_seg": (C.c_int, [_vp, _i64, _i64, _i64, _i64, _i64, _i32, _vp, _vp, _f32, _vp, _i64, _vp,
                                    _vp, _i64, _i64, _i64, _i32, _vp]),
    "mtt_zero_insert": (C.c_int, [_vp, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_dwconv3x3_s2": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i64, _vp]),
    "mtt_avgpool": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_invpt_fuse_softmax": (C.c_int, [_vp, _i32, _i32, _i32, _f32, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i64,
                                         _vp]),
    "mtt_workspace_bytes": (C.c_size_t, [_i32, C.POINTER(Shape)]),
    "mtt_ln_qkv": (C.c_int, [_vp, _i64, _vp, _vp, _f32, C.POINTER(Weight), _vp, _vp, _vp, _i64, C.POINTER(Shape), _vp,
                             C.c_size_t, _vp]),
    "mtt_proj_residual": (C.c_int, [_vp, _vp, _i64, C.POINTER(Weight), _vp, _vp, _i64, C.POINTER(Shape), _vp]),
    "mtt_ln_mlp_residual": (C.c_int, [_vp, _i64, _vp, _vp, _f32, C.POINTER(Weight), _vp, C.POINTER(Weight), _vp,
                                      C.POINTER(Shape), _vp, C.c_size_t, _vp]),
    "mtt_gated_conv1x1": (C.c_int, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, C.POINTER(GatedTask), _i32, _i32, _i32, _i32,
                                    _i32, _i64, _i32, C.POINTER(Shape), _vp, C.c_size_t, _vp]),
    "mtt_conv3x3_bn_act": (C.c_int, [_vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, C.POINTER(Weight), _vp, _i32, _i32,
                                     _vp, _vp, _i64, C.POINTER(Weight), _vp, _i32, _vp, _i64, _i32, _vp, C.c_size_t,
                                     _vp]),
    "mtt_pack_weight": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_pack_conv_weight": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _f32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i64,
                                       _vp, _vp, _vp]),
    "mtt_loss_workspace_bytes": (C.c_size_t, []),
    "mtt_loss_cross_entropy": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32, _vp, _vp, _vp]),
    "mtt_loss_cross_entropy_grad": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32, _vp, _vp, _vp, _vp]),
    "mtt_loss_balanced_bce": (C.c_int, [_vp, _vp, _i64, _f32, _f32, _i32, _vp, _vp, _vp]),
    "mtt_loss_balanced_bce_grad": (C.c_int, [_vp, _vp, _i64, _f32, _f32, _i32, _vp, _vp, _vp, _vp]),
    "mtt_loss_l1": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32, _i32, _vp, _vp, _vp]),
    "mtt_loss_l1_grad": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _i32, _i32, _vp, _vp, _vp, _vp]),
    # evaluation meters (csrc/metrics.cu)
    "mtt_meter_state_bytes": (C.c_size_t, [_i32, _i32]),
    "mtt_meter_reset": (C.c_int, [_vp, _i32, _i32, _vp]),
    "mtt_meter_confusion_update": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "mtt_meter_confusion_update_i64": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _vp, _vp]),
    "mtt_meter_saliency_update": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _vp, _i32, _f32, _vp, _vp]),
    "mtt_meter_normals_update": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp]),
    "mtt_meter_depth_update": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _f32, _f32, _f32, _vp, _vp]),
    "mtt_meter_edge_update": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _f32, _f32, _vp, _vp]),
    "mtt_boxes_bev_pairwise": (C.c_int, [_vp, _i32, _vp, _i32, _i32, _vp, _vp]),
    "mtt_nms_workspace_bytes": (C.c_size_t, [_i32]),
    "mtt_nms_bev": (C.c_int, [_vp, _i32, _f32, _i32, _vp, _vp, _vp, C.c_size_t, _vp]),
    "mtt_swin_window_gather": (C.c_int, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_swin_window_attention": (C.c_int, [_vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp,
                                            _i64, _vp, _vp]),
    "mtt_swin_window_scatter": (C.c_int, [_vp, _i64, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i64,
                                          _vp, _i64, _vp, _i64, _vp, _vp]),
    "mtt_transpose_split": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_swin_chan_attention": (C.c_int, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _vp, _vp,
                                          _i64, _vp, _vp]),
    "mtt_swin_merge_gather": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _i64, _vp]),
    "mtt_conv3x3_s2_maps": (C.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i64, _i32, _i64, _i32, _vp, _vp]),
    "mtt_swin_chan_up": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "mtt_swin_logit_maps": (C.c_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp]),
    "mtt_nchw_to_nhwc_split": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_nhwc_to_nchw": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp]),
    # training step (csrc/train_ops.cu)
    "mtt_colsum": (C.c_int, [_vp, _i64, _i64, _i32, _i64, _i64, _i64, _vp, _i32, _vp]),
    "mtt_layernorm_bwd": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _f32, _i64, _i32, _vp, _i64, _i32, _vp, _vp, _vp, _vp]),
    "mtt_act_split": (C.c_int, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_act_bwd": (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i32, _i32, _vp, _i64, _vp]),
    "mtt_axpy_rows": (C.c_int, [_vp, _i64, _vp, _i64, _vp, _i64, _i32, _vp, _i64, _vp]),
    "mtt_transpose_planes": (C.c_int, [_vp, _vp, _i64, _i64, _i32, _i32, _i32, _vp, _vp, _i64, _i64, _vp]),
    "mtt_bn_stats": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _vp]),
    "mtt_bn_finalize": (C.c_int, [_vp, C.c_double, _i32, _f32, _f32, _vp, _vp, _vp, _vp]),
    "mtt_bn_act": (C.c_int, [_vp, _i64, _i64, _i32, _vp, _vp, _vp, _i32, _vp, _i64, _vp, _vp, _i64, _vp]),
    "mtt_bn_bwd_reduce": (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i32, _vp, _vp, _vp, _i32, _vp, _vp]),
    "mtt_bn_bwd_apply": (C.c_int, [_vp, _i64, _vp, _i64, _i64, _i32, _vp, _vp, _vp, _i32, _vp, _f32, _vp, _i64, _vp]),
    "mtt_attn_delta": (C.c_int, [_vp, _i64, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp]),
    "mtt_attn_softmax_bwd": (C.c_int, [_vp, _vp, _vp, _i64, _i32, _i32, _f32, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "mtt_bilinear_bwd": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _i64, _i32, _vp]),
    "mtt_gate_bwd": (C.c_int, [_vp, _i64, _i64, _i64, _vp, _vp, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32,
                               _vp, _vp, _i64, _vp, _i64, _vp, _vp, _vp]),
    "mtt_chan_logits_bwd": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _i32, _vp, _vp,
                                      _i64, _vp]),
    "mtt_ctr_bwd": (C.c_int, [_vp, _vp, _i32, _i64, _i32, _i64, _i32, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                              _vp, _vp, _vp, _vp]),
    "mtt_im2col3x3_t": (C.c_int, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_im2col_patch_t": (C.c_int, [_vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i64, _vp]),
    "mtt_sumsq": (C.c_int, [_vp, _i64, _vp, _i32, _vp]),
    "mtt_adam_step": (C.c_int, [_vp, _vp, _vp, _vp, _i64, _f32, C.c_double, C.c_double, _f32, _f32, _i32, _vp, _f32, _f32,
                                _vp]),
}

_lib = None


def load():
    """Load the shared library (once). Raises RuntimeError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU or eager fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().mtt_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{what} failed ({rc}): {msg}")
