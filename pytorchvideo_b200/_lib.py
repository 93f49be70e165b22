"""ctypes binding of libpvb200.so (the C ABI declared in include/pv_b200.h).

There is deliberately NO fallback: if the library is missing or a call fails, a RuntimeError is
raised.  PyTorch is used only for device memory and streams; nothing here calls ATen compute.
"""
import ctypes as C
import os

from . import _build

PV_F16, PV_F32, PV_U8, PV_I64 = 0, 1, 2, 3
ACT_NONE, ACT_RELU, ACT_SWISH, ACT_GELU, ACT_SIGMOID, ACT_HSWISH = 0, 1, 2, 3, 4, 5
ALGO_AUTO, ALGO_DIRECT, ALGO_TCGEN05 = 0, 1, 2
POOL_MAX, POOL_AVG = 0, 1
MPOOL_MAX, MPOOL_AVG, MPOOL_SUM = 0, 1, 2          # pv_masked_pool modes
REDUCE_MAX, REDUCE_SUM, REDUCE_PROD = 0, 1, 2     # pv_reduce_fusion ops
ATTN_WGMMA, ATTN_MMA, ATTN_SIMT, ATTN_WIDE = 1, 2, 3, 4

c_ll = C.c_longlong
c_vp = C.c_void_p


class ClipTransformDesc(C.Structure):
    _fields_ = [("C", C.c_int), ("n_t", C.c_int), ("out_h", C.c_int), ("out_w", C.c_int),
                ("sc", c_ll), ("st", c_ll), ("sh", c_ll), ("sw", c_ll),
                ("mean", C.c_float * 4), ("stdv", C.c_float * 4),
                ("src_dtype", C.c_int), ("dst_dtype", C.c_int), ("div255", C.c_int)]


class ClipBatchDesc(C.Structure):
    _fields_ = [("C", C.c_int), ("n_clips", C.c_int), ("n_t", C.c_int), ("n_slow", C.c_int),
                ("in_h", C.c_int), ("in_w", C.c_int), ("new_h", C.c_int), ("new_w", C.c_int),
                ("top", C.c_int), ("left", C.c_int), ("out_h", C.c_int), ("out_w", C.c_int),
                ("hflip", C.c_int),
                ("sc", c_ll), ("st", c_ll), ("sh", c_ll), ("sw", c_ll), ("s_clip", c_ll),
                ("d_clip", c_ll), ("d_slow_clip", c_ll),
                ("mean", C.c_float * 4), ("stdv", C.c_float * 4),
                ("div255", C.c_int), ("normalize", C.c_int), ("src_dtype", C.c_int), ("dst_dtype", C.c_int)]


BOX_F32, BOX_F64 = 1, 3                             # pv_boxes_desc.dtype
BOX_CLIP_SRC, BOX_SCALE, BOX_CROP, BOX_CLIP_CROP, BOX_FLIP, BOX_CLIP_OUT = 1, 2, 4, 8, 16, 32   # pv_boxes_desc.steps
BOX_DENORM = 64                                     # pv_clip_boxes_transform_ragged only


class BoxesDesc(C.Structure):
    _fields_ = [("n_clips", C.c_int), ("n_boxes", C.c_int), ("steps", C.c_int), ("dtype", C.c_int),
                ("in_h", C.c_int), ("in_w", C.c_int), ("new_h", C.c_int), ("new_w", C.c_int),
                ("top", C.c_int), ("left", C.c_int), ("hflip", C.c_int), ("out_h", C.c_int), ("out_w", C.c_int)]


class AugOp(C.Structure):
    _fields_ = [("kind", C.c_int), ("ival", C.c_int), ("ratio", C.c_float), ("omr", C.c_float),
                ("theta", C.c_float * 6), ("fill", C.c_float * 3)]


class AugFrameStats(C.Structure):
    _fields_ = [("mn", C.c_float * 3), ("mx", C.c_float * 3), ("gray_sum", C.c_double), ("lut", (C.c_ubyte * 256) * 3)]


class AugmentDesc(C.Structure):
    _fields_ = [("n_clips", C.c_int), ("src_div", C.c_int), ("T", C.c_int), ("C", C.c_int), ("H", C.c_int),
                ("W", C.c_int), ("s_clip", c_ll), ("st", c_ll), ("sc", c_ll), ("sh", c_ll), ("sw", c_ll),
                ("dtype", C.c_int)]


class MixDesc(C.Structure):
    _fields_ = [("B", C.c_int), ("dtype", C.c_int), ("size", c_ll * 4), ("stride", c_ll * 4), ("s_batch", c_ll)]


class MixLabelDesc(C.Structure):
    _fields_ = [("B", C.c_int), ("K", C.c_int), ("one_hot", C.c_int), ("mode", C.c_int),
                ("lam", C.c_float), ("oml", C.c_float), ("on", C.c_float), ("off", C.c_float),
                ("s_row", c_ll), ("s_col", c_ll)]


class CjView(C.Structure):
    _fields_ = [("clip", C.c_int), ("n_ops", C.c_int), ("ops", C.c_int * 4), ("factor", C.c_float * 3),
                ("hue_shift", C.c_int), ("gray", C.c_int), ("blur_r", C.c_int), ("blur_ww", C.c_uint),
                ("blur_fw", C.c_uint)]


class ColorJitterDesc(C.Structure):
    _fields_ = [("n_views", C.c_int), ("n_t", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("s_clip", c_ll), ("sc", c_ll), ("st", c_ll), ("sh", c_ll), ("sw", c_ll),
                ("src_dtype", C.c_int), ("src_scale", C.c_int)]


JPEG_GRAY, JPEG_H1V1, JPEG_H2V1, JPEG_H1V2, JPEG_H2V2 = 0, 1, 2, 3, 4     # pv_jpeg_mode
JPEG_BAD_CODE, JPEG_BAD_OVERRUN, JPEG_BAD_RESTART = 1, 2, 4             # pv_jpeg_decode status bits
# pv_jpeg_parse's rejections, by code
JPEG_ERRORS = {-20: "progressive", -21: "arithmetic", -22: "lossless", -23: "hierarchical", -24: "precision",
               -25: "components", -26: "colorspace", -27: "orientation", -28: "multiscan", -29: "dnl", -30: "sampling"}


class JpegHuff(C.Structure):
    _fields_ = [("look", C.c_uint16 * 512), ("maxcode", C.c_int32 * 18), ("valoff", C.c_int32 * 18),
                ("val", C.c_uint8 * 256)]


class JpegFrame(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("ncomp", C.c_int), ("mode", C.c_int),
                ("mcus_x", C.c_int), ("mcus_y", C.c_int), ("restart_interval", C.c_int), ("n_segments", C.c_int),
                ("n_blocks", C.c_int), ("scan_comp", C.c_int * 3), ("h", C.c_int * 3), ("v", C.c_int * 3),
                ("bw", C.c_int * 3), ("bh", C.c_int * 3), ("dw", C.c_int * 3), ("dh", C.c_int * 3),
                ("block_off", C.c_int * 3), ("dc_tbl", C.c_int * 3), ("ac_tbl", C.c_int * 3),
                ("data_off", c_ll), ("seg_base", c_ll), ("block_base", c_ll), ("out_off", c_ll),
                ("qt", (C.c_uint16 * 64) * 3), ("dc", JpegHuff * 2), ("ac", JpegHuff * 2)]


class JpegBatch(C.Structure):
    _fields_ = [("n_frames", C.c_int), ("mode_mask", C.c_int), ("max_blocks", C.c_int), ("max_pixels", C.c_int),
                ("n_segments", c_ll), ("n_blocks", c_ll), ("data_bytes", c_ll), ("out_elems", c_ll),
                ("ws_bytes", c_ll)]


class BottleneckDesc(C.Structure):
    _fields_ = [("N", C.c_int), ("T", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("Cin", C.c_int), ("Cmid", C.c_int), ("Cout", C.c_int), ("kt", C.c_int), ("sb", C.c_int),
                ("has_shortcut", C.c_int), ("act", C.c_int), ("x_row_stride", c_ll), ("y_row_stride", c_ll)]


class Conv3dDesc(C.Structure):
    _fields_ = [("dtype", C.c_int),
                ("N", C.c_int), ("Ti", C.c_int), ("Hi", C.c_int), ("Wi", C.c_int), ("Ci", C.c_int),
                ("To", C.c_int), ("Ho", C.c_int), ("Wo", C.c_int), ("Co", C.c_int),
                ("kt", C.c_int), ("kh", C.c_int), ("kw", C.c_int),
                ("st", C.c_int), ("sh", C.c_int), ("sw", C.c_int),
                ("pt", C.c_int), ("ph", C.c_int), ("pw", C.c_int),
                ("dt", C.c_int), ("dh", C.c_int), ("dw", C.c_int),
                ("groups", C.c_int), ("act", C.c_int), ("has_residual", C.c_int),
                ("x_row_stride", c_ll), ("y_row_stride", c_ll), ("res_row_stride", c_ll),
                ("ci_pad64", C.c_int), ("x_w_pad", C.c_int), ("x_w_phys", C.c_int),
                ("x_batch_stride", c_ll), ("y_batch_stride", c_ll),
                ("addend", c_vp), ("add_n_stride", c_ll), ("add_t_stride", c_ll), ("add_ch_off", C.c_int),
                ("pre_scale", c_vp), ("pre_bias", c_vp), ("pre_act", C.c_int)]


class Pool3dDesc(C.Structure):
    _fields_ = [("dtype", C.c_int), ("mode", C.c_int),
                ("N", C.c_int), ("Ti", C.c_int), ("Hi", C.c_int), ("Wi", C.c_int), ("C", C.c_int),
                ("To", C.c_int), ("Ho", C.c_int), ("Wo", C.c_int),
                ("kt", C.c_int), ("kh", C.c_int), ("kw", C.c_int),
                ("st", C.c_int), ("sh", C.c_int), ("sw", C.c_int),
                ("pt", C.c_int), ("ph", C.c_int), ("pw", C.c_int),
                ("x_row_stride", c_ll), ("y_row_stride", c_ll),
                ("x_batch_stride", c_ll), ("y_batch_stride", c_ll)]


class AttentionDesc(C.Structure):
    _fields_ = [("dtype", C.c_int), ("B", C.c_int), ("H", C.c_int), ("Nq", C.c_int),
                ("Nk", C.c_int), ("D", C.c_int),
                ("q_row_stride", c_ll), ("k_row_stride", c_ll), ("v_row_stride", c_ll),
                ("o_row_stride", c_ll),
                ("q_batch_stride", c_ll), ("k_batch_stride", c_ll), ("v_batch_stride", c_ll),
                ("o_batch_stride", c_ll),
                ("scale", C.c_float), ("add_q_residual", C.c_int), ("normalize", C.c_int)]


# name -> (restype, argtypes); mirrors include/pv_b200.h one to one (tests check this list
# against the header and against the symbols the .so exports).
SIGNATURES = {
    "pv_abi_version": (C.c_int, []),
    "pv_last_error": (C.c_char_p, []),
    "pv_device_info": (C.c_int, [C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "pv_launch_count": (c_ll, []),
    "pv_kernel_counts": (C.c_int, [C.c_char_p, C.c_int]),
    "pv_clip_transform_fwd": (C.c_int, [C.POINTER(ClipTransformDesc), c_vp, c_vp, c_vp, c_vp, c_vp,
                                        c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_clip_transform_batch": (C.c_int, [C.POINTER(ClipBatchDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_clip_transform_rrc": (C.c_int, [C.POINTER(ClipBatchDesc), c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_clip_transform_ragged": (C.c_int, [C.POINTER(ClipBatchDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_clip_boxes_transform": (C.c_int, [C.POINTER(BoxesDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_clip_boxes_transform_ragged": (C.c_int, [C.POINTER(BoxesDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_augment_stats": (C.c_int, [C.POINTER(AugmentDesc), c_vp, c_vp, c_vp]),
    "pv_augment_apply": (C.c_int, [C.POINTER(AugmentDesc), c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_augment_mix": (C.c_int, [C.POINTER(AugmentDesc), c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp]),
    "pv_mixup": (C.c_int, [C.POINTER(MixDesc), c_vp, C.c_float, C.c_float, c_vp]),
    "pv_cutmix": (C.c_int, [C.POINTER(MixDesc), c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp]),
    "pv_mix_labels": (C.c_int, [C.POINTER(MixLabelDesc), c_vp, c_vp, c_vp, c_vp]),
    "pv_view_reduce": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp]),
    "pv_ncdhw_to_ndhwc": (C.c_int, [c_vp, C.c_int, c_vp, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_int, C.c_int, c_ll, c_vp]),
    "pv_ncdhw_to_ndhwc_padw": (C.c_int, [c_vp, C.c_int, c_vp, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, c_vp]),
    "pv_zero_f32": (C.c_int, [c_vp, c_ll, c_vp]),
    "pv_ndhwc_to_ncdhw": (C.c_int, [c_vp, C.c_int, c_ll, c_vp, C.c_int, C.c_int, C.c_int,
                                    C.c_int, C.c_int, c_vp]),
    "pv_conv3d_fwd": (C.c_int, [C.POINTER(Conv3dDesc), C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp,
                                c_vp, c_vp]),
    "pv_dwconv3d_fwd": (C.c_int, [C.POINTER(Conv3dDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_dwplane_supported": (C.c_int, [C.POINTER(Conv3dDesc)]),
    "pv_dwplane_fwd": (C.c_int, [C.POINTER(Conv3dDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_temporal_tap_sum": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_ll, C.c_int, C.c_int,
                                      C.c_int, C.c_int, C.c_int, c_vp, c_vp, C.c_int, c_ll, c_ll, c_vp]),
    "pv_conv3d_tcgen05_supported": (C.c_int, [C.POINTER(Conv3dDesc)]),
    "pv_conv3d_group_span": (C.c_int, [C.POINTER(Conv3dDesc), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "pv_conv3d_stem_rows_supported": (C.c_int, [C.POINTER(Conv3dDesc)]),
    "pv_conv3d_stem_rows_fwd": (C.c_int, [C.POINTER(Conv3dDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_conv3d_stem_stream_supported": (C.c_int, [C.POINTER(Conv3dDesc)]),
    "pv_conv3d_stem_stream_fwd": (C.c_int, [C.POINTER(Conv3dDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_bottleneck_fused_supported": (C.c_int, [C.POINTER(BottleneckDesc)]),
    "pv_bottleneck_fused_fwd": (C.c_int, [C.POINTER(BottleneckDesc)] + [c_vp] * 15),
    "pv_bottleneck_fused_tiling": (C.c_int, [C.POINTER(BottleneckDesc), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                             C.POINTER(C.c_int), C.POINTER(c_ll)]),
    "pv_pool3d_fwd": (C.c_int, [C.POINTER(Pool3dDesc), c_vp, c_vp, c_vp]),
    "pv_channel_sum": (C.c_int, [c_vp, C.c_int, c_ll, C.c_int, c_ll, C.c_int, c_vp, c_vp]),
    "pv_se_gate": (C.c_int, [c_vp, c_ll, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp,
                             C.c_int, c_vp, c_vp]),
    "pv_scale_act": (C.c_int, [c_vp, c_vp, C.c_int, c_ll, c_ll, C.c_int, c_ll, C.c_int, c_vp,
                               C.c_int, c_vp]),
    "pv_head_reduce": (C.c_int, [c_vp, C.c_int, c_ll, C.c_int, c_ll, C.c_int, C.c_int, c_vp,
                                 c_vp]),
    "pv_roi_align_fwd": (C.c_int, [c_vp, C.c_int, c_ll, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, C.c_int, C.c_int,
                                   C.c_int, C.c_float, C.c_int, c_vp, c_ll, c_vp]),
    "pv_layernorm": (C.c_int, [c_vp, c_vp, C.c_int, c_ll, C.c_int, C.c_int, c_ll, c_ll, c_vp, c_vp,
                               C.c_float, c_vp]),
    "pv_layernorm_sets": (C.c_int, [c_vp, c_vp, C.c_int, c_ll, C.c_int, C.c_int, c_ll, c_ll, c_vp, c_vp, C.c_int, c_vp,
                                    c_ll, c_ll, C.c_float, c_vp]),
    "pv_copy_rows": (C.c_int, [c_vp, c_vp, C.c_int, c_ll, C.c_int, c_ll, c_ll, c_vp]),
    "pv_add_pos_cls": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, c_ll, C.c_int, c_ll, c_vp, C.c_int, c_vp]),
    "pv_add_pos_cls_to": (C.c_int, [c_vp, C.c_int, c_vp, C.c_int, C.c_int, c_ll, C.c_int, c_ll, c_vp, C.c_int, c_vp]),
    "pv_add_layernorm": (C.c_int, [c_vp, C.c_int, c_ll, c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_ll, C.c_int, c_vp, c_vp,
                                   C.c_float, c_vp]),
    "pv_attention_fwd": (C.c_int, [C.POINTER(AttentionDesc), c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_attention_kernel_for": (C.c_int, [C.POINTER(AttentionDesc), c_vp, c_vp, c_vp, c_vp]),
    "pv_attention_masked_fwd": (C.c_int, [C.POINTER(AttentionDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_attention_weights": (C.c_int, [C.POINTER(AttentionDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_masked_pool": (C.c_int, [c_vp, C.c_int, c_ll, C.c_int, C.c_int, C.c_int, c_vp, C.c_int, c_vp, c_ll, c_vp]),
    "pv_masked_default": (C.c_int, [c_vp, C.c_int, c_ll, C.c_int, C.c_int, c_vp, C.c_int, c_vp, c_vp, c_ll, c_vp]),
    "pv_mask_force_first": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, c_vp]),
    "pv_reduce_fusion": (C.c_int, [c_vp, c_vp, C.c_int, C.c_int, c_ll, C.c_int, C.c_int, c_vp, c_ll, c_vp]),
    "pv_lstm_recurrence": (C.c_int, [c_vp, C.c_int, c_ll, c_vp, c_vp, C.c_int, C.c_int, C.c_int, C.c_int, c_vp, c_ll,
                                     c_vp]),
    "pv_rows_l2_normalize": (C.c_int, [c_vp, C.c_int, c_ll, c_vp, c_ll, C.c_int, C.c_int, c_vp]),
    "pv_contrastive_ce": (C.c_int, [c_vp, c_ll, c_vp, c_ll, C.c_int, C.c_int, C.c_int, C.c_float, c_ll, C.c_int, c_vp,
                                    c_vp, c_vp]),
    "pv_memory_bank_ce": (C.c_int, [c_vp, c_ll, c_vp, c_ll, C.c_int, c_vp, C.c_int, C.c_int, C.c_float, c_vp, c_vp, c_vp,
                                    c_vp, c_vp]),
    "pv_soft_target_ce": (C.c_int, [c_vp, C.c_int, c_ll, c_vp, C.c_int, c_ll, C.c_int, C.c_int, C.c_int, C.c_float,
                                    C.c_int, c_vp, c_vp, c_vp]),
    "pv_ema_update": (C.c_int, [c_vp, c_vp, c_vp, c_vp, C.c_int, C.c_float, C.c_float, c_vp]),
    "pv_weights_refresh": (C.c_int, [c_vp, c_vp, C.c_int, c_vp, c_vp, c_vp, C.c_int, c_vp]),
    "pv_colorjitter_stats": (C.c_int, [C.POINTER(ColorJitterDesc), c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_colorjitter_apply": (C.c_int, [C.POINTER(ColorJitterDesc), c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_colorjitter_vblur": (C.c_int, [C.POINTER(ColorJitterDesc), c_vp, c_vp, c_vp]),
    "pv_bank_workspace": (C.c_int, [C.c_int, C.c_int, c_ll, C.c_int, C.POINTER(c_ll)]),
    "pv_bank_topk": (C.c_int, [c_vp, c_ll, C.c_int, c_vp, c_ll, C.c_int, C.c_int, c_vp, C.c_int, C.c_float, c_vp, c_ll,
                               c_vp, c_vp, c_vp, c_vp, c_vp]),
    "pv_bank_update": (C.c_int, [c_vp, c_ll, C.c_int, c_vp, c_vp, c_ll, C.c_int, C.c_float, C.c_float, c_vp, c_vp]),
    "pv_queue_ce": (C.c_int, [c_vp, c_ll, C.c_int, C.c_int, c_vp, c_ll, c_vp, c_ll, C.c_int, C.c_int, c_vp, c_ll,
                              C.c_int, C.c_float, c_vp, c_ll, C.c_int, c_vp, c_vp, c_vp]),
    "pv_jpeg_parse": (C.c_int, [c_vp, c_ll, C.POINTER(JpegBatch), C.POINTER(JpegFrame), c_vp, c_ll]),
    "pv_jpeg_decode": (C.c_int, [C.POINTER(JpegBatch), c_vp, c_vp, c_vp, c_vp, c_ll, c_vp, C.c_int, c_vp, c_vp]),
}

_lib = None


def lib_path():
    return _build.LIB_PATH


def load():
    """Load (building first if sources are newer) and return the ctypes library handle."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB_PATH
    if not os.path.exists(path) or _build.needs_build():
        path = _build.build()
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.pv_abi_version() != 1:
        raise RuntimeError("libpvb200 ABI version mismatch")
    _lib = lib
    return lib


def last_error():
    return load().pv_last_error().decode("utf-8", "replace")


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError("libpvb200 %s failed (status %d): %s" % (what, rc, last_error()))


def require_device():
    """Raise unless an sm_90 GPU is visible (the product path has no CPU implementation)."""
    sm, cc = C.c_int(0), C.c_int(0)
    rc = load().pv_device_info(C.byref(sm), C.byref(cc))
    check(rc, "pv_device_info")
    return sm.value, cc.value


def launch_count():
    return int(load().pv_launch_count())


def group_span(desc):
    """(taken, span_groups, span_k, span_n) of a grouped Conv3dDesc (pv_conv3d_group_span, host only)."""
    sg, sk, sn = C.c_int(0), C.c_int(0), C.c_int(0)
    ok = load().pv_conv3d_group_span(C.byref(desc), C.byref(sg), C.byref(sk), C.byref(sn))
    return bool(ok), sg.value, sk.value, sn.value


def kernel_counts():
    """{kernel instance name: launches since load}, e.g. {"conv3d_igemm_kernel<64,128>": 3, ...}."""
    lib = load()
    n = lib.pv_kernel_counts(None, 0)
    while True:
        buf = C.create_string_buffer(n + 1)
        m = lib.pv_kernel_counts(buf, n + 1)
        if m <= n:
            break
        n = m                      # another thread launched a new instance in between
    out = {}
    for line in buf.value.decode().splitlines():
        name, count = line.rsplit(" ", 1)
        out[name] = int(count)
    return out
