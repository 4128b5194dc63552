"""ctypes binding of libc3d.so (C ABI declared in include/c3d.h).  No torch types cross it.

Every entry point and every struct of c3d.h is declared here once; tests/test_abi.py checks both against the header."""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# C3D_LIB_PATH: developer override (an alternative build of the library); never a fallback
LIB_PATH = os.environ.get("C3D_LIB_PATH") or os.path.join(_HERE, "libc3d.so")
_lib = None

C3D_OK, C3D_EINVAL, C3D_EWORKSPACE, C3D_ECUDA = 0, -1, -2, -3

vp, i32, i64, f32, f64, sz = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_double, ctypes.c_size_t


class C3DError(RuntimeError):
    pass


# ---- struct mirrors (field names and order as in c3d.h) ----------------------------------------------------------------
class ConvDesc(ctypes.Structure):
    _fields_ = [("N", i32), ("H", i32), ("W", i32), ("Cin", i32), ("Cout", i32), ("KH", i32), ("KW", i32),
                ("stride", i32), ("pad", i32), ("relu", i32), ("out_fp32", i32), ("add_mode", i32),
                ("y_pix_stride", i64),
                ("y_img_stride", i64), ("y_h_stride", i64), ("y_w_stride", i64), ("y_offset", i64),
                ("out_h", i32), ("out_w", i32), ("x_img_stride", i64), ("y_split_c", i32), ("pad_", i32),
                ("y_split_off", i64)]


class PackDesc(ctypes.Structure):
    _fields_ = [("src", vp), ("fwd", vp), ("dgrad", vp), ("phase", vp * 4), ("start", i64), ("Cout", i32), ("Cin", i32),
                ("KH", i32), ("KW", i32), ("src_is_ohwi", i32), ("merged_phases", i32)]


class RoiLevels(ctypes.Structure):
    _fields_ = [("feat", vp * 5), ("grad", vp * 5), ("H", i32 * 5), ("W", i32 * 5), ("scale", f32 * 5),
                ("num_levels", i32), ("num_images", i32), ("grad_bf16", i32)]


class TopkSeg(ctypes.Structure):
    _fields_ = [("vals", vp), ("row_stride", i64), ("n", i32), ("k", i32), ("out_col", i32)]


class LabelSampleArgs(ctypes.Structure):
    _fields_ = [("prop_boxes", vp), ("prop_count", vp), ("gt_boxes", vp), ("gt_classes", vp), ("gt_present", vp),
                ("gt_boxes3D", vp), ("gt_poses", vp), ("B", i32), ("P", i32), ("G", i32), ("K", i32), ("S", i32),
                ("Fcap", i32), ("append_gt", i32), ("iou_thresh", f32), ("ignore_thresh", f32), ("rng", vp),
                ("bump_rng", i32), ("matched_idx", vp), ("matched_iou", vp), ("labels", vp), ("s_boxes", vp),
                ("s_valid", vp), ("s_classes", vp), ("s_gt_boxes", vp), ("s_gt_boxes3D", vp), ("s_gt_poses", vp),
                ("s_index", vp), ("stats", vp)]


STRUCTS = {"c3d_conv_desc": ConvDesc, "c3d_pack_desc": PackDesc, "c3d_roi_levels": RoiLevels, "c3d_topk_seg": TopkSeg,
           "c3d_label_sample_args": LabelSampleArgs}

# ---- entry points: name -> (restype, argtypes), in c3d.h order ---------------------------------------------------------
# every pointer is c_void_p (device buffers, host arrays, ctypes.byref of a scalar) except the struct descriptors
_conv, _roi = ctypes.POINTER(ConvDesc), ctypes.POINTER(RoiLevels)
SIGNATURES = {
    "c3d_last_error": (ctypes.c_char_p, []),
    "c3d_abi_version": (i32, []),
    # oriented-box 3D IoU
    "c3d_iou_box3d_workspace_bytes": (sz, [i64, i64]),
    "c3d_iou_box3d": (i32, [vp, i64, vp, i64, vp, vp, vp, vp, sz, vp]),
    "c3d_iou_box3d_paired": (i32, [vp, vp, i64, vp, vp, vp, vp, sz, vp]),
    "c3d_box3d_overlap": (i32, [vp, i64, vp, i64, f32, f32, vp, vp, vp, sz, vp]),
    "c3d_box3d_overlap_segmented_workspace_bytes": (sz, [i64, i64, i64]),
    "c3d_box3d_overlap_segmented": (i32, [vp, i64, vp, i64, vp, vp, vp, i32, i64, f32, f32, vp, vp, vp, sz, vp]),
    # convolution
    "c3d_conv2d_tiles": (i32, [_conv, vp, vp, vp]),
    "c3d_conv2d_fwd": (i32, [_conv, vp, vp, vp, vp, vp, vp, vp]),
    "c3d_conv2d_wgrad": (i32, [_conv, vp, vp, vp, i32, vp]),
    "c3d_pack_conv_weight": (i32, [ctypes.POINTER(PackDesc), vp]),
    "c3d_pack_conv_weights_batched": (i32, [vp, i32, i64, vp]),
    # fully-connected layers
    "c3d_pack_linear_weight": (i32, [vp, i32, i32, i32, i32, vp, vp, vp]),
    "c3d_linear_fwd": (i32, [vp, vp, vp, vp, i32, i64, i64, i32, i32, i32, i32, vp]),
    "c3d_linear_dgrad": (i32, [vp, vp, vp, i32, i64, i64, i32, i32, i32, vp]),
    "c3d_linear_wgrad": (i32, [vp, vp, vp, i32, i64, i64, i32, i32, i32, i32, vp]),
    # NHWC kernels around the convolutions
    "c3d_bn_scratch_bytes": (sz, [i32]),
    "c3d_bn_finalize": (i32, [vp, i32, i32, f64, f32, f32, vp, vp, vp, vp, vp, vp]),
    "c3d_bn_apply": (i32, [vp, vp, vp, vp, vp, vp, i32, vp, i64, i32, vp]),
    "c3d_bn_bwd_blocks": (i32, [i64, i32]),
    "c3d_bn_bwd": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, i64, i32, i64, i64, vp, vp]),
    "c3d_bias_act_bwd": (i32, [vp, vp, i32, i32, vp, vp, vp, i64, i32, vp, vp]),
    "c3d_sumpool2": (i32, [vp, vp, i32, i32, i32, i32, vp]),
    "c3d_zero_stuff2": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    "c3d_maxpool2_fwd": (i32, [vp, vp, i32, i32, i32, i32, vp]),
    "c3d_maxpool2_bwd": (i32, [vp, vp, vp, i32, i32, i32, i32, i64, i64, i32, vp]),
    "c3d_maxpool3s2_fwd": (i32, [vp, vp, i32, i32, i32, i32, vp]),
    "c3d_maxpool3s2_bwd": (i32, [vp, vp, vp, i32, i32, i32, i32, i64, vp]),
    "c3d_preprocess_batch": (i32, [vp, vp, vp, i32, i32, vp, i32, i32, i32, vp, vp, vp]),
    "c3d_grad_finite": (i32, [vp, i64, vp, vp]),
    "c3d_sgd_momentum": (i32, [vp, vp, vp, i64, f32, vp, f32, f32, f32, vp, vp]),
    # Adam-family update and per-parameter gradient clipping
    "c3d_adam": (i32, [vp, vp, vp, vp, vp, i64, f32, vp, vp, f64, f64, f64, f64, i32, f32, vp, vp]),
    "c3d_clip_grad_chunks": (i32, [vp, i32, vp]),
    "c3d_clip_grad_workspace_bytes": (sz, [i32]),
    "c3d_clip_grad": (i32, [vp, i64, i32, f32, f32, f32, vp, vp, i32, i32, vp, vp, vp, sz, vp]),
    # ROIAlign
    "c3d_roi_align_fwd": (i32, [_roi, vp, i32, i32, i32, i32, vp, vp]),
    "c3d_roi_align_bwd": (i32, [_roi, vp, i32, i32, i32, i32, vp, vp]),
    # NMS
    "c3d_nms_workspace_bytes": (sz, [i32, i32]),
    "c3d_nms_batched": (i32, [vp, vp, vp, vp, i32, i32, i32, f32, i32, vp, vp, vp, sz, vp]),
    "c3d_nms_batched_grouped": (i32, [vp, vp, vp, vp, i32, i32, i32, f32, i32, i32, i32, vp, vp, vp, sz, vp]),
    # RPN
    "c3d_anchor_match": (i32, [vp, i64, vp, vp, vp, i32, i32, f32, vp, vp, vp, vp, vp, vp, vp]),
    "c3d_rpn_loss_fwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i64, i32, vp, vp, vp]),
    "c3d_rpn_loss_bwd": (i32, [vp, vp, vp, vp, vp, vp, i32, i64, i32, vp, vp, vp, vp, vp, vp]),
    "c3d_rpn_decode_level": (i32, [vp, vp, i64, vp, vp, vp, i32, i32, i64, vp, f32, f32, i32, i32, i32, vp, vp, vp, vp,
                                   vp, vp]),
    # cube head losses
    "c3d_cube_loss_fwd": (i32, [vp, vp, i32, vp, vp]),
    "c3d_cube_loss_bwd": (i32, [vp, vp, vp, i32, vp, vp]),
    # selection / sampling
    "c3d_topk_segments": (i32, [ctypes.POINTER(TopkSeg), i32, i32, i32, vp, vp, vp, vp, vp]),
    "c3d_label_sample_proposals": (i32, [ctypes.POINTER(LabelSampleArgs), vp]),
    "c3d_anchor_sample_keys": (i32, [vp, vp, i32, i64, vp, vp, vp, vp]),
    "c3d_anchor_sample_finish": (i32, [vp, vp, vp, vp, vp, vp, vp, i32, i32, i64, i32, i32, i32, f32, vp, vp, vp]),
    "c3d_det_candidates": (i32, [vp, vp, vp, vp, i32, i32, i32, f32, vp, vp, vp, vp, vp]),
    # ROI-head loss assembly
    "c3d_box_loss_fwd": (i32, [vp, i32, vp, vp, vp, vp, i32, i32, vp, vp, vp]),
    "c3d_box_loss_bwd": (i32, [vp, i32, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp]),
    "c3d_cube_gather": (i32, [vp, i32, vp, vp, vp, vp, vp, vp, i32, i32, i32, f32, vp, vp, vp]),
    "c3d_cube_reduce_fwd": (i32, [vp, vp, i32, vp, vp, vp]),
    "c3d_cube_reduce_bwd": (i32, [vp, vp, i32, vp, vp, vp, vp]),
    "c3d_cube_scatter": (i32, [vp, vp, i32, i32, i32, vp, vp]),
    # input pipeline
    "c3d_resize_bilinear_u8": (i32, [vp, i32, i32, i32, vp, vp, i32, vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp]),
}


def lib():
    """Load libc3d.so with every entry point's signature applied, or raise — the product path has no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise C3DError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(make -C omni3d_b200/csrc). omni3d_b200 has no CPU / library fallback.")
    L = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = L
    return L


def ptr(t):
    """device address of a tensor (None -> NULL)"""
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream(device=None):
    """the current CUDA stream of `device` (default: the current device) as the ABI's `void* stream`"""
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


# number of libc3d kernel launches issued through the python front-ends (bench.py's gpu_launches)
LAUNCHES = {"n": 0}


def check(code, launches=1):
    LAUNCHES["n"] += launches
    if code != C3D_OK:
        raise C3DError(f"libc3d error {code}: {lib().c3d_last_error().decode()}")
