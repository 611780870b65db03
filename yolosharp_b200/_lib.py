"""ctypes binding of include/yolob200.h.  The library is the product: if it is missing the
import fails loudly - there is no Python/CPU fallback for any op."""
import ctypes as C
import os

from ._build import LIB_PATH

c_i32, c_f32, c_vp, c_cp = C.c_int32, C.c_float, C.c_void_p, C.c_char_p


class yb_config(C.Structure):
    _fields_ = [(n, c_i32) for n in ("arch", "size", "task", "nc", "reg_max", "precision", "device",
                                     "max_batch", "height", "width", "flags")]


YB_OK = 0
STATUS_NAMES = {0: "YB_OK", -1: "YB_ERR_INVALID_ARG", -2: "YB_ERR_NOT_IMPLEMENTED", -3: "YB_ERR_CUDA",
                -4: "YB_ERR_STATE", -5: "YB_ERR_MISSING_WEIGHT", -6: "YB_ERR_SHAPE", -7: "YB_ERR_NO_DEVICE"}
YB_ARCH_V8, YB_ARCH_V11 = 8, 11
SIZES = {"n": 0, "s": 1, "m": 2, "l": 3, "x": 4}
YB_TASK_DETECT, YB_TASK_SEGMENT = 0, 1
YB_PREC_F32, YB_PREC_F16 = 0, 1
YB_U8, YB_F16, YB_F32, YB_BF16 = 0, 5, 6, 15
YB_FLAG_NO_TCGEN05, YB_FLAG_NO_GRAPH, YB_FLAG_DRY_RUN, YB_FLAG_NO_CONCURRENCY = 1, 2, 4, 8

# name -> (restype, argtypes); must list every function declared in include/yolob200.h
SIGNATURES = {
    "yb_abi_version": (c_i32, []),
    "yb_build_info": (c_cp, []),
    "yb_last_error": (c_cp, []),
    "yb_create": (c_i32, [C.POINTER(yb_config), C.POINTER(c_vp)]),
    "yb_destroy": (None, [c_vp]),
    "yb_num_anchors": (c_i32, [c_vp]),
    "yb_pred_channels": (c_i32, [c_vp]),
    "yb_load_tensor": (c_i32, [c_vp, c_cp, c_i32, c_i32, C.POINTER(C.c_int64), c_vp]),
    "yb_finalize_weights": (c_i32, [c_vp]),
    "yb_ckpt_open": (c_i32, [c_cp, C.POINTER(c_vp)]),
    "yb_ckpt_count": (c_i32, [c_vp]),
    "yb_ckpt_tensor": (c_i32, [c_vp, c_i32, C.POINTER(c_cp), C.POINTER(c_i32), C.POINTER(c_i32), C.POINTER(C.POINTER(C.c_int64)),
                               C.POINTER(c_vp), C.POINTER(C.c_int64)]),
    "yb_ckpt_close": (None, [c_vp]),
    "yb_load_checkpoint": (c_i32, [c_vp, c_cp, C.POINTER(c_i32), C.POINTER(c_i32)]),
    "yb_ckpt_write_bin": (c_i32, [c_cp, c_i32, C.POINTER(c_cp), C.POINTER(c_i32), C.POINTER(c_i32), C.POINTER(C.POINTER(C.c_int64)),
                                  C.POINTER(c_vp)]),
    "yb_num_expected_tensors": (c_i32, [c_vp]),
    "yb_expected_tensor_name": (c_cp, [c_vp, c_i32]),
    "yb_forward": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "yb_forward_padded": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "yb_nms": (c_i32, [c_vp, c_i32, c_i32, c_i32, c_i32, c_f32, c_f32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp]),
    "yb_topk_postprocess": (c_i32, [c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "yb_obb_decode": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "yb_pose_decode": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "yb_probiou": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_f32, c_vp, c_vp]),
    "yb_nms_rotated": (c_i32, [c_vp, c_vp, c_i32, c_f32, c_vp, c_vp, c_vp]),
    "yb_box_iou": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_f32, c_vp, c_vp]),
    "yb_match_predictions": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_vp, c_i32, c_vp, c_i32, c_vp, c_vp]),
    "yb_linspace01": (c_i32, [c_i32, c_vp]),
    "yb_mask_iou": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_i32, c_f32, c_vp, c_vp]),
    "yb_segmentation_loss": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_f32, c_f32, c_f32, c_vp, c_vp,
                                     c_vp, c_vp]),
    "yb_ap_per_class": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                c_vp, c_vp, c_vp, c_vp]),
    "yb_masks": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "yb_detection_loss": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_i32, c_i32, c_f32, c_f32, c_f32,
                                  c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "yb_bn_silu_train_forward": (c_i32, [c_vp, C.c_int64, c_i32, c_i32, c_vp, c_vp, c_f32, c_f32, c_i32, c_vp, c_vp, c_vp, c_i32,
                                         c_vp, c_vp, c_vp]),
    "yb_bn_silu_backward": (c_i32, [c_vp, c_vp, C.c_int64, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp, c_i32, c_vp,
                                    c_vp, c_vp]),
    "yb_conv_forward_f32": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "yb_conv_backward_data": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "yb_conv_backward_weight": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "yb_conv_tc_workspace_bytes": (C.c_int64, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32]),
    "yb_conv_forward_tc": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, C.c_int64, c_vp]),
    "yb_conv_backward_data_tc": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, C.c_int64, c_vp]),
    "yb_conv_backward_weight_tc": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, C.c_int64, c_vp]),
    "yb_trainer_create": (c_i32, [C.POINTER(yb_config), C.POINTER(c_vp)]),
    "yb_trainer_destroy": (None, [c_vp]),
    "yb_trainer_num_tensors": (c_i32, [c_vp, c_i32]),
    "yb_trainer_tensor_info": (c_i32, [c_vp, c_i32, c_i32, C.POINTER(c_cp), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(c_i32),
                                       C.POINTER(C.POINTER(C.c_int64))]),
    "yb_trainer_flat_size": (C.c_int64, [c_vp, c_i32]),
    "yb_trainer_bind": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "yb_train_backward": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_vp, c_i32, c_vp, c_vp]),
    "yb_train_apply": (c_i32, [c_vp, c_f32, c_f32, c_f32, c_vp]),
    "yb_train_step": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_vp, c_i32, c_f32, c_f32, c_f32, c_vp, c_vp]),
    "yb_get_grad": (c_i32, [c_vp, c_cp, c_vp, C.c_int64]),
    "yb_get_tensor": (c_i32, [c_vp, c_cp, c_vp, C.c_int64]),
    "yb_trainer_evaluate": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp]),
    "yb_trainer_val_begin": (c_i32, [c_vp, c_i32, c_i32, c_vp]),
    "yb_trainer_val_batch": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_vp, c_i32, c_vp]),
    "yb_trainer_val_append": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_i32, c_vp, c_i32, c_vp]),
    "yb_trainer_val_rows": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp]),
    "yb_trainer_val_end": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_vp]),
    "yb_stem_conv_forward_f32": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "yb_stem_conv_backward_weight_f32": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, C.c_int64, c_vp]),
    "yb_dwconv3x3_forward_f32": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp]),
    "yb_dwconv3x3_backward_f32": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "yb_attention_forward_f32": (c_i32, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_f32, c_vp, c_vp]),
    "yb_attention_backward_f32": (c_i32, [c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_f32, c_vp, c_vp, c_vp, c_vp]),
    "yb_adamw_step": (c_i32, [c_vp, c_vp, c_vp, c_vp, C.c_int64, c_i32, c_f32, c_f32, c_f32, c_f32, c_f32, c_vp]),
    "yb_predict_u8": (c_i32, [c_vp, c_vp, c_i32, c_f32, c_f32, c_i32, c_vp, c_vp, c_vp]),
    "yb_predict_u8_submit": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_f32, c_f32, c_i32, c_vp, c_vp]),
    "yb_predict_u8_wait": (c_i32, [c_vp, c_i32]),
    "yb_predict_seg_u8_submit": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_f32, c_f32, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "yb_predict_u8_submit_gather": (c_i32, [c_vp, c_vp, c_i32, c_vp, c_i32, c_f32, c_f32, c_i32, c_vp, c_vp]),
    "yb_comm_handle_bytes": (c_i32, []),
    "yb_comm_create": (c_i32, [c_i32, c_i32, c_i32, C.c_int64, c_i32, C.POINTER(c_vp)]),
    "yb_comm_local_handle": (c_i32, [c_vp, c_vp]),
    "yb_comm_connect": (c_i32, [c_vp, c_vp]),
    "yb_comm_info": (c_i32, [c_vp, C.POINTER(c_i32), C.POINTER(c_i32), C.POINTER(C.c_int64), C.POINTER(c_i32)]),
    "yb_comm_send_buffer": (c_vp, [c_vp, c_i32]),
    "yb_comm_window": (c_vp, [c_vp, c_i32]),
    "yb_comm_allgather": (c_i32, [c_vp, c_i32, c_vp]),
    "yb_comm_release": (c_i32, [c_vp, c_i32, c_vp]),
    "yb_comm_destroy": (None, [c_vp]),
    "yb_comm_detection_payload_bytes": (C.c_int64, [c_i32, c_i32, c_i32]),
    "yb_num_ops": (c_i32, [c_vp]),
    "yb_debug_read_activation": (c_i32, [c_vp, c_i32, c_i32, c_vp, C.c_int64, C.POINTER(c_i32 * 3)]),
    "yb_op_name": (c_cp, [c_vp, c_i32]),
    "yb_launches_per_forward": (c_i32, [c_vp]),
    "yb_profile_forward": (c_i32, [c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_i32, c_vp]),
    "yb_time_op": (c_i32, [c_vp, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, c_i32, C.POINTER(c_f32), c_vp]),
    "yb_op_cost": (c_i32, [c_vp, c_i32, c_i32, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "yb_op_kind": (c_i32, [c_vp, c_i32]),
    "yb_debug_timeline": (c_i32, [c_vp, c_i32]),
    "yb_debug_conv_f16": (c_i32, [c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32,
                                  c_vp, c_i32, c_i32, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32,
                                  c_i32, c_f32, c_vp, c_vp, c_i32]),
    "yb_debug_bneck_f16": (c_i32, [c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp, c_i32, c_vp, c_vp, c_i32, c_i32, c_vp,
                                   c_i32, c_i32, c_vp, c_i32]),
    "yb_debug_conv_tf32": (c_i32, [c_i32, c_vp, c_i32, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_vp, c_vp,
                                   C.c_int64, c_vp, c_i32]),
    "yb_debug_conv_tf32_eval": (c_i32, [c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32,
                                        c_i32, c_vp, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_i32]),
}

_lib = None


class YbError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"{STATUS_NAMES.get(status, status)}: {msg}")
        self.status = status


def lib():
    """Load (once) the in-tree shared library; never builds, never falls back."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing - run `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(nvcc, sm_90a). yolosharp_b200 has no CPU fallback.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)  # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        _lib = l
    return _lib


def check(status):
    if status != YB_OK:
        raise YbError(status, lib().yb_last_error().decode("utf-8", "replace"))
