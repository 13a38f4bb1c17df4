"""ctypes binding of the C-ABI library (include/detectorch_b200.h).  There is NO fallback: if the
CUDA library is missing or fails to load, importing an operator raises."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DETECTORCH_B200_LIB selects another build of the same library (A/B experiments with compile-time kernel switches); default: the in-tree build
LIB_PATH = os.environ.get("DETECTORCH_B200_LIB") or os.path.join(_HERE, "csrc", "libdetectorch_b200.so")
_lib = None

c_void_p, c_int, c_int64, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float

# symbol -> (restype, argtypes); mirrors include/detectorch_b200.h
SIGNATURES = {
    "dt_version": (ctypes.c_char_p, []),
    "launch_roi_align_forward_cuda": (c_int, [c_int, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_int, c_int, c_int,
                                              c_void_p, c_void_p]),
    "launch_roi_align_backward_cuda": (c_int, [c_int, c_void_p, c_int, c_float, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                               c_int, c_void_p]),
    "dt_roi_align_forward_nchw": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int,
                                          c_void_p, c_void_p]),
    "dt_roi_align_fast_workspace_bytes": (c_int64, [c_int, c_int, c_int, c_int, c_int64, c_int, c_int]),
    "dt_roi_align_forward_nchw_fast": (c_int, [c_void_p, c_int, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int,
                                               c_void_p, c_void_p, c_void_p]),
    "dt_roi_align_forward_nhwc": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int,
                                          c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "dt_nms_workspace_bytes": (c_int64, [c_int64]),
    "dt_nms": (c_int, [c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_segm_workspace_bytes": (c_int64, [c_int, c_int]),
    "dt_segm_strings_bytes": (c_int64, [c_int, c_int]),
    "dt_segm_rle": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float,
                            c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_segm_batch_workspace_bytes": (c_int64, [c_int, c_int, c_int]),
    "dt_segm_batch_strings_bytes": (c_int64, [c_int, c_int, c_int]),
    "dt_segm_rle_batch": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_int,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_segm_rle_batch_append": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_int,
                                         c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_segm_paste": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float,
                              c_void_p, c_void_p]),
    "dt_roi_align_backward_det_workspace_bytes": (c_int64, [c_int64, c_int64]),
    "dt_roi_align_backward_plan": (c_int, [c_void_p, c_int64, c_int, c_float, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "dt_roi_align_backward_deterministic": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int,
                                                    c_int64, c_void_p, c_void_p, c_void_p]),
    "dt_prep_image": (c_int, [c_void_p, c_int, c_int, c_void_p, ctypes.c_double, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "dt_tf32_residual": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "dt_fp16_split": (c_int, [c_void_p, c_int64, c_float, c_void_p, c_void_p, c_void_p]),
    "dt_conv2d_nhwc_f16x3": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                     c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                     c_void_p, c_int, c_void_p]),
    "dt_conv2d_nhwc": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                               c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                               c_void_p, c_int, c_void_p]),
    "dt_conv2d_nhwc_two_phase": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                         c_void_p, c_void_p]),
    "dt_coco_gt_workspace_bytes": (c_int64, [c_int64, c_int64, c_int64]),
    "dt_coco_gt_build": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p]),
    "dt_coco_det_check": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_coco_eval_workspace_bytes": (c_int64, [c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int]),
    "dt_coco_eval": (c_int, [c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int64,
                             c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_void_p, c_void_p]),
    "dt_coco_eval_imgs": (c_int, [c_int, c_int, c_void_p, c_int, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_void_p]),
    "dt_coco_results_append": (c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p,
                                       c_void_p, c_void_p, c_void_p]),
    "dt_coco_results_count": (c_int, [c_int64, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int64, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "dt_coco_results_write": (c_int, [c_int64, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                      c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_coco_json": (c_int, [c_int, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_void_p, c_void_p]),
    "dt_coco_file_struct_workspace_bytes": (c_int64, [c_int64]),
    "dt_coco_file_struct": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_coco_file_separators": (c_int, [c_int64, c_void_p, c_void_p, c_void_p]),
    "dt_coco_file_records": (c_int, [c_int64, c_int64, c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_coco_file_finish_workspace_bytes": (c_int64, [c_int64, c_int64, c_int]),
    "dt_coco_file_finish": (c_int, [c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p,
                                    c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "dt_proposal_recall_smem_bytes": (c_int64, [c_int, c_int64]),
    "dt_proposal_recall": (c_int, [c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64,
                                   c_void_p, c_void_p, c_void_p]),
}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("detectorch_b200: %s not built. Run `python -m detectorch_b200.build` "
                               "(or __graft_entry__.build()). There is no CPU fallback." % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)   # AttributeError if the library does not export a declared symbol
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(ok, what):
    if ok != 1:
        raise RuntimeError("detectorch_b200: %s failed (see stderr)" % what)
