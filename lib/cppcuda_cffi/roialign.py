"""`cppcuda_cffi.roialign` with the reference's cffi calling convention (caller allocates and zeroes `output`,
lib/cppcuda_cffi/src/roi_align_forward_cuda.h:1-7) so that the UNMODIFIED reference lib/model/roi_align.py
(which imports this module on torch != 0.4, roi_align.py:20) runs on the sm_90a kernel."""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from detectorch_b200 import _lib  # noqa: E402


def roi_align_forward_cuda(input, rois, output, pooled_height, pooled_width, spatial_scale, sampling_ratio):
    if not (input.is_cuda and rois.is_cuda and output.is_cuda):
        raise TypeError("roi_align_forward_cuda: CUDA tensors required")
    input, rois = input.contiguous(), rois.contiguous()
    ok = _lib.lib().dt_roi_align_forward_nchw(input.data_ptr(), rois.data_ptr(), rois.size(0), rois.size(1), input.size(1), input.size(2),
                                              input.size(3), int(pooled_height), int(pooled_width), float(spatial_scale), int(sampling_ratio),
                                              output.data_ptr(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return 1 if ok == 1 else 0


def roi_align_forward_cpu(*args, **kwargs):
    raise RuntimeError("detectorch_b200 has no CPU RoIAlign (the reference CPU loop is the parity oracle, oracle/_ref)")


def roi_align_backward_cuda(rois, grad_output, grad_input, pooled_height, pooled_width, spatial_scale, sampling_ratio):
    """cffi convention of lib/cppcuda_cffi/src/roi_align_backward_cuda.h:1-7: the caller allocates and zeroes `grad_input` [B,C,H,W]
    (lib/model/roi_align.py:117); the pooled gradient is scattered into it."""
    if not (rois.is_cuda and grad_output.is_cuda and grad_input.is_cuda):
        raise TypeError("roi_align_backward_cuda: CUDA tensors required")
    rois, grad_output = rois.contiguous(), grad_output.contiguous()
    ok = _lib.lib().launch_roi_align_backward_cuda(int(grad_output.numel() & 0x7fffffff), grad_output.data_ptr(), rois.size(0), float(spatial_scale),
                                                   grad_input.size(1), grad_input.size(2), grad_input.size(3), int(pooled_height), int(pooled_width),
                                                   int(sampling_ratio), grad_input.data_ptr(), rois.data_ptr(), rois.size(1),
                                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return 1 if ok == 1 else 0
