"""The reference's torch-0.4 flavour of the native op: a module named `roialign` with the pybind11 entry points of
lib/cppcuda/roi_align_binding.cpp:7-12 / roi_align_cuda.h:4-22 (JIT-loaded by lib/model/roi_align.py:11-18 when torch is 0.4) --
callee-allocates convention, argument order and AT_CHECK conditions (-> RuntimeError) as in
lib/cppcuda/roi_align_forward_cuda.cu:162-212 and roi_align_backward_cuda.cu:210-260, over the sm_90a kernels."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectorch_b200 import ops  # noqa: E402


def _check(cond, msg):
    if not cond:
        raise RuntimeError(msg)       # AT_CHECK -> C++ exception -> Python RuntimeError


def roi_align_forward_cuda(input, bottom_rois, pooled_height, pooled_width, spatial_scale, sampling_ratio):
    _check(input.dim() == 4, "Input to RoI Align should be a NCHW Tensor")
    _check(bottom_rois.dim() == 2, "RoI Proposals should be a 2D Tensor, (batch_sz x proposals)")
    _check(bottom_rois.size(1) == 5, "Proposals should be of the form [batch_index startW startH endW enH]")
    _check(input.is_contiguous(), "input must be contiguous")
    _check(bottom_rois.is_contiguous(), "bottom_rois must be contiguous")
    _check(input.is_cuda and bottom_rois.is_cuda, "roi_align_forward_cuda: CUDA tensors required")
    return ops.roi_align_forward_nchw(input, bottom_rois, int(pooled_height), int(pooled_width), float(spatial_scale), int(sampling_ratio))


def roi_align_backward_cuda(bottom_rois, grad_output, b_size, channels, height, width, pooled_height, pooled_width, spatial_scale, sampling_ratio):
    _check(bottom_rois.dim() == 2, "RoI Proposals should be a 2D Tensor, (batch_sz x proposals)")
    _check(bottom_rois.size(1) in (4, 5), "RoI Proposals should have 4 or 5 columns")
    _check(bottom_rois.is_contiguous(), "bottom_rois must be contiguous")
    _check(bottom_rois.is_cuda and grad_output.is_cuda, "roi_align_backward_cuda: CUDA tensors required")
    return ops.roi_align_backward_nchw(bottom_rois, grad_output.contiguous(), (int(b_size), int(channels), int(height), int(width)),
                                       int(pooled_height), int(pooled_width), float(spatial_scale), int(sampling_ratio))


def roi_align_forward_cpu(*args, **kwargs):
    raise RuntimeError("detectorch_b200 has no CPU RoIAlign (the reference CPU loop is the parity oracle, oracle/_ref)")


def roi_align_backward_cpu(*args, **kwargs):
    raise RuntimeError("detectorch_b200 has no CPU RoIAlign (the reference CPU loop is the parity oracle, oracle/_ref)")
