"""Drop-in mirror of the reference op wrapper lib/model/roi_align.py (RoIAlignFunction :23-145,
RoIAlign :150-169, preprocess_rois :172-188) over the sm_90a kernel.  Same names, argument order
and error behaviour; CUDA only (the reference's CPU branch is the parity oracle, not a product path)."""
import os

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable
from torch.nn.modules.module import Module

from .. import ops


class RoIAlignFunction(Function):
    @staticmethod
    def forward(ctx, features, rois, pooled_height, pooled_width, spatial_scale, sampling_ratio):
        ctx.rois = rois
        ctx.features_size = features.size()
        ctx.pooled_height, ctx.pooled_width = pooled_height, pooled_width
        ctx.spatial_scale, ctx.sampling_ratio = spatial_scale, sampling_ratio
        if features.is_cuda != rois.is_cuda:
            raise TypeError('features and rois should be on same device (CPU or GPU)')   # roi_align.py:43-44
        if not features.is_cuda:
            raise TypeError('detectorch_b200 RoIAlign runs on CUDA tensors only (no CPU fallback)')
        # the reference kernel requires NCHW-contiguous input (roi_align_forward_cuda.cu:189)
        return ops.roi_align_forward_nchw(features.contiguous(), rois.contiguous(), int(pooled_height), int(pooled_width),
                                          float(spatial_scale), int(sampling_ratio))

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        """Gradient w.r.t. the features (roi_align.py:91-147): zero-initialised [B,C,H,W] that the pooled gradient is scattered into.
        Default: the DETERMINISTIC kernel (every cell summed in the order of the reference's CPU backward: bit-identical to it, bit-reproducible
        training steps).  DT_ROIALIGN_BACKWARD=atomic selects the reference GPU kernel's fp32 atomic scatter (faster, order-dependent last bits)."""
        if not grad_output.is_cuda:
            raise TypeError('detectorch_b200 RoIAlign runs on CUDA tensors only (no CPU fallback)')
        fn = ops.roi_align_backward_nchw if os.environ.get("DT_ROIALIGN_BACKWARD", "deterministic") == "atomic" else ops.roi_align_backward_nchw_deterministic
        grad_input = fn(ctx.rois.contiguous(), grad_output.contiguous().float(), tuple(ctx.features_size),
                        int(ctx.pooled_height), int(ctx.pooled_width), float(ctx.spatial_scale), int(ctx.sampling_ratio))
        return grad_input, None, None, None, None, None


class RoIAlign(Module):
    def __init__(self, pooled_height, pooled_width, spatial_scale, sampling_ratio=0):
        super(RoIAlign, self).__init__()
        self.pooled_height = int(pooled_height)
        self.pooled_width = int(pooled_width)
        self.spatial_scale = float(spatial_scale)
        self.sampling_ratio = int(sampling_ratio)

    def forward(self, features, rois):
        rois = preprocess_rois(rois)
        return RoIAlignFunction.apply(features, rois, self.pooled_height, self.pooled_width, self.spatial_scale, self.sampling_ratio)


def preprocess_rois(rois):
    """list -> cat; [1,R,4|5] -> squeeze; [R,4] -> prepend a zero batch column (roi_align.py:172-188)."""
    if isinstance(rois, list):
        rois = torch.cat(tuple(rois), 0)
    if torch.is_tensor(rois):
        if rois.dim() == 3:
            if rois.size(0) == 1:
                rois = rois.squeeze(0)
            else:
                raise RuntimeError("rois has wrong size")
        if rois.size(1) == 4:
            zeros = torch.zeros((rois.size(0), 1), dtype=rois.dtype, device=rois.device)
            rois = torch.cat((zeros, rois), 1).contiguous()
    return rois
