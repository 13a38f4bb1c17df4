"""Mirror of the hot-path part of the reference lib/utils/boxes.py: nms (:332-336) backed by the
sm_90a NMS kernel, numpy in / numpy out like the reference."""
import numpy as np
import torch

from .. import ops


def nms(dets, thresh):
    """Apply classic DPM-style greedy NMS.  dets [N,5] float32 numpy (or CUDA tensor) -> ascending kept indices."""
    if dets.shape[0] == 0:
        return []
    if torch.is_tensor(dets):
        return ops.nms(dets, thresh)
    d = torch.from_numpy(np.ascontiguousarray(dets, dtype=np.float32)).cuda()
    return ops.nms(d, float(thresh)).cpu().numpy()
