"""One engine run under the kernel switches of the calling environment (DT_CONV_KIND, DT_PLANE_HANDOVER, DT_CONV_PDL, DT_RPN_SPLIT,
DT_RPN_NMS_SPLIT: they are read once per process), compared with the oracle: prints one JSON line with the
worst relative error over C2..C5 / P2..P6, the worst absolute error of the RPN maps and of the teacher-forced mask logits.
Run by tests/test_gpu_engine.py::test_conv_kernel_variants in a subprocess per setting."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectorch_b200 import engine as E  # noqa: E402
from oracle import network as net  # noqa: E402


def main():
    h, w = 320, 416
    dev = torch.device("cuda:0")
    P = net.synthetic_params("resnet50")
    img = net.synthetic_image(1, h, w)
    S = net.detect_and_mask_fpn(img, P)
    eng = E.Engine(arch="resnet50", batch=1, height=h, width=w, emit_full_masks=True, det_cap=128, exact_roialign=True)
    eng.load_state_dict(P)
    eng.run(img.to(dev), 1.0)
    torch.cuda.synchronize()

    def rel(got, want):
        got = got.detach().cpu().double(); want = want.double()
        return float((got - want).abs().max() / want.abs().max())

    def ab(got, want):
        return float((got.detach().cpu().double() - want.double()).abs().max())

    out = {"act_rel": 0.0, "rpn_abs": 0.0}
    for i in range(4):
        out["act_rel"] = max(out["act_rel"], rel(eng.buffer("C%d" % (i + 2)).permute(0, 3, 1, 2), S["C"][i]),
                             rel(eng.buffer("P%d" % (i + 2)).permute(0, 3, 1, 2), S["P"][i]))
    out["act_rel"] = max(out["act_rel"], rel(eng.buffer("P6").permute(0, 3, 1, 2), S["P6"]))
    for i in range(5):
        o = eng.buffer("rpn_out%d" % (i + 2))
        out["rpn_abs"] = max(out["rpn_abs"], ab(o[..., 0:3].permute(0, 3, 1, 2), S["rpn"][i][0]), ab(o[..., 3:15].permute(0, 3, 1, 2), S["rpn"][i][1]))
    # teacher-forced mask head (oracle feature maps and detections in, logits out)
    for i in range(4):
        eng.buffer("P%d" % (i + 2)).copy_(S["P"][i].permute(0, 2, 3, 1).to(dev))
    D = len(S["boxes_final"])
    want_cl = np.concatenate([np.full(len(S["cls_boxes"][j]), j) for j in range(1, 81)]).astype(np.int32)
    eng.buffer("det_boxes")[0].zero_()
    eng.buffer("det_boxes")[0, :D] = torch.from_numpy(S["boxes_final"]).to(dev)
    eng.buffer("det_counts")[0] = D
    eng.buffer("det_classes")[0, :D] = torch.from_numpy(want_cl).to(dev)
    eng.run(None, 1.0, E.ST_MASK_ROIS, E.ST_MASK_OUT)
    torch.cuda.synchronize()
    out["mask_logit_abs"] = ab(eng.buffer("mask_logits")[:D, :, :, :81].permute(0, 3, 1, 2), S["mask_logits"])
    out["range_flag"] = int(eng.buffer("range_flag").item())
    # un-forced proposals / detections of the first run (the proposal kernels have switches too)
    out["launches"] = eng.count_launches()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
