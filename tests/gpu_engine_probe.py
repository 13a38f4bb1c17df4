"""GPU bring-up probe for the fused engine: stage-by-stage comparison with the oracle on a small image,
teacher-forced checks of the integer stages, and per-stage timing at the headline shape.
  python tests/gpu_engine_probe.py parity | timing [batch]
"""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectorch_b200 import engine as E  # noqa: E402
from oracle import network as net  # noqa: E402
from oracle import ref  # noqa: E402

dev = torch.device("cuda:0")


def cmp(tag, got, want, tol=None):
    got = got.detach().cpu().double() if torch.is_tensor(got) else torch.as_tensor(np.asarray(got)).double()
    want = want.detach().cpu().double() if torch.is_tensor(want) else torch.as_tensor(np.asarray(want)).double()
    if got.shape != want.shape:
        print("CMP %-34s SHAPE MISMATCH got %s want %s" % (tag, tuple(got.shape), tuple(want.shape)), flush=True)
        return
    err = (got - want).abs().max().item() if got.numel() else 0.0
    mx = want.abs().max().item() if want.numel() else 0.0
    print("CMP %-34s max_abs_err %.3e  ref_max %.3e  rel %.3e %s" % (tag, err, mx, err / max(mx, 1e-30), "" if tol is None else ("OK" if err <= tol else "FAIL")), flush=True)


def nhwc_to_nchw(t):
    return t.permute(0, 3, 1, 2)


def parity(h=320, w=416, arch="resnet50"):
    P = net.synthetic_params(arch)
    img = net.synthetic_image(1, h, w)
    t0 = time.time()
    S = net.detect_and_mask_fpn(img, P, arch)
    print("oracle forward %.2fs; dets %d" % (time.time() - t0, len(S["scores_final"])), flush=True)
    eng = E.Engine(arch=arch, batch=1, height=h, width=w, emit_full_masks=True, det_cap=128, exact_roialign=True)
    eng.load_state_dict(P)
    eng.run(img.to(dev), 1.0)
    torch.cuda.synchronize()
    print("engine ran (exact_roialign=True)", flush=True)
    for i in range(4):
        cmp("C%d" % (i + 2), nhwc_to_nchw(eng.buffer("C%d" % (i + 2))), S["C"][i])
    for i in range(4):
        cmp("P%d" % (i + 2), nhwc_to_nchw(eng.buffer("P%d" % (i + 2))), S["P"][i])
    cmp("P6", nhwc_to_nchw(eng.buffer("P6")), S["P6"])
    for i in range(5):
        o = eng.buffer("rpn_out%d" % (i + 2))
        cmp("rpn_cls lvl%d" % i, nhwc_to_nchw(o[..., 0:3]), S["rpn"][i][0])
        cmp("rpn_box lvl%d" % i, nhwc_to_nchw(o[..., 3:15]), S["rpn"][i][1])
    cnt = eng.buffer("prop_counts")[0].cpu().numpy()
    print("prop counts engine", cnt.tolist(), "oracle", [len(p[0]) for p in S["props"]], flush=True)
    n = int(eng.buffer("roi_counts")[0].item())
    print("rois engine", n, "oracle", len(S["rois"]), flush=True)
    if n == len(S["rois"]):
        cmp("rois (e2e)", eng.buffer("rois")[0, :n, 1:5], S["rois"])
        lv = eng.buffer("roi_levels")[0, :n].cpu().numpy()
        print("levels equal:", np.array_equal(lv + 2, S["lvls"].astype(np.int32)), flush=True)
        cmp("cls_prob (e2e)", eng.buffer("cls_prob")[:n], S["cls_score"])
        cmp("bbox_pred (e2e)", eng.buffer("bbox_pred")[:n], S["bbox_pred"])
    dc = int(eng.buffer("det_counts")[0].item())
    print("dets engine", dc, "oracle", len(S["scores_final"]), flush=True)
    if dc == len(S["scores_final"]):
        cmp("det scores (e2e)", eng.buffer("det_scores")[0, :dc], S["scores_final"])
        cmp("det boxes (e2e)", eng.buffer("det_boxes")[0, :dc], S["boxes_final"])

    # ---------------- teacher forcing: oracle RPN maps -> proposals + collect must match bit-for-bit
    for i in range(5):
        o = eng.buffer("rpn_out%d" % (i + 2))
        o[..., 0:3] = S["rpn"][i][0].permute(0, 2, 3, 1).to(dev)
        o[..., 3:15] = S["rpn"][i][1].permute(0, 2, 3, 1).to(dev)
    eng.run(None, 1.0, E.ST_PROPOSALS, E.ST_COLLECT)
    torch.cuda.synchronize()
    cnt = eng.buffer("prop_counts")[0].cpu().numpy()
    print("TF prop counts engine", cnt.tolist(), "oracle", [len(p[0]) for p in S["props"]], flush=True)
    for i in range(5):
        k = min(int(cnt[i]), len(S["props"][i][0]))
        order = eng.buffer("rpn_order")[0, i, :len(S["props"][i][2]["order"])].cpu().numpy()
        print("TF lvl%d order equal: %s" % (i, np.array_equal(order, S["props"][i][2]["order"])), flush=True)
        cmp("TF props lvl%d" % i, eng.buffer("props")[0, i, :k], S["props"][i][0][:k])
        cmp("TF prop scores lvl%d" % i, eng.buffer("prop_scores")[0, i, :k], S["props"][i][1][:k, 0])
    n = int(eng.buffer("roi_counts")[0].item())
    if n == len(S["rois"]):
        r = eng.buffer("rois")[0, :n, 1:5].cpu()
        print("TF rois bit-equal:", torch.equal(r, S["rois"]), flush=True)
        cmp("TF rois", r, S["rois"])
        lv = eng.buffer("roi_levels")[0, :n].cpu().numpy()
        print("TF levels equal:", np.array_equal(lv + 2, S["lvls"].astype(np.int32)), flush=True)

    # ---------------- teacher forcing: oracle rois -> RoIAlign (P from engine replaced by oracle P)
    for i in range(4):
        eng.buffer("P%d" % (i + 2)).copy_(S["P"][i].permute(0, 2, 3, 1).to(dev))
    eng.buffer("rois")[0, :, 1:5] = 0
    eng.buffer("rois")[0, :len(S["rois"]), 1:5] = S["rois"].to(dev)
    eng.buffer("roi_levels")[0, :len(S["rois"])] = torch.from_numpy(S["lvls"].astype(np.int32) - 2).to(dev)
    eng.run(None, 1.0, E.ST_ROI_BOX, E.ST_BOX_HEAD)
    torch.cuda.synchronize()
    rf = eng.buffer("roi_feat")[:len(S["rois"])].permute(0, 3, 1, 2).cpu()
    print("TF roi_feat bit-equal:", torch.equal(rf, S["roi_feats"]), flush=True)
    cmp("TF cls_prob", eng.buffer("cls_prob")[:len(S["rois"])], S["cls_score"])
    cmp("TF bbox_pred", eng.buffer("bbox_pred")[:len(S["rois"])], S["bbox_pred"])

    # ---------------- teacher forcing: oracle class scores / deltas -> detections must match exactly
    nr = len(S["rois"])
    eng.buffer("cls_prob")[:nr] = S["cls_score"].to(dev)
    eng.buffer("bbox_pred")[:nr] = S["bbox_pred"].to(dev)
    eng.buffer("roi_counts")[0] = nr
    eng.run(None, 1.0, E.ST_DETECT, E.ST_DETECT)
    torch.cuda.synchronize()
    dc = int(eng.buffer("det_counts")[0].item())
    print("TF dets engine", dc, "oracle", len(S["scores_final"]), flush=True)
    if dc == len(S["scores_final"]):
        sc = eng.buffer("det_scores")[0, :dc].cpu().numpy()
        bx = eng.buffer("det_boxes")[0, :dc].cpu().numpy()
        cl = eng.buffer("det_classes")[0, :dc].cpu().numpy()
        want_cl = np.concatenate([np.full(len(S["cls_boxes"][j]), j) for j in range(1, 81)])
        print("TF det scores bit-equal:", np.array_equal(sc, S["scores_final"]), " classes equal:", np.array_equal(cl, want_cl), flush=True)
        cmp("TF det boxes", bx, S["boxes_final"])
    # ---------------- teacher forcing: oracle detections -> mask head
    if "masks" in S:
        D = len(S["boxes_final"])
        eng.buffer("det_boxes")[0].zero_()
        eng.buffer("det_boxes")[0, :D] = torch.from_numpy(S["boxes_final"]).to(dev)
        eng.buffer("det_counts")[0] = D
        eng.buffer("det_classes")[0, :D] = torch.from_numpy(want_cl.astype(np.int32)).to(dev) if dc == D else 1
        eng.run(None, 1.0, E.ST_MASK_ROIS, E.ST_MASK_OUT)
        torch.cuda.synchronize()
        mf = eng.buffer("mask_feat")[:D].permute(0, 3, 1, 2).cpu()
        print("TF mask roi feat bit-equal:", torch.equal(mf, S["mask_roi_feats"]), flush=True)
        cmp("TF mask probs", eng.buffer("masks_full")[:D], S["masks"])
        lg = eng.buffer("mask_logits")[:D, :, :, :81].permute(0, 3, 1, 2)
        cmp("TF mask logits", lg, S["mask_logits"], tol=1e-4)


def timing(batch=8, h=800, w=1216, arch="resnet50", passes=3):
    P = net.synthetic_params(arch)
    eng = E.Engine(arch=arch, batch=batch, height=h, width=w, passes=passes)
    eng.load_state_dict(P)
    img = net.synthetic_image(batch, h, w).to(dev)
    for _ in range(2):
        eng.run(img, 1.0)
    torch.cuda.synchronize()
    names = ["trunk", "fpn", "rpn", "proposals", "collect", "roi_box", "box_head", "detect", "mask_rois", "mask_roi_feat", "mask_head", "mask_out"]
    tot = 0.0
    for st in range(12):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 3
        ev0.record()
        for _ in range(reps):
            eng.run(img, 1.0, st, st)
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / reps
        tot += ms
        print("STAGE %-14s %8.3f ms  (launches %d)" % (names[st], ms, eng.count_launches(st, st)), flush=True)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(3):
        eng.run(img, 1.0)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / 3
    print("TOTAL batch %d: %.3f ms/step  -> %.1f img/s  (sum of stages %.3f) passes=%d  counts rois %s dets %s" % (
        batch, ms, batch * 1000.0 / ms, tot, passes, eng.buffer("roi_counts").cpu().tolist(), eng.buffer("det_counts").cpu().tolist()), flush=True)


def ops(batch=8, h=800, w=1216, arch="resnet50", **kw):
    P = net.synthetic_params(arch)
    eng = E.Engine(arch=arch, batch=batch, height=h, width=w, **kw)
    eng.load_state_dict(P)
    img = net.synthetic_image(batch, h, w).to(dev)
    for _ in range(3):
        eng.run(img, 1.0)
    torch.cuda.synchronize()
    acc = None
    reps = 5
    for _ in range(reps):
        pr = eng.profile(img, 1.0)
        acc = [list(x) for x in pr] if acc is None else [[a[0] + b[0]] + a[1:] for a, b in zip(acc, pr)]
    tot = sum(a[0] for a in acc) / reps
    for i, (ms, fl, st, bn) in enumerate(acc):
        ms /= reps
        print("OP %3d stage %2d bn %3d  %9.1f us  %8.2f GFLOP  %7.1f TFLOP/s alg" % (i, st, bn, ms * 1e3, fl / 1e9, fl / (ms * 1e-3) / 1e12 if ms > 0 else 0), flush=True)
    print("OPS total %.3f ms  %s" % (tot, kw), flush=True)


if __name__ == "__main__":
    print("device:", torch.cuda.get_device_name(0), flush=True)
    mode = sys.argv[1]
    if mode == "parity":
        parity()
    elif mode == "c4":
        # BASELINE configs[1]: Faster R-CNN R-50-C4, batch 1, 1000 RPN proposals (plus the 'upshare' mask head)
        P = net.synthetic_params("resnet50", fpn=False)
        eng = E.Engine(arch="resnet50", model="c4", batch=1, height=800, width=1216, pre_nms_top_n=6000, post_nms_top_n=1000)
        eng.load_state_dict(P)
        img = net.synthetic_image(1, 800, 1216).to(dev)
        for _ in range(3):
            eng.run(img, 1.0)
        torch.cuda.synchronize()
        for (a, b, tag) in ((0, 7, "faster_rcnn_c4 (trunk..detect)"), (0, 11, "mask_rcnn_c4 (trunk..masks)")):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                eng.run(img, 1.0, a, b)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            print("C4 %-34s batch 1: %.3f ms/img -> %.1f img/s; rois %s dets %s" % (tag, ms, 1000.0 / ms, eng.buffer("roi_counts").cpu().tolist(), eng.buffer("det_counts").cpu().tolist()), flush=True)
        pr = eng.profile(img, 1.0)
        fl = sum(f for (_, f, _, _) in pr); tm = sum(m for (m, f, _, bn) in pr if bn > 0)
        print("C4 conv launches: %.1f GFLOP algorithmic in %.3f ms = %.1f TFLOP/s" % (fl / 1e9, tm, fl / tm / 1e9), flush=True)
    elif mode == "ops":
        ops()
    elif mode == "timing":
        timing(int(sys.argv[2]) if len(sys.argv) > 2 else 8, passes=int(sys.argv[3]) if len(sys.argv) > 3 else 3)
    print("==== done", flush=True)
