"""GPU parity at the BENCHED configuration and sizes (BASELINE.json configs[1..4]):

  * Mask R-CNN R-50-FPN, 3x800x1216, batch 2 of distinct images, exactly the engine bench.py times
    (conv_kind f16, fast RoIAlign, det_cap 100, no full-mask materialisation) against
    oracle.network.detect_and_mask_fpn per image: activations, RPN outputs, teacher-forced integer
    stages bit-exact, mask logits < 1e-4 absolute, un-forced detections as matched sets;
  * Faster R-CNN R-50-C4 at 800x1216 (the 6000-of-57000 argpartition branch of generate_proposals.py:80-86);
  * Mask R-CNN R-101-FPN at 800x1216, one image;
  * RoIAlign 100k RoIs x 256 ch x 50x68 (configs[4]) against the oracle on a 2k-RoI subsample;
  * NMS of 100k boxes against oracle/nms_ref.c (bit-exact kept ids).

Tolerances are BASELINE.json's: bit-exact for sorted indices / kept ids, 1e-4 for fp32 (relative to the tensor's
max-abs for activations, absolute for probabilities and mask logits)."""
import numpy as np
import pytest
import torch

import os

pytestmark = pytest.mark.gpu
H, W = 800, 1216


def report(line):
    """Measured errors (shown with pytest -s); never fails a test."""
    print(line)


def _t(x):
    return x.detach().cpu().double() if torch.is_tensor(x) else torch.as_tensor(np.asarray(x)).double()


def rel_err(got, want):
    got, want = _t(got), _t(want)
    assert got.shape == want.shape, (got.shape, want.shape)
    return (got - want).abs().max().item() / max(1.0, want.abs().max().item())


def abs_err(got, want):
    got, want = _t(got), _t(want)
    assert got.shape == want.shape, (got.shape, want.shape)
    return (got - want).abs().max().item() if got.numel() else 0.0


def assert_same_order_up_to_ties(got, want, scores_of):
    """Sorted-index parity: identical wherever the sort key is unique; inside a run of EQUAL keys the reference's own order is
    implementation-defined (numpy's argsort / argpartition are unstable, generate_proposals.py:77-86), so a run is compared as a set."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape
    sg, sw = scores_of(got), scores_of(want)
    assert np.array_equal(sg, sw), "the key sequence along the order differs"
    if np.array_equal(got, want):
        return 0
    bounds = np.flatnonzero(np.diff(sw) != 0) + 1
    ties = 0
    for a, b in zip(np.r_[0, bounds], np.r_[bounds, len(sw)]):
        if b - a > 1:
            ties += 1
            assert np.array_equal(np.sort(got[a:b]), np.sort(want[a:b]))
        else:
            assert got[a] == want[a]
    return ties


def assert_rows_equal_up_to_ties(got, want, tol, max_moved, extra=None):
    """Row-wise equality of two [n,k] arrays, except that at most `max_moved` rows may sit at permuted positions (members of equal-score
    runs, see assert_same_order_up_to_ties); the displaced rows must still be the same set.  `extra` = (got_col, want_col) integer
    columns that must follow the same permutation (the FPN level of each RoI)."""
    got, want = _t(got).numpy(), _t(want).numpy()
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.abs(got - want).max(1) > tol
    assert int(bad.sum()) <= max_moved, "%d rows differ, only %d belong to equal-score runs" % (int(bad.sum()), max_moved)
    if extra is not None:
        assert np.array_equal(np.asarray(extra[0])[~bad], np.asarray(extra[1])[~bad])
    if bad.any():
        g, w = got[bad], want[bad]
        ge = np.asarray(extra[0])[bad][:, None].astype(np.float64) if extra is not None else np.zeros((len(g), 0))
        we = np.asarray(extra[1])[bad][:, None].astype(np.float64) if extra is not None else np.zeros((len(w), 0))
        g, w = np.hstack([g, ge]), np.hstack([w, we])
        g = g[np.lexsort(np.round(g, 1).T[::-1])]
        w = w[np.lexsort(np.round(w, 1).T[::-1])]
        assert np.abs(g - w).max() <= tol


def match_detections(sc, bx, S, box_tol=2e-2, score_tol=1e-4):
    n = len(sc)
    assert n == len(S["scores_final"])
    used = np.zeros(n, bool)
    for s, b in zip(S["scores_final"], S["boxes_final"]):
        d = np.abs(bx - b).max(1) + 1e3 * np.abs(sc - s) + 1e9 * used
        j = int(d.argmin())
        assert np.abs(bx[j] - b).max() < box_tol and abs(sc[j] - s) < score_tol
        used[j] = True


# ------------------------------------------------------------------------------------------ configs[2]: Mask R-CNN R-50-FPN as benched
@pytest.fixture(scope="module")
def fpn_ctx(built):
    assert torch.cuda.is_available()
    from detectorch_b200 import engine as E
    from oracle import network as net
    dev = torch.device("cuda:0")
    P = net.synthetic_params("resnet50")
    imgs = [net.synthetic_image(1, H, W, seed=s) for s in (0, 1)]
    S = [net.detect_and_mask_fpn(im, P) for im in imgs]
    # exactly bench.py's engine: defaults (conv_kind f16, exact_roialign False), det_cap 100, no full masks
    eng = E.Engine(arch="resnet50", batch=2, height=H, width=W, det_cap=100, use_mask=True, emit_full_masks=False)
    assert eng.cfg.conv_kind == 0 and eng.cfg.exact_roialign == 0
    eng.load_state_dict(P)
    eng.run(torch.cat(imgs, 0).to(dev), 1.0)
    torch.cuda.synchronize()
    eng.check_range()
    keys = ["C2", "C3", "C4", "C5", "P2", "P3", "P4", "P5", "P6"] + ["rpn_out%d" % l for l in range(2, 7)] + \
           ["roi_counts", "det_scores", "det_boxes", "det_classes", "det_counts", "masks"]
    snap = {k: eng.buffer(k).cpu().clone() for k in keys}
    return {"E": E, "eng": eng, "S": S, "P": P, "dev": dev, "snap": snap}


def test_fpn_fullsize_activations(fpn_ctx):
    S, snap = fpn_ctx["S"], fpn_ctx["snap"]
    for b in range(2):
        for i in range(4):
            ec = rel_err(snap["C%d" % (i + 2)][b:b + 1].permute(0, 3, 1, 2), S[b]["C"][i])
            ep = rel_err(snap["P%d" % (i + 2)][b:b + 1].permute(0, 3, 1, 2), S[b]["P"][i])
            report("R-50-FPN 800x1216 batch-2 image %d: C%d rel %.2e  P%d rel %.2e" % (b, i + 2, ec, i + 2, ep))
            assert ec < 1e-4 and ep < 1e-4, ("C/P", i + 2, b)
        assert rel_err(snap["P6"][b:b + 1].permute(0, 3, 1, 2), S[b]["P6"]) < 1e-4
        for i in range(5):
            o = snap["rpn_out%d" % (i + 2)][b:b + 1]
            e0, e1 = abs_err(o[..., 0:3].permute(0, 3, 1, 2), S[b]["rpn"][i][0]), abs_err(o[..., 3:15].permute(0, 3, 1, 2), S[b]["rpn"][i][1])
            report("R-50-FPN 800x1216 batch-2 image %d: RPN level P%d objectness abs %.2e  deltas abs %.2e" % (b, i + 2, e0, e1))
            assert e0 < 1e-4        # objectness probabilities
            assert e1 < 1e-4        # box deltas


def test_fpn_fullsize_unforced_detections(fpn_ctx):
    """R = 1000 proposals and D = 100 detections per image (the workload bench.py claims), detections matched as sets."""
    S, snap = fpn_ctx["S"], fpn_ctx["snap"]
    for b in range(2):
        assert int(snap["roi_counts"][b]) == len(S[b]["rois"]) == 1000
        n = int(snap["det_counts"][b])
        assert n == len(S[b]["scores_final"]) == 100
        match_detections(snap["det_scores"][b, :n].numpy(), snap["det_boxes"][b, :n].numpy(), S[b])


def test_fpn_fullsize_teacher_forced_proposals(fpn_ctx):
    E, eng, S, dev = fpn_ctx["E"], fpn_ctx["eng"], fpn_ctx["S"], fpn_ctx["dev"]
    for b in range(2):
        for i in range(5):
            o = eng.buffer("rpn_out%d" % (i + 2))
            o[b, ..., 0:3] = S[b]["rpn"][i][0][0].permute(1, 2, 0).to(dev)
            o[b, ..., 3:15] = S[b]["rpn"][i][1][0].permute(1, 2, 0).to(dev)
    eng.run(None, 1.0, E.ST_PROPOSALS, E.ST_COLLECT)
    torch.cuda.synchronize()
    for b in range(2):
        cnt = eng.buffer("prop_counts")[b].cpu().numpy()
        assert cnt.tolist() == [len(p[0]) for p in S[b]["props"]]
        tied = 0
        for i in range(5):
            order = S[b]["props"][i][2]["order"]
            sc = S[b]["rpn"][i][0][0].permute(1, 2, 0).reshape(-1).numpy()
            assert_same_order_up_to_ties(eng.buffer("rpn_order")[b, i, :len(order)].cpu().numpy(), order, lambda o: sc[o])
            so = sc[order]
            eq = np.r_[False, np.diff(so) == 0]
            lvl_tied = int((eq | np.r_[eq[1:], False]).sum())        # members of equal-score runs on this level
            tied += lvl_tied
            k = int(cnt[i])
            assert torch.equal(eng.buffer("prop_scores")[b, i, :k].cpu(), S[b]["props"][i][1][:k, 0])     # kept ids: identical score sequence
            assert_rows_equal_up_to_ties(eng.buffer("props")[b, i, :k], S[b]["props"][i][0][:k], 2e-4, lvl_tied)    # expf ulp
        n = int(eng.buffer("roi_counts")[b])
        assert n == len(S[b]["rois"])
        assert_rows_equal_up_to_ties(eng.buffer("rois")[b, :n, 1:5], S[b]["rois"], 2e-4, tied,
                                     extra=(eng.buffer("roi_levels")[b, :n].cpu().numpy() + 2, S[b]["lvls"].astype(np.int32)))


def _force_rois(eng, S, dev):
    for b in range(2):
        for i in range(4):
            eng.buffer("P%d" % (i + 2))[b].copy_(S[b]["P"][i][0].permute(1, 2, 0).to(dev))
        n = len(S[b]["rois"])
        eng.buffer("rois")[b, :, 1:5] = 0
        eng.buffer("rois")[b, :n, 1:5] = S[b]["rois"].to(dev)
        eng.buffer("roi_levels")[b, :n] = torch.from_numpy(S[b]["lvls"].astype(np.int32) - 2).to(dev)
        eng.buffer("roi_counts")[b] = n


def test_fpn_fullsize_teacher_forced_box_head(fpn_ctx):
    E, eng, S, dev = fpn_ctx["E"], fpn_ctx["eng"], fpn_ctx["S"], fpn_ctx["dev"]
    _force_rois(eng, S, dev)
    eng.run(None, 1.0, E.ST_ROI_BOX, E.ST_BOX_HEAD)
    torch.cuda.synchronize()
    R = eng.cfg.post_nms_top_n
    for b in range(2):
        n = len(S[b]["rois"])
        rf = eng.buffer("roi_feat")[b * R:b * R + n].permute(0, 3, 1, 2)
        assert abs_err(rf, S[b]["roi_feats"]) < 1e-5 * max(1.0, S[b]["roi_feats"].abs().max().item())     # fast RoIAlign: fp32 re-association only
        assert abs_err(eng.buffer("cls_prob")[b * R:b * R + n], S[b]["cls_score"]) < 1e-4
        assert rel_err(eng.buffer("bbox_pred")[b * R:b * R + n], S[b]["bbox_pred"]) < 1e-4


def test_fpn_fullsize_teacher_forced_detect(fpn_ctx):
    E, eng, S, dev = fpn_ctx["E"], fpn_ctx["eng"], fpn_ctx["S"], fpn_ctx["dev"]
    _force_rois(eng, S, dev)
    R = eng.cfg.post_nms_top_n
    for b in range(2):
        n = len(S[b]["rois"])
        eng.buffer("cls_prob")[b * R:b * R + n] = S[b]["cls_score"].to(dev)
        eng.buffer("bbox_pred")[b * R:b * R + n] = S[b]["bbox_pred"].to(dev)
    eng.run(None, 1.0, E.ST_DETECT, E.ST_DETECT)
    torch.cuda.synchronize()
    for b in range(2):
        d = int(eng.buffer("det_counts")[b])
        assert d == len(S[b]["scores_final"])
        want_cls = np.concatenate([np.full(len(S[b]["cls_boxes"][j]), j) for j in range(1, 81)])
        assert np.array_equal(eng.buffer("det_scores")[b, :d].cpu().numpy(), S[b]["scores_final"])        # kept ids / order: bit-exact
        assert np.array_equal(eng.buffer("det_classes")[b, :d].cpu().numpy(), want_cls)
        assert abs_err(eng.buffer("det_boxes")[b, :d], S[b]["boxes_final"]) < 2e-4


def test_fpn_fullsize_teacher_forced_mask_head(fpn_ctx):
    E, eng, S, dev = fpn_ctx["E"], fpn_ctx["eng"], fpn_ctx["S"], fpn_ctx["dev"]
    _force_rois(eng, S, dev)
    cap = eng.cfg.det_cap
    for b in range(2):
        D = len(S[b]["boxes_final"])
        want_cls = np.concatenate([np.full(len(S[b]["cls_boxes"][j]), j) for j in range(1, 81)])
        eng.buffer("det_boxes")[b].zero_()
        eng.buffer("det_boxes")[b, :D] = torch.from_numpy(S[b]["boxes_final"]).to(dev)
        eng.buffer("det_counts")[b] = D
        eng.buffer("det_classes")[b, :D] = torch.from_numpy(want_cls.astype(np.int32)).to(dev)
    eng.run(None, 1.0, E.ST_MASK_ROIS, E.ST_MASK_OUT)
    torch.cuda.synchronize()
    for b in range(2):
        D = len(S[b]["boxes_final"])
        want_cls = np.concatenate([np.full(len(S[b]["cls_boxes"][j]), j) for j in range(1, 81)])
        mf = eng.buffer("mask_feat")[b * cap:b * cap + D].permute(0, 3, 1, 2)
        assert abs_err(mf, S[b]["mask_roi_feats"]) < 1e-5 * max(1.0, S[b]["mask_roi_feats"].abs().max().item())
        lg = eng.buffer("mask_logits")[b * cap:b * cap + D, :, :, :81].permute(0, 3, 1, 2)
        e = abs_err(lg, S[b]["mask_logits"])
        report("R-50-FPN 800x1216 batch-2 image %d (teacher-forced): mask logits abs err %.3e (|logit| max %.2f)" % (b, e, S[b]["mask_logits"].abs().max().item()))
        assert e < 1e-4                                                                                   # north_star: 1e-4 on mask logits
        own = eng.buffer("masks")[b * cap:b * cap + D].cpu().numpy()
        assert np.abs(own - S[b]["masks"].numpy()[np.arange(D), want_cls]).max() < 1e-4


# ------------------------------------------------------------------------------------------ configs[1]: Faster R-CNN R-50-C4 at 800x1216
def test_c4_fullsize_faster_rcnn(built):
    """57 000 anchors > pre_nms_top_n = 6000: the argpartition + argsort branch of generate_proposals.py:80-86 (never reached at the
    small test sizes), then RoIAlign with the adaptive grid on 1000 proposals, the res5 head and the detection post-processing."""
    from detectorch_b200 import engine as E
    from oracle import network as net
    dev = torch.device("cuda:0")
    P = net.synthetic_params("resnet50", fpn=False, mask=False)
    img = net.synthetic_image(1, H, W)
    S = net.detect_and_mask_c4(img, P, use_mask=False)
    eng = E.Engine(arch="resnet50", model="c4", batch=1, height=H, width=W, pre_nms_top_n=6000, post_nms_top_n=1000, det_cap=100, use_mask=False,
                   exact_roialign=True)
    eng.load_state_dict(P)
    eng.run(img.to(dev), 1.0)
    torch.cuda.synchronize()
    eng.check_range()
    assert rel_err(eng.buffer("C4").permute(0, 3, 1, 2), S["C4"]) < 1e-4
    o = eng.buffer("rpn_out4")
    assert o.shape[1] * o.shape[2] * 15 == 57000
    assert abs_err(o[..., 0:15].permute(0, 3, 1, 2), S["rpn"][0]) < 1e-4 and abs_err(o[..., 15:75].permute(0, 3, 1, 2), S["rpn"][1]) < 1e-4
    n = int(eng.buffer("det_counts")[0])
    match_detections(eng.buffer("det_scores")[0, :n].cpu().numpy(), eng.buffer("det_boxes")[0, :n].cpu().numpy(), S)
    # teacher-forced proposals: the 6000-of-57000 select, order and kept set
    o[..., 0:15] = S["rpn"][0].permute(0, 2, 3, 1).to(dev)
    o[..., 15:75] = S["rpn"][1].permute(0, 2, 3, 1).to(dev)
    eng.run(None, 1.0, E.ST_PROPOSALS, E.ST_COLLECT)
    torch.cuda.synchronize()
    n = int(eng.buffer("roi_counts")[0])
    assert n == len(S["rois"]) == 1000
    order = S["props"][2]["order"]
    assert len(order) == 6000
    sc = S["rpn"][0][0].permute(1, 2, 0).reshape(-1).numpy()
    assert_same_order_up_to_ties(eng.buffer("rpn_order")[0, 0, :6000].cpu().numpy(), order, lambda x: sc[x])
    assert torch.equal(eng.buffer("prop_scores")[0, 0, :n].cpu(), S["props"][1][:n, 0])
    so = sc[order]
    eq = np.r_[False, np.diff(so) == 0]
    assert_rows_equal_up_to_ties(eng.buffer("rois")[0, :n, 1:5], S["rois"], 2e-4, int((eq | np.r_[eq[1:], False]).sum()))
    # teacher-forced RoIAlign (adaptive grid, bit-exact) + res5 head + detections
    eng.buffer("C4").copy_(S["C4"].permute(0, 2, 3, 1).to(dev))
    eng.buffer("rois")[0, :, 1:5] = 0
    eng.buffer("rois")[0, :n, 1:5] = S["rois"].to(dev)
    eng.run(None, 1.0, E.ST_ROI_BOX, E.ST_BOX_HEAD)
    torch.cuda.synchronize()
    assert torch.equal(eng.buffer("roi_feat")[:n].permute(0, 3, 1, 2).cpu(), S["roi_feats"])
    assert rel_err(eng.buffer("pooled")[:n], S["pooled"]) < 1e-4
    assert abs_err(eng.buffer("cls_prob")[:n], S["cls_score"]) < 1e-4 and rel_err(eng.buffer("bbox_pred")[:n], S["bbox_pred"]) < 1e-4
    eng.buffer("cls_prob")[:n] = S["cls_score"].to(dev)
    eng.buffer("bbox_pred")[:n] = S["bbox_pred"].to(dev)
    eng.run(None, 1.0, E.ST_DETECT, E.ST_DETECT)
    torch.cuda.synchronize()
    d = int(eng.buffer("det_counts")[0])
    assert d == len(S["scores_final"]) and np.array_equal(eng.buffer("det_scores")[0, :d].cpu().numpy(), S["scores_final"])


# ------------------------------------------------------------------------------------------ configs[3] model: Mask R-CNN R-101-FPN at 800x1216
def test_r101_fullsize(built):
    from detectorch_b200 import engine as E
    from oracle import network as net
    dev = torch.device("cuda:0")
    P = net.synthetic_params("resnet101")
    img = net.synthetic_image(1, H, W, seed=3)
    S = net.detect_and_mask_fpn(img, P, arch="resnet101")
    eng = E.Engine(arch="resnet101", batch=1, height=H, width=W, det_cap=100)
    eng.load_state_dict(P)
    eng.run(img.to(dev), 1.0)
    torch.cuda.synchronize()
    eng.check_range()
    for i in range(4):
        assert rel_err(eng.buffer("C%d" % (i + 2)).permute(0, 3, 1, 2), S["C"][i]) < 1e-4
        assert rel_err(eng.buffer("P%d" % (i + 2)).permute(0, 3, 1, 2), S["P"][i]) < 1e-4
    for i in range(5):
        o = eng.buffer("rpn_out%d" % (i + 2))
        assert abs_err(o[..., 0:3].permute(0, 3, 1, 2), S["rpn"][i][0]) < 1e-4
    n = int(eng.buffer("det_counts")[0])
    match_detections(eng.buffer("det_scores")[0, :n].cpu().numpy(), eng.buffer("det_boxes")[0, :n].cpu().numpy(), S)
    # masks of the matched detections: teacher-force the oracle's detections, compare the logits
    D = len(S["boxes_final"])
    want_cls = np.concatenate([np.full(len(S["cls_boxes"][j]), j) for j in range(1, 81)])
    for i in range(4):
        eng.buffer("P%d" % (i + 2)).copy_(S["P"][i].permute(0, 2, 3, 1).to(dev))
    eng.buffer("det_boxes")[0].zero_()
    eng.buffer("det_boxes")[0, :D] = torch.from_numpy(S["boxes_final"]).to(dev)
    eng.buffer("det_counts")[0] = D
    eng.buffer("det_classes")[0, :D] = torch.from_numpy(want_cls.astype(np.int32)).to(dev)
    eng.run(None, 1.0, E.ST_MASK_ROIS, E.ST_MASK_OUT)
    torch.cuda.synchronize()
    e = abs_err(eng.buffer("mask_logits")[:D, :, :, :81].permute(0, 3, 1, 2), S["mask_logits"])
    report("R-101-FPN 800x1216 (teacher-forced): mask logits abs err %.3e (|logit| max %.2f)" % (e, S["mask_logits"].abs().max().item()))
    assert e < 1e-4


# ------------------------------------------------------------------------------------------ configs[4]: RoIAlign / NMS microbench sizes
def _synth_rois(n, seed=0, Wf=1088, Hf=800):
    """SURVEY.md 8d distribution: centres U(0,W)xU(0,H), width log-U(16,600) px, aspect log-U(e^-0.7, e^0.7), clipped."""
    rng = np.random.RandomState(seed)
    cx, cy = rng.uniform(0, Wf, n), rng.uniform(0, Hf, n)
    w = np.exp(rng.uniform(np.log(16), np.log(600), n))
    a = np.exp(rng.uniform(-0.7, 0.7, n))
    bw, bh = w * np.sqrt(a), w / np.sqrt(a)
    b = np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1)
    b[:, 0::2] = np.clip(b[:, 0::2], 0, Wf - 1)
    b[:, 1::2] = np.clip(b[:, 1::2], 0, Hf - 1)
    return b.astype(np.float32)


@pytest.mark.parametrize("pooled", [7, 14])
def test_roialign_100k_vs_oracle(built, pooled):
    """100 000 RoIs x 256 channels x 50x68 map: the exact kernel bit-identical to the reference CPU loop, the fast kernel within 1e-5,
    on a random 2048-RoI subsample (the oracle loop is single-threaded); plus a checksum of ALL rows of the fast output against the
    exact output (every RoI of the 100k is covered by the exact-vs-fast comparison on the device)."""
    from detectorch_b200 import ops
    from oracle import ref
    dev = torch.device("cuda:0")
    R, C, Hf, Wf = 100000, 256, 50, 68
    g = torch.Generator().manual_seed(0)
    feat = torch.randn((1, C, Hf, Wf), generator=g)
    rois = np.hstack([np.zeros((R, 1), np.float32), _synth_rois(R)])
    fd, rd = feat.to(dev), torch.from_numpy(rois).to(dev)
    exact = ops.roi_align_forward_nchw(fd, rd, pooled, pooled, 1 / 16., 2)
    fast = ops.roi_align_forward_nchw_fast(fd, rd, pooled, pooled, 1 / 16., 2)
    torch.cuda.synchronize()
    # whole-output comparison on the device, in slabs (the 14x14 output is 20 GB)
    worst = 0.0
    for s in range(0, R, 10000):
        worst = max(worst, float((exact[s:s + 10000] - fast[s:s + 10000]).abs().max()))
    assert worst < 1e-5 * max(1.0, float(feat.abs().max()))
    sub = np.random.RandomState(1).choice(R, 2048, replace=False)
    sub.sort()
    want = ref.roi_align_forward(feat.numpy(), rois[sub], pooled, pooled, 1 / 16., 2)
    idx = torch.from_numpy(sub).to(dev)
    assert np.array_equal(exact[idx].cpu().numpy(), want)                                  # bit-exact
    assert np.abs(fast[idx].cpu().numpy() - want).max() < 1e-5 * max(1.0, float(np.abs(want).max()))


def test_nms_100k_vs_oracle(built):
    from detectorch_b200 import ops
    from oracle import ref
    dev = torch.device("cuda:0")
    n = 100000
    rng = np.random.RandomState(n)
    d = np.hstack([_synth_rois(n, seed=n, Wf=1216), rng.permutation(n).astype(np.float32)[:, None] / n]).astype(np.float32)
    got = ops.nms(torch.from_numpy(d).to(dev), 0.5).cpu().numpy()
    want = ref.nms(d, 0.5)
    assert np.array_equal(got, want)
