"""
ORACLE -- test infrastructure only (never imported by detectorch_b200/).

Torch-CPU fp32 restatement of the reference detector graph, written functionally
over a flat {reference-parameter-name: tensor} dict so that the same weights load
into the reference `detector` (state_dict names), into this oracle, and into the
H100 engine.

  trunk (torchvision Bottleneck, stride on conv1 of layer{2,3,4}[0])   detector.py:170-183
  BN in eval mode with running stats (0,1): y = x*g/sqrt(1+1e-5) + b     detector.py:231,301
  fpn_body                                                              detector.py:12-52
  rpn_head (shared over levels), P6 = stride-2 subsample of P5          detector.py:114-127,250-251
  two_layer_mlp_head + classif/bbox heads (+softmax)                    detector.py:54-65,273-284
  mask_head '1up4convs'                                                 detector.py:67-112
  res5 head / 'upshare' mask head for the C4 models                     detector.py:136,191,217-218

"parity unpinned" caveat (SURVEY.md 8c): the conv/GEMM arithmetic itself lives in
torch / torchvision, which the reference does not vendor or pin; this file is pinned
against the reference's own modules executed by the torch in this image
(tests/test_oracle.py::test_network_matches_reference, tests/golden/).
"""
import time
import zlib

import numpy as np
import torch
import torch.nn.functional as F

from . import ref

BN_EPS = 1e-5
BLOCKS = {"resnet50": (3, 4, 6, 3), "resnet101": (3, 4, 23, 3)}


# ----------------------------------------------------------------------------- synthetic weights
def param_shapes(arch="resnet50", fpn=True, rpn=True, mask=True, n_classes=81):
    """Flat {name: shape} of every parameter on the hot path, using the reference's
    state_dict names (detector.py module attribute names + torchvision resnet names)."""
    s = {}
    s["model.conv1.weight"] = (64, 3, 7, 7)
    s["model.bn1.weight"] = (64,)
    s["model.bn1.bias"] = (64,)
    inpl = 64
    last = 4 if (fpn or True) else 3
    for li, nb in enumerate(BLOCKS[arch], start=1):
        planes = 64 * 2 ** (li - 1)
        for b in range(nb):
            p = "model.layer%d.%d." % (li, b)
            s[p + "conv1.weight"] = (planes, inpl, 1, 1)
            s[p + "conv2.weight"] = (planes, planes, 3, 3)
            s[p + "conv3.weight"] = (planes * 4, planes, 1, 1)
            for k, c in (("bn1", planes), ("bn2", planes), ("bn3", planes * 4)):
                s[p + k + ".weight"] = (c,)
                s[p + k + ".bias"] = (c,)
            if b == 0:
                s[p + "downsample.0.weight"] = (planes * 4, inpl, 1, 1)
                s[p + "downsample.1.weight"] = (planes * 4,)
                s[p + "downsample.1.bias"] = (planes * 4,)
            inpl = planes * 4
    if fpn:
        for i, c in enumerate((256, 512, 1024, 2048)):
            s["conv_body.fpn_lateral.%d.weight" % i] = (256, c, 1, 1)
            s["conv_body.fpn_lateral.%d.bias" % i] = (256,)
            s["conv_body.fpn_output.%d.weight" % i] = (256, 256, 3, 3)
            s["conv_body.fpn_output.%d.bias" % i] = (256,)
        s["conv_head.fc6.weight"] = (1024, 256 * 7 * 7)
        s["conv_head.fc6.bias"] = (1024,)
        s["conv_head.fc7.weight"] = (1024, 1024)
        s["conv_head.fc7.bias"] = (1024,)
        feat = 1024
        rc, ra = 256, 3
    else:
        feat = 2048
        rc, ra = 1024, 15
    if rpn:
        s["rpn.conv_rpn.weight"] = (rc, rc, 3, 3)
        s["rpn.conv_rpn.bias"] = (rc,)
        s["rpn.rpn_cls_prob.weight"] = (ra, rc, 1, 1)
        s["rpn.rpn_cls_prob.bias"] = (ra,)
        s["rpn.rpn_bbox_pred.weight"] = (4 * ra, rc, 1, 1)
        s["rpn.rpn_bbox_pred.bias"] = (4 * ra,)
    s["bbox_head.weight"] = (4 * n_classes, feat)
    s["bbox_head.bias"] = (4 * n_classes,)
    s["classif_head.weight"] = (n_classes, feat)
    s["classif_head.bias"] = (n_classes,)
    if mask:
        if fpn:
            for i in range(1, 5):
                s["mask_head.conv_head.fcn%d.weight" % i] = (256, 256, 3, 3)
                s["mask_head.conv_head.fcn%d.bias" % i] = (256,)
            s["mask_head.transposed_conv.weight"] = (256, 256, 2, 2)
        else:
            s["mask_head.transposed_conv.weight"] = (2048, 256, 2, 2)
        s["mask_head.transposed_conv.bias"] = (256,)
        s["mask_head.classif_logits.weight"] = (n_classes, 256, 1, 1)
        s["mask_head.classif_logits.bias"] = (n_classes,)
    return s


# substring -> multiplier on the He std; tuned (oracle stats) so FPN maps are O(1), RPN logits
# have std ~2 (no sigmoid saturation), box deltas are small, class logits std ~2.5, mask logits ~3
_STD_MULT = [
    ("model.conv1.weight", 1.0 / 50.0),      # pixels are N(0, 50^2)
    ("downsample.0", 0.7),
    ("fpn_lateral", 0.27),
    ("fpn_output", 0.35),
    ("rpn.conv_rpn", 0.7),
    ("rpn.rpn_cls_prob", 2.2),
    ("rpn.rpn_bbox_pred", 0.12),
    ("conv_head.fc6", 0.75),
    ("bbox_head", 0.3),
    ("classif_head", 1.8),
    ("mask_head.classif_logits", 2.0),
]


# the C4 heads see different feature statistics (1024-ch C4 map, 2048-d pooled res5 features): own multipliers
_STD_MULT_C4 = [
    ("model.conv1.weight", 1.0 / 50.0),
    ("downsample.0", 0.7),
    ("rpn.conv_rpn", 0.35),
    ("rpn.rpn_cls_prob", 1.0),
    ("rpn.rpn_bbox_pred", 0.06),
    ("bbox_head", 0.12),
    ("classif_head", 0.6),
    ("mask_head.transposed_conv", 0.5),
    ("mask_head.classif_logits", 1.0),
]


def synthetic_params(arch="resnet50", fpn=True, rpn=True, mask=True, seed=0, n_classes=81):
    """Deterministic synthetic weights (SURVEY.md 8d): per-parameter generator seeded by
    crc32(name)^seed, He-style conv scale, BN gains chosen so activations stay O(1-10),
    head scales chosen so sigmoid/softmax do not saturate and scores are tie-free."""
    out = {}
    for name, shape in param_shapes(arch, fpn, rpn, mask, n_classes).items():
        g = torch.Generator().manual_seed((zlib.crc32(name.encode()) ^ seed) & 0x7FFFFFFF)
        leaf = name.split(".")[-1]
        is_bn = (".bn" in name or "downsample.1" in name or name.startswith("model.bn1"))
        if is_bn and leaf == "weight":
            base = 0.35 if (name.endswith("bn3.weight")) else 1.0
            if arch == "resnet101" and name.endswith("bn3.weight") and ".layer3." in name:
                base = 0.18      # 23 residual additions instead of 6: keeps the R-101 maps at the R-50 scale (activations O(1-10), mask logits |x| < ~15)
            t = base * (0.8 + 0.4 * torch.rand(shape, generator=g))
        elif leaf == "bias":
            t = 0.1 * torch.randn(shape, generator=g)
            if name == "classif_head.bias":
                t[0] += 1.0          # background prior: most RoIs are background
        else:
            fan_in = int(np.prod(shape[1:]))
            if name == "mask_head.transposed_conv.weight":
                fan_in = shape[0]      # ConvTranspose2d weight is [Cin, Cout, kh, kw], stride==kernel
            std = (2.0 / fan_in) ** 0.5
            for pat, mult in (_STD_MULT if fpn else _STD_MULT_C4):
                if pat in name:
                    std *= mult
                    break
            t = std * torch.randn(shape, generator=g)
        out[name] = t.float().contiguous()
    return out


def synthetic_image(batch, h, w, seed=0):
    g = torch.Generator().manual_seed(1000 + seed)
    return (50.0 * torch.randn((batch, 3, h, w), generator=g)).float()


# ----------------------------------------------------------------------------- graph
def _bn(x, P, name):
    scale = P[name + ".weight"] / torch.sqrt(torch.ones(1) + BN_EPS)
    return x * scale.view(1, -1, 1, 1) + P[name + ".bias"].view(1, -1, 1, 1)


def _bn_ref(x, P, name):
    """Exactly what torch's eval BatchNorm2d computes with running stats (0,1)."""
    c = P[name + ".weight"].numel()
    return F.batch_norm(x, torch.zeros(c), torch.ones(c), P[name + ".weight"], P[name + ".bias"], False, 0.0, BN_EPS)


def _bottleneck(x, P, p, stride, has_ds):
    idt = x
    y = F.relu(_bn_ref(F.conv2d(x, P[p + "conv1.weight"], stride=stride), P, p + "bn1"))
    y = F.relu(_bn_ref(F.conv2d(y, P[p + "conv2.weight"], padding=1), P, p + "bn2"))
    y = _bn_ref(F.conv2d(y, P[p + "conv3.weight"]), P, p + "bn3")
    if has_ds:
        idt = _bn_ref(F.conv2d(x, P[p + "downsample.0.weight"], stride=stride), P, p + "downsample.1")
    return F.relu(y + idt)


def layer(x, P, arch, li):
    nb = BLOCKS[arch][li - 1]
    for b in range(nb):
        stride = 2 if (b == 0 and li > 1) else 1
        x = _bottleneck(x, P, "model.layer%d.%d." % (li, b), stride, b == 0)
    return x


def trunk(image, P, arch="resnet50", upto=4):
    """Returns [C2, C3, C4, C5][:upto].  detector.py:170-183."""
    x = F.relu(_bn_ref(F.conv2d(image, P["model.conv1.weight"], stride=2, padding=3), P, "model.bn1"))
    x = F.max_pool2d(x, 3, 2, 1)
    feats = []
    for li in range(1, upto + 1):
        x = layer(x, P, arch, li)
        feats.append(x)
    return feats


def fpn(feats, P):
    """detector.py:35-52: lateral 1x1, top-down nearest x2 + add, output 3x3."""
    lat = [F.conv2d(f, P["conv_body.fpn_lateral.%d.weight" % i], P["conv_body.fpn_lateral.%d.bias" % i])
           for i, f in enumerate(feats)]
    for i in range(len(lat) - 2, -1, -1):
        lat[i] = F.interpolate(lat[i + 1], scale_factor=2, mode="nearest") + lat[i]
    return [F.conv2d(l, P["conv_body.fpn_output.%d.weight" % i], P["conv_body.fpn_output.%d.bias" % i], padding=1)
            for i, l in enumerate(lat)]


def rpn_head(x, P):
    """detector.py:123-127."""
    t = F.relu(F.conv2d(x, P["rpn.conv_rpn.weight"], P["rpn.conv_rpn.bias"], padding=1))
    cls = torch.sigmoid(F.conv2d(t, P["rpn.rpn_cls_prob.weight"], P["rpn.rpn_cls_prob.bias"]))
    box = F.conv2d(t, P["rpn.rpn_bbox_pred.weight"], P["rpn.rpn_bbox_pred.bias"])
    return cls, box


FPN_SCALES = [0.25, 0.125, 0.0625, 0.03125]


def box_head_fpn(roi_feats, P, output_prob=True):
    """detector.py:61-64,273-284."""
    x = roi_feats.reshape(roi_feats.size(0), -1)
    x = F.relu(F.linear(x, P["conv_head.fc6.weight"], P["conv_head.fc6.bias"]))
    x = F.relu(F.linear(x, P["conv_head.fc7.weight"], P["conv_head.fc7.bias"]))
    cls = F.linear(x, P["classif_head.weight"], P["classif_head.bias"])
    logits = cls
    if output_prob:
        cls = F.softmax(cls, dim=1)
    box = F.linear(x, P["bbox_head.weight"], P["bbox_head.bias"])
    return cls, box, logits


def mask_head_fpn(feats, rois_per_level, idx_restore, P, output_prob=True, return_logits=False):
    """detector.py:99-112 ('1up4convs'): RoIAlign 14x14 sr=2 per level, cat, reorder, 4x conv3x3+ReLU,
    deconv 2x2 s2 + ReLU, 1x1 -> 81, sigmoid."""
    xs = []
    for i, r in enumerate(rois_per_level):
        if r is None or len(r) == 0:
            continue
        r = torch.as_tensor(r, dtype=torch.float32)
        xs.append(torch.from_numpy(ref.roi_align_forward(feats[i].numpy(), r.numpy(), 14, 14, FPN_SCALES[i], 2)))
    x = torch.cat(xs, 0)[torch.as_tensor(np.asarray(idx_restore), dtype=torch.long)]
    roi_feat = x
    for i in range(1, 5):
        x = F.relu(F.conv2d(x, P["mask_head.conv_head.fcn%d.weight" % i], P["mask_head.conv_head.fcn%d.bias" % i], padding=1))
    x = F.relu(F.conv_transpose2d(x, P["mask_head.transposed_conv.weight"], P["mask_head.transposed_conv.bias"], stride=2))
    logits = F.conv2d(x, P["mask_head.classif_logits.weight"], P["mask_head.classif_logits.bias"])
    out = torch.sigmoid(logits) if output_prob else logits
    if return_logits:
        return out, logits, roi_feat
    return out


class StageTimer:
    """Wall-clock per stage of the CPU path (bench.py's per-stage break-out of the reference arm); a no-op when `timers` is None."""

    def __init__(self, timers):
        self.timers, self.t = timers, time.perf_counter()

    def lap(self, name):
        if self.timers is not None:
            now = time.perf_counter()
            self.timers[name] = self.timers.get(name, 0.0) + (now - self.t)
            self.t = now


def forward_fpn(image, P, arch="resnet50", scaling_factor=1.0, pre_nms=1000, post_nms=1000, output_prob=True, timers=None):
    """detector.forward for the FPN + RPN configuration, batch 1 (detector.py:233-286).
    Returns a dict of every teacher-forcing stage (SURVEY.md 7.1 G1..G7)."""
    assert image.size(0) == 1
    h, w = image.size(2), image.size(3)
    S = {}
    tm = StageTimer(timers)
    with torch.no_grad():
        S["C"] = trunk(image, P, arch, 4)
        tm.lap("trunk")
        S["P"] = fpn(S["C"], P)
        tm.lap("fpn")
        lv = S["P"] + [F.max_pool2d(S["P"][-1], 1, stride=2)]
        S["P6"] = lv[-1]
        S["rpn"] = [rpn_head(f, P) for f in lv]
        tm.lap("rpn_head")
        scales = FPN_SCALES + [FPN_SCALES[-1] / 2.]
        S["props"] = []
        for i, (cls, box) in enumerate(S["rpn"]):
            pr, sc, st = ref.generate_proposals_level(cls, box, h, w, scaling_factor, scales[i], (32 * 2 ** i,),
                                                      pre_nms_top_n=pre_nms, post_nms_top_n=post_nms, return_stages=True)
            S["props"].append((pr, sc, st))
        per_level, idx_restore, rois, lvls = ref.collect_and_distribute([p[0] for p in S["props"]],
                                                                        [p[1] for p in S["props"]], 2, 5, post_nms)
        S["rois_per_level"], S["idx_restore"], S["lvls"] = per_level, idx_restore, lvls
        tm.lap("proposals_nms_collect")
        feats = []
        for i, r in enumerate(per_level):
            feats.append(torch.from_numpy(ref.roi_align_forward(S["P"][i].numpy(), r.numpy(), 7, 7, FPN_SCALES[i], 2))
                         if len(r) else torch.zeros((0, 256, 7, 7)))
        roi_feats = torch.cat(feats, 0)[torch.as_tensor(idx_restore, dtype=torch.long)]
        S["rois"] = torch.cat(tuple(per_level), 0)[torch.as_tensor(idx_restore, dtype=torch.long)]
        assert torch.equal(S["rois"], rois)
        S["roi_feats"] = roi_feats
        tm.lap("roialign_box")
        S["cls_score"], S["bbox_pred"], S["cls_logits"] = box_head_fpn(roi_feats, P, output_prob)
        tm.lap("box_head")
    return S


def forward_fpn_precomputed(image, P, proposals, arch="resnet50", output_prob=True):
    """detector.forward for Fast R-CNN on the FPN body (eval_fast_FPN.ipynb; detector.py:259-270 with `rois` a per-level list and
    `roi_original_idx`): proposals [R,4] (network-input pixels) are distributed over P2..P5 by add_multilevel_rois_for_test
    (preprocess_sample.py:43-46), pooled per level, concatenated and restored to the original order."""
    assert image.size(0) == 1
    S = {}
    with torch.no_grad():
        S["C"] = trunk(image, P, arch, 4)
        S["P"] = fpn(S["C"], P)
        pr = np.asarray(proposals, dtype=np.float32)
        per_level, idx_restore = ref.multilevel_rois_for_test(pr)
        feats = []
        for i, r in enumerate(per_level):
            feats.append(torch.from_numpy(ref.roi_align_forward(S["P"][i].numpy(), r, 7, 7, FPN_SCALES[i], 2)) if len(r) else torch.zeros((0, 256, 7, 7)))
        idx = torch.as_tensor(idx_restore.astype(np.int64))
        S["roi_feats"] = torch.cat(feats, 0)[idx]
        S["rois"] = torch.from_numpy(np.concatenate(per_level, 0))[idx]
        assert np.array_equal(S["rois"].numpy(), pr)
        S["cls_score"], S["bbox_pred"], S["cls_logits"] = box_head_fpn(S["roi_feats"], P, output_prob)
    return S


def detect_and_mask_fpn(image, P, arch="resnet50", scaling_factor=1.0, im_size=None, **kw):
    """The full notebook step (eval_mask_FPN.ipynb cell 10): forward, postprocess_output,
    re-split detections by level, mask head.  Returns the stage dict + detections + masks.
    im_size: the ORIGINAL image (h, w) the boxes are clipped to (batch['original_im_size']); default: the blob size / scaling_factor."""
    S = forward_fpn(image, P, arch, scaling_factor, **kw)
    tm = StageTimer(kw.get("timers"))
    h, w = image.size(2), image.size(3)
    im_size = np.array([h / scaling_factor, w / scaling_factor] if im_size is None else im_size[:2], dtype=np.float32)
    sf, bf, cb = ref.postprocess_output(S["rois"], scaling_factor, im_size, S["cls_score"], S["bbox_pred"])
    S["scores_final"], S["boxes_final"], S["cls_boxes"] = sf, bf, cb
    tm.lap("postprocess_nms")
    if len(bf):
        per_level, idx = ref.multilevel_rois_for_test((bf * scaling_factor).astype(np.float32))
        S["mask_rois_per_level"], S["mask_idx_restore"] = per_level, idx
        with torch.no_grad():
            S["masks"], S["mask_logits"], S["mask_roi_feats"] = mask_head_fpn(S["P"], per_level, idx.astype(np.int64), P,
                                                                              True, return_logits=True)
        tm.lap("mask_head")
    return S


# ----------------------------------------------------------------------------- C4 model family
C4_ANCHOR_SIZES = (32, 64, 128, 256, 512)


def res5_head(x, P, arch="resnet50"):
    """conv_head = [layer4, avgpool] run per RoI (detector.py:136,191,273): [R,1024,14,14] -> ([R,2048], [R,2048,7,7])."""
    y = layer(x, P, arch, 4)
    return F.adaptive_avg_pool2d(y, (1, 1)).view(y.size(0), -1), y


def forward_c4(image, P, arch="resnet50", proposals=None, scaling_factor=1.0, pre_nms=6000, post_nms=1000, output_prob=True, timers=None):
    """detector.forward for the C4 configurations, batch 1 (detector.py:233-286): Fast R-CNN when `proposals` [R,4] is given
    (eval_fast.ipynb), Faster R-CNN otherwise (single-level RPN, eval_faster.ipynb)."""
    assert image.size(0) == 1
    h, w = image.size(2), image.size(3)
    S = {}
    tm = StageTimer(timers)
    with torch.no_grad():
        S["C4"] = trunk(image, P, arch, 3)[-1]
        tm.lap("trunk")
        if proposals is None:
            S["rpn"] = rpn_head(S["C4"], P)
            pr, sc, st = ref.generate_proposals_level(S["rpn"][0], S["rpn"][1], h, w, scaling_factor, 0.0625, C4_ANCHOR_SIZES,
                                                      pre_nms_top_n=pre_nms, post_nms_top_n=post_nms, return_stages=True)
            S["props"] = (pr, sc, st)
            rois = pr
        else:
            rois = torch.as_tensor(proposals, dtype=torch.float32)
        S["rois"] = rois
        tm.lap("rpn_proposals_nms")
        feats = torch.from_numpy(ref.roi_align_forward(S["C4"].numpy(), rois.numpy(), 14, 14, 0.0625, 0))
        S["roi_feats"] = feats
        tm.lap("roialign_box")
        pooled, S["res5"] = res5_head(feats, P, arch)
        S["pooled"] = pooled
        cls = F.linear(pooled, P["classif_head.weight"], P["classif_head.bias"])
        S["cls_logits"] = cls
        S["cls_score"] = F.softmax(cls, dim=1) if output_prob else cls
        S["bbox_pred"] = F.linear(pooled, P["bbox_head.weight"], P["bbox_head.bias"])
        tm.lap("res5_head")
    return S


def mask_head_c4(c4_feat, rois, P, arch="resnet50", output_prob=True):
    """mask_head 'upshare' (detector.py:84-112, 217-218): RoIAlign 14x14 sr=0 -> layer4 -> deconv 2x2 s2 + ReLU -> 1x1 -> 81."""
    with torch.no_grad():
        x = torch.from_numpy(ref.roi_align_forward(c4_feat.numpy(), np.asarray(rois, dtype=np.float32), 14, 14, 0.0625, 0))
        roi_feat = x
        x = layer(x, P, arch, 4)
        x = F.relu(F.conv_transpose2d(x, P["mask_head.transposed_conv.weight"], P["mask_head.transposed_conv.bias"], stride=2))
        logits = F.conv2d(x, P["mask_head.classif_logits.weight"], P["mask_head.classif_logits.bias"])
    return (torch.sigmoid(logits) if output_prob else logits), logits, roi_feat


def detect_and_mask_c4(image, P, arch="resnet50", proposals=None, scaling_factor=1.0, use_mask=True, im_size=None, **kw):
    S = forward_c4(image, P, arch, proposals, scaling_factor, **kw)
    tm = StageTimer(kw.get("timers"))
    h, w = image.size(2), image.size(3)
    im_size = np.array([h / scaling_factor, w / scaling_factor] if im_size is None else im_size[:2], dtype=np.float32)
    sf, bf, cb = ref.postprocess_output(S["rois"], scaling_factor, im_size, S["cls_score"], S["bbox_pred"])
    S["scores_final"], S["boxes_final"], S["cls_boxes"] = sf, bf, cb
    tm.lap("postprocess_nms")
    if use_mask and len(bf):
        S["masks"], S["mask_logits"], S["mask_roi_feats"] = mask_head_c4(S["C4"], (bf * scaling_factor).astype(np.float32), P, arch)
    return S
