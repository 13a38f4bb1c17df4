"""Seeded inputs shared by the tests that compare with the reference's own code and by tests/golden/make_ref_golden.py, which runs the
reference on them and stores what it computed in tests/golden/ref_golden.npz."""
import pickle

import numpy as np
import torch

FPN = dict(arch='resnet50', conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3', 'layer4'],
           conv_head_layers='two_layer_mlp', fpn_layers=['layer1', 'layer2', 'layer3', 'layer4'],
           roi_height=7, roi_width=7, roi_spatial_scale=[0.25, 0.125, 0.0625, 0.03125], roi_sampling_ratio=2)
# name -> (constructor kwargs as the notebook passes them, oracle parameter-set flags)
CONFIGS = {
    "eval_fast": (dict(arch='resnet50'), dict(fpn=False, rpn=False, mask=False)),
    "eval_faster": (dict(arch='resnet50', use_rpn_head=True), dict(fpn=False, rpn=True, mask=False)),
    "eval_mask": (dict(arch='resnet50', use_rpn_head=True, use_mask_head=True), dict(fpn=False, rpn=True, mask=True)),
    "eval_fast_FPN": (dict(FPN), dict(fpn=True, rpn=False, mask=False)),
    "eval_faster_FPN": (dict(FPN, fpn_extra_lvl=True, use_rpn_head=True), dict(fpn=True, rpn=True, mask=False)),
    "eval_mask_FPN": (dict(FPN, fpn_extra_lvl=True, use_rpn_head=True, use_mask_head=True, mask_head_type='1up4convs'), dict(fpn=True, rpn=True, mask=True)),
}
ROI_CFGS = ((7, 2), (14, 0))
ROI_KEEP = {7: 80, 14: 16}           # RoIs of the stored RoIAlign outputs (the 14x14 case is sampled to keep the fixture small)


def bitsum(t):
    """Sum of the float32 bit patterns of a tensor as integers: exact and independent of summation order (unlike a float sum)."""
    return int(t.detach().float().contiguous().view(torch.int32).to(torch.int64).sum().item())


def head8(t):
    """First 8 values of a tensor (flattened), NaN-padded: with bitsum, the fingerprint of a loaded parameter."""
    v = t.detach().reshape(-1)[:8].float().numpy()
    return np.concatenate([v, np.full(8 - len(v), np.nan, np.float32)])


def write_detectron_pickle(path, layout, P, flags):
    """A pickle in the published checkpoints' format ({'blobs': {caffe2 name: ndarray}}), filled from the flat parameter dict P.
    layout: the reference detector's trunk keys ("trunk"), their caffe2 blob names ("c2") and the caffe2 stems of the FPN layers ("fpn")."""
    blobs = {}
    for k in layout["trunk"]:                                                # trunk: torchvision name -> caffe2 blob name
        if 'running' in k or 'fc' in k:
            continue
        if 'num_batches' in k:
            # torch >= 0.4.1 adds this buffer; the reference's loader (detector.py:300-304) does not skip it, so a blob must exist
            blobs[layout["c2"][k]] = np.zeros((), np.float32)
            continue
        w = P["model." + k].numpy()
        blobs[layout["c2"][k]] = w[:, (2, 1, 0), :, :].copy() if k == 'conv1.weight' else w     # pickles hold BGR

    def put(wn, bn, name):
        blobs[wn], blobs[bn] = P[name + ".weight"].numpy(), P[name + ".bias"].numpy()
    put('bbox_pred_w', 'bbox_pred_b', 'bbox_head'); put('cls_score_w', 'cls_score_b', 'classif_head')
    if flags["rpn"]:
        sfx = '_fpn2' if flags["fpn"] else ''
        put('conv_rpn%s_w' % sfx, 'conv_rpn%s_b' % sfx, 'rpn.conv_rpn')
        put('rpn_cls_logits%s_w' % sfx, 'rpn_cls_logits%s_b' % sfx, 'rpn.rpn_cls_prob')
        put('rpn_bbox_pred%s_w' % sfx, 'rpn_bbox_pred%s_b' % sfx, 'rpn.rpn_bbox_pred')
    if flags["mask"]:
        put('conv5_mask_w', 'conv5_mask_b', 'mask_head.transposed_conv'); put('mask_fcn_logits_w', 'mask_fcn_logits_b', 'mask_head.classif_logits')
        if flags["fpn"]:
            for i in range(1, 5):
                put('_[mask]_fcn%d_w' % i, '_[mask]_fcn%d_b' % i, 'mask_head.conv_head.fcn%d' % i)
    if flags["fpn"]:
        for i, kc in enumerate(layout["fpn"]):
            kc = kc[:kc.rfind("_")]
            suffix = '_sum_lateral' if i < 3 else '_sum'
            put('fpn_inner_' + kc + suffix + '_w', 'fpn_inner_' + kc + suffix + '_b', 'conv_body.fpn_lateral.%d' % i)
            put('fpn_' + kc + '_sum_w', 'fpn_' + kc + '_sum_b', 'conv_body.fpn_output.%d' % i)
        put('fc6_w', 'fc6_b', 'conv_head.fc6'); put('fc7_w', 'fc7_b', 'conv_head.fc7')
    with open(path, "wb") as f:
        pickle.dump({'blobs': blobs}, f, protocol=2)


def nms_cases():
    rng = np.random.RandomState(7)
    cases = []
    for n in (5, 333, 1500):
        x1 = rng.uniform(0, 900, n); y1 = rng.uniform(0, 600, n)
        d = np.stack([x1, y1, x1 + rng.uniform(2, 300, n), y1 + rng.uniform(2, 300, n), rng.uniform(0, 1, n)], 1).astype(np.float32)
        for t in (0.3, 0.7):
            cases.append((d, t))
    return cases


def roi_case():
    rng = np.random.RandomState(8)
    f = rng.randn(1, 4, 13, 19).astype(np.float32)
    x1 = rng.uniform(-40, 500, 80); y1 = rng.uniform(-40, 300, 80)
    r = np.stack([np.zeros(80), x1, y1, x1 + rng.uniform(1, 400, 80), y1 + rng.uniform(1, 300, 80)], 1).astype(np.float32)
    return f, r


def prep_cases():
    rng = np.random.RandomState(123)
    return [(rng.randint(0, 256, (h, w, 3)).astype(np.uint8), ts, ms)
            for (h, w, ts, ms) in ((37, 52, 60, 100), (80, 41, 40, 1333), (64, 96, 32, 1333))]       # up, portrait cap, exact 1/2


def segm_case():
    rng = np.random.RandomState(124)
    M, K, im_h, im_w = 28, 3, 120, 150
    boxes = np.array([[3.2, 4.1, 60.7, 80.3], [100, 20, 149, 119], [0, 0, 149, 119], [70, 70, 83, 83], [10, 90, 40, 119]], np.float32)
    cls = np.array([1, 1, 2, 2, 2])
    masks = rng.rand(5, K, M, M).astype(np.float32)
    cls_boxes = [[], np.hstack([boxes[cls == 1], np.ones((2, 1), np.float32)]), np.hstack([boxes[cls == 2], np.ones((3, 1), np.float32)])]
    return M, K, im_h, im_w, boxes, cls, masks, cls_boxes
