"""Drop-in mirror of the reference model API (lib/model/detector.py:130-286): same constructor
kwargs, same forward signature / return tuple, same attribute names (`model`, `conv_body`,
`conv_head`, `rpn`, `bbox_head`, `classif_head`, `mask_head`), same state_dict names and the same
Detectron-pkl loader entry point -- but forward() runs the fused sm_90a engine
(detectorch_b200/csrc/capi_engine.cu) instead of torch.nn ops + host numpy.

The torch modules below are PARAMETER CONTAINERS ONLY (so state_dict()/load_state_dict()/the pkl
loader keep working); none of their forward() methods is ever called.

Supported configurations = the constructor kwargs of the reference's eight eval_*.ipynb notebooks, ResNet-50/101:
  FPN family  eval_fast_FPN (pre-computed per-level proposals), eval_faster_FPN, eval_mask_FPN ('1up4convs')
  C4 family   eval_fast (pre-computed proposals), eval_faster, eval_mask ('upshare')

Aliasing: forward() returns zero-copy VIEWS of engine buffers (cls_score, bbox_pred, rois, the FPN maps); they are overwritten by the
next forward() on an engine of the same input shape.  Clone what must outlive the next image (the notebooks do not).
Weights: engines pack the parameters when they are created; call load_state_dict / load_pretrained_weights (or bump
`model._weights_version`) after editing parameters in place.
"""
import numpy as np
import torch
import torchvision.models as models

import collections
import os

from ..engine import Engine, engine_owning, ST_TRUNK, ST_FPN, ST_ROI_BOX, ST_BOX_HEAD, ST_DETECT, ST_MASK_ROI_FEAT, ST_MASK_OUT


def caffe2_blob_name(key):
    """torchvision ResNet state_dict key -> Detectron (caffe2) blob name, the mapping utils/utils.py:44-71 (parse_th_to_caffe2) implements:
    conv1.weight -> conv1_w; bn1.{weight,bias} -> res_conv1_bn_{s,b}; layerL.B.convK.weight -> res{L+1}_{B}_branch2{a,b,c}_w;
    layerL.B.bnK.{weight,bias} -> res{L+1}_{B}_branch2{a,b,c}_bn_{s,b}; layerL.B.downsample.{0.weight,1.weight,1.bias} -> res{L+1}_{B}_branch1_{w,bn_s,bn_b}."""
    t = key.split('.')
    leaf = {'weight': '_s', 'bias': '_b'}
    if t[0] == 'conv1':
        return 'conv1_w'
    if t[0] == 'bn1':
        return 'res_conv1_bn' + leaf[t[1]]
    stage = 'res%d_%s' % (int(t[0][-1]) + 1, t[1])
    if t[2] == 'downsample':
        return stage + '_branch1' + ('_w' if t[3] == '0' else '_bn' + leaf[t[4]])
    branch = stage + '_branch2' + 'abc'[int(t[2][-1]) - 1]
    return branch + ('_w' if t[2].startswith('conv') else '_bn' + leaf[t[3]])


class _FpnBody(torch.nn.Module):           # parameter container: detector.py:12-33
    def __init__(self, conv_body, in_channels, fpn_layers):
        super().__init__()
        self.conv_body = conv_body
        self.fpn_lateral = torch.nn.ModuleList([torch.nn.Conv2d(c, 256, 1) for c in in_channels])
        self.fpn_output = torch.nn.ModuleList([torch.nn.Conv2d(256, 256, 3, padding=1) for _ in in_channels])
        self.fpn_layers = fpn_layers


class _TwoLayerMlp(torch.nn.Module):       # detector.py:54-59
    def __init__(self):
        super().__init__()
        self.fc6 = torch.nn.Linear(256 * 7 * 7, 1024)
        self.fc7 = torch.nn.Linear(1024, 1024)


class _FourConv(torch.nn.Module):          # detector.py:67-74
    def __init__(self):
        super().__init__()
        for i in range(1, 5):
            setattr(self, "fcn%d" % i, torch.nn.Conv2d(256, 256, 3, padding=1))


class _RpnHead(torch.nn.Module):           # detector.py:114-121
    def __init__(self, in_channels, out_channels, n_anchors):
        super().__init__()
        self.conv_rpn = torch.nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.rpn_cls_prob = torch.nn.Conv2d(out_channels, n_anchors, 1)
        self.rpn_bbox_pred = torch.nn.Conv2d(out_channels, 4 * n_anchors, 1)


class _MaskHead(torch.nn.Module):
    """mask_head of the reference (detector.py:84-112); forward(x, rois, roi_original_idx) keeps its signature."""

    def __init__(self, owner, output_prob, conv_head=None):
        super().__init__()
        # '1up4convs': own 4-conv tower; 'upshare': the res5 block shared with the box head (detector.py:217-221)
        self.conv_head = _FourConv() if conv_head is None else conv_head
        self.transposed_conv = torch.nn.ConvTranspose2d(256 if conv_head is None else 2048, 256, 2, stride=2)
        self.classif_logits = torch.nn.Conv2d(256, 81, 1)
        self.output_prob = output_prob
        self.roi_height = self.roi_width = 14
        object.__setattr__(self, "_owner", owner)

    def forward(self, x, rois, roi_original_idx=None):
        return self._owner._run_mask_head(x, rois, roi_original_idx)


class detector(torch.nn.Module):
    def __init__(self,
                 train=False,
                 arch='resnet50',
                 conv_body_layers=['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3'],
                 conv_head_layers=['layer4', 'avgpool'],
                 fpn_layers=[],
                 fpn_extra_lvl=True,
                 use_rpn_head=False,
                 use_mask_head=False,
                 mask_head_type='upshare',
                 roi_feature_channels=2048,
                 N_classes=81,
                 detector_pkl_file=None,
                 base_cnn_pkl_file=None,
                 output_prob=True,
                 roi_height=14,
                 roi_width=14,
                 roi_spatial_scale=0.0625,
                 roi_sampling_ratio=0):
        super(detector, self).__init__()
        self.roi_height, self.roi_width = int(roi_height), int(roi_width)
        self.roi_spatial_scale = [float(i) for i in roi_spatial_scale] if isinstance(roi_spatial_scale, list) else float(roi_spatial_scale)
        self.roi_sampling_ratio = int(roi_sampling_ratio)
        self.train = train           # shadows nn.Module.train exactly like the reference (detector.py:159)
        self.arch = arch
        self.mask_head_type = mask_head_type
        self.use_fpn_body = len(fpn_layers) > 0
        self.fpn_extra_lvl = fpn_extra_lvl
        self.use_rpn_head = use_rpn_head
        self.use_mask_head = use_mask_head
        self.use_two_layer_mlp_head = conv_head_layers == 'two_layer_mlp'
        self.output_prob = output_prob
        self.N_classes = N_classes
        fpn_ok = (self.use_fpn_body and self.use_two_layer_mlp_head and (fpn_extra_lvl or not use_rpn_head) and
                  list(fpn_layers) == ['layer1', 'layer2', 'layer3', 'layer4'] and self.roi_height == 7 and self.roi_width == 7 and
                  self.roi_sampling_ratio == 2 and self.roi_spatial_scale == [0.25, 0.125, 0.0625, 0.03125] and
                  (not use_mask_head or (mask_head_type == '1up4convs' and use_rpn_head)))
        c4_ok = (not self.use_fpn_body and list(conv_body_layers) == ['conv1', 'bn1', 'relu', 'maxpool', 'layer1', 'layer2', 'layer3'] and
                 list(conv_head_layers) == ['layer4', 'avgpool'] and self.roi_height == 14 and self.roi_width == 14 and
                 self.roi_sampling_ratio == 0 and self.roi_spatial_scale == 0.0625 and (not use_mask_head or mask_head_type == 'upshare'))
        if not ((fpn_ok or c4_ok) and arch in ('resnet50', 'resnet101') and not train):
            raise NotImplementedError("detectorch_b200 implements the reference's inference configurations (eval_*.ipynb kwargs): "
                                      "R-50/101-FPN Fast/Faster/Mask (1up4convs) and R-50/101-C4 Fast/Faster/Mask (upshare); got something else")
        self.family = "fpn" if fpn_ok else "c4"
        if arch.startswith('resnet'):
            self.model = getattr(models, arch)()
        else:
            raise NotImplementedError('Only resnet implemented so far!')
        if self.family == "fpn":
            self.conv_body = _FpnBody(torch.nn.Sequential(*[getattr(self.model, l) for l in conv_body_layers]), (256, 512, 1024, 2048), fpn_layers)
            self.conv_head = _TwoLayerMlp()
            if self.use_rpn_head:
                self.rpn = _RpnHead(256, 256, 3)
            feat = 1024      # two-layer MLP head (detector.py:143,212: the 2048 default only fits the C4 head)
        else:
            self.conv_body = torch.nn.Sequential(*[getattr(self.model, l) for l in conv_body_layers])
            self.conv_head = torch.nn.Sequential(*[getattr(self.model, l) for l in conv_head_layers])
            if self.use_rpn_head:
                self.rpn = _RpnHead(1024, 1024, 15)
            feat = roi_feature_channels
        self.bbox_head = torch.nn.Linear(feat, 4 * N_classes)
        self.classif_head = torch.nn.Linear(feat, N_classes)
        if self.use_mask_head:
            self.mask_head = _MaskHead(self, output_prob, None if self.family == "fpn" else self.conv_head[0])
        # Engine options of the mirror: full [D,81,M,M] masks are what model.mask_head returns (reference layout); a caller that only uses the
        # fused detect() path may switch them off and size the padded detection slots (bench.py does)
        self.engine_defaults = dict(emit_full_masks=True, det_cap=128)
        self.capture_graphs = os.environ.get("DT_DETECT_GRAPH", "1") != "0"      # detect(host batch): replay a captured CUDA graph of the step
        self._engines = collections.OrderedDict()      # LRU: (batch, h, w, overrides) -> (Engine, weights_version)
        self.max_cached_engines = int(os.environ.get("DT_ENGINE_CACHE", "6"))
        self._weights_version = 0
        if detector_pkl_file is not None:
            self.load_pretrained_weights(detector_pkl_file, model='detector')
        elif base_cnn_pkl_file is not None:
            self.load_pretrained_weights(base_cnn_pkl_file, model='base_cnn')
        self.model.eval()

    # ------------------------------------------------------------------ weights
    def load_pretrained_weights(self, caffe_pkl_file, model='detector'):
        """Detectron caffe2-pickle import (detector.py:289-374), 'next' row of SURVEY.md 8f."""
        import pickle
        with open(caffe_pkl_file, 'rb') as f:
            blobs = pickle.load(f, encoding='latin1')
        if model == 'detector':
            blobs = blobs['blobs']
        sd = self.model.state_dict()
        for k in sd.keys():
            if 'running' in k or 'fc' in k or 'num_batches' in k:
                continue
            kc = caffe2_blob_name(k)
            w = torch.FloatTensor(blobs[kc])
            sd[k] = w[:, (2, 1, 0), :, :] if k == 'conv1.weight' else w     # BGR -> RGB
        self.model.load_state_dict(sd)
        if model == 'detector':
            def put(mod, wn, bn):
                mod.weight.data = torch.FloatTensor(blobs[wn]); mod.bias.data = torch.FloatTensor(blobs[bn])
            put(self.bbox_head, 'bbox_pred_w', 'bbox_pred_b'); put(self.classif_head, 'cls_score_w', 'cls_score_b')
            # the blob names depend on the configuration exactly as in detector.py:317-374
            if self.use_rpn_head:
                sfx = '_fpn2' if self.use_fpn_body else ''
                put(self.rpn.conv_rpn, 'conv_rpn%s_w' % sfx, 'conv_rpn%s_b' % sfx)
                put(self.rpn.rpn_cls_prob, 'rpn_cls_logits%s_w' % sfx, 'rpn_cls_logits%s_b' % sfx)
                put(self.rpn.rpn_bbox_pred, 'rpn_bbox_pred%s_w' % sfx, 'rpn_bbox_pred%s_b' % sfx)
            if self.use_mask_head:
                put(self.mask_head.transposed_conv, 'conv5_mask_w', 'conv5_mask_b')
                put(self.mask_head.classif_logits, 'mask_fcn_logits_w', 'mask_fcn_logits_b')
                if self.mask_head_type == '1up4convs':
                    for i in range(1, 5):
                        put(getattr(self.mask_head.conv_head, 'fcn%d' % i), '_[mask]_fcn%d_w' % i, '_[mask]_fcn%d_b' % i)
            if self.use_fpn_body:
                for i, l in enumerate(self.conv_body.fpn_layers):
                    # the FPN blobs are named after the last conv of the stage's last block, e.g. fpn_inner_res5_2_sum (detector.py:357-359)
                    kc = 'res%d_%d' % (int(l[-1]) + 1, len(getattr(self.model, l)) - 1)
                    suffix = '_sum_lateral' if i < len(self.conv_body.fpn_layers) - 1 else '_sum'
                    put(self.conv_body.fpn_lateral[i], 'fpn_inner_' + kc + suffix + '_w', 'fpn_inner_' + kc + suffix + '_b')
                    put(self.conv_body.fpn_output[i], 'fpn_' + kc + '_sum_w', 'fpn_' + kc + '_sum_b')
            if self.use_two_layer_mlp_head:
                put(self.conv_head.fc6, 'fc6_w', 'fc6_b'); put(self.conv_head.fc7, 'fc7_w', 'fc7_b')
        self._weights_version += 1

    def load_state_dict(self, state_dict, strict=True):
        r = super().load_state_dict(state_dict, strict)
        self._weights_version += 1
        return r

    # ------------------------------------------------------------------ engine plumbing
    def engine_for(self, batch, h, w, **overrides):
        """Engine for one input shape.  The cache is a small LRU (`max_cached_engines`, env DT_ENGINE_CACHE): the notebook flow over COCO meets
        dozens of 32-aligned sizes and a workspace is ~1.5 GB at batch 1; the packed weights (0.5 GB) exist ONCE per model and are shared by
        every engine (they do not depend on the shape), so building an engine for a new size costs descriptors + one workspace allocation."""
        key = (batch, h, w, tuple(sorted(overrides.items())), tuple(sorted(self.engine_defaults.items())))
        ent = self._engines.get(key)
        if ent is not None and ent[1] == self._weights_version:
            self._engines.move_to_end(key)
            return ent[0]
        dev = next(self.parameters()).device
        if dev.type != 'cuda':
            raise RuntimeError("detectorch_b200.detector runs on CUDA only: call model.cuda() first (no CPU fallback)")
        kw = dict(arch=self.arch, batch=batch, height=h, width=w, num_classes=self.N_classes, use_mask=self.use_mask_head,
                  output_prob=self.output_prob, use_rpn=self.use_rpn_head, device=dev)
        kw.update(self.engine_defaults)
        if self.family == "c4":
            kw.update(model="c4", pre_nms_top_n=6000, post_nms_top_n=1000, exact_roialign=True)
        kw.update(overrides)
        for k in [k for k, v in self._engines.items() if v[1] != self._weights_version]:
            del self._engines[k]                                    # stale weights
        while len(self._engines) >= max(1, self.max_cached_engines):
            self._engines.popitem(last=False)                       # least recently used
        # what shapes the packed weight buffer (and the per-launch scale vectors in it): the model, not the image size / capacities
        mk = tuple(sorted((k, str(v)) for k, v in kw.items() if k in ("arch", "num_classes", "use_mask", "model", "use_rpn", "conv_kind", "precise_mask", "passes")))
        donor = next((e for e, _ in self._engines.values() if getattr(e, "_mirror_model_key", None) == mk), None)
        if donor is not None:
            eng = Engine(share_weights_with=donor, **kw)
        else:
            eng = Engine(**kw)
            eng.load_state_dict(self.state_dict())
        eng._mirror_model_key = mk
        self._engines[key] = (eng, self._weights_version)
        return eng

    def forward(self, image, rois=None, scaling_factor=None, roi_original_idx=None):
        """-> (cls_score [R,81], bbox_pred [R,324], rois [R,4], img_features [P2..P5])   detector.py:233-286.
        Batch 1 like the reference; `detect()` below is the batched fused path."""
        if image.size(0) != 1:
            raise RuntimeError("detector.forward keeps the reference's batch-1 contract; use detector.detect for batches")
        sf = float(scaling_factor.reshape(-1)[0]) if torch.is_tensor(scaling_factor) else float(1.0 if scaling_factor is None else scaling_factor)
        image = image.contiguous().float()
        if self.family == "fpn":
            if self.use_rpn_head:
                # the reference overwrites any `rois` argument with the RPN's proposals in this configuration (detector.py:241-257)
                eng = self.engine_for(1, image.size(2), image.size(3))
                eng.last_scaling_factor = sf
                eng.run(image, sf, ST_TRUNK, ST_BOX_HEAD)
                n = int(eng.buffer("roi_counts")[0].item())
            else:
                # Fast R-CNN on the FPN body (eval_fast_FPN.ipynb): rois = per-level list [rois_fpn2..5] (+ roi_original_idx), detector.py:263-270
                if rois is None or not isinstance(rois, (list, tuple)):
                    raise RuntimeError("Fast R-CNN with the FPN body needs the per-level proposal list [rois_fpn2, .., rois_fpn5] (eval_fast_FPN.ipynb)")
                dev = image.device
                parts, lv = [], []
                for i, r in enumerate(rois):
                    if r is None or r.numel() == 0:
                        continue
                    r = r.to(dev).float().reshape(-1, r.shape[-1])[:, -4:]          # preprocess_rois: [1,R,4] / [R,4] / [R,5]
                    parts.append(r)
                    lv.append(torch.full((r.size(0),), i, dtype=torch.int32, device=dev))
                cat, lvl = torch.cat(parts, 0), torch.cat(lv, 0)
                if roi_original_idx is not None:
                    idx = roi_original_idx.to(dev).long().reshape(-1)
                    cat, lvl = cat[idx], lvl[idx]
                n = cat.size(0)
                cap = min(1000, max(100, (n + 99) // 100 * 100))
                if n > cap:
                    raise RuntimeError("at most 1000 proposals per image are supported")
                eng = self.engine_for(1, image.size(2), image.size(3), post_nms_top_n=cap)
                eng.last_scaling_factor = sf
                eng.run(image, sf, ST_TRUNK, ST_FPN)
                er, el = eng.buffer("rois"), eng.buffer("roi_levels")
                er.zero_(); el.zero_()
                er[0, :n, 1:5] = cat
                el[0, :n] = lvl
                eng.buffer("roi_counts")[0] = n
                eng.run(None, sf, ST_ROI_BOX, ST_BOX_HEAD)
            eng.check_range()
            feats = [eng.buffer("P%d" % l).permute(0, 3, 1, 2) for l in (2, 3, 4, 5)]     # NCHW-shaped views of the NHWC maps
        else:
            if self.use_rpn_head:
                eng = self.engine_for(1, image.size(2), image.size(3))
                eng.last_scaling_factor = sf
                eng.run(image, sf, ST_TRUNK, ST_BOX_HEAD)
                n = int(eng.buffer("roi_counts")[0].item())
                eng.check_range()
            else:
                if rois is None:
                    raise RuntimeError("Fast R-CNN needs pre-computed proposals (eval_fast.ipynb passes batch['rois'])")
                r = rois.reshape(-1, rois.shape[-1])[:, -4:].float()
                n = r.size(0)
                cap = min(1000, max(100, (n + 99) // 100 * 100))
                if n > cap:
                    raise RuntimeError("at most 1000 proposals per image are supported")
                eng = self.engine_for(1, image.size(2), image.size(3), post_nms_top_n=cap)
                eng.last_scaling_factor = sf
                eng.run(image, sf, ST_TRUNK, ST_TRUNK)
                er = eng.buffer("rois")
                er.zero_()
                er[0, :n, 1:5] = r.to(eng.device)
                eng.buffer("roi_counts")[0] = n
                eng.run(None, sf, ST_ROI_BOX, ST_BOX_HEAD)
                eng.check_range()
            feats = eng.buffer("C4").permute(0, 3, 1, 2)
        cls_score = eng.buffer("cls_prob")[:n]
        bbox_pred = eng.buffer("bbox_pred")[:n]
        out_rois = eng.buffer("rois")[0, :n, 1:5]
        return (cls_score, bbox_pred, out_rois, feats)

    def _run_mask_head(self, img_features, rois, roi_original_idx):
        # the engine is found from the feature maps it produced (no "current engine" state: two models / two image sizes may interleave)
        eng = engine_owning(img_features)
        if eng is None:
            raise RuntimeError("mask_head: `img_features` must be the maps returned by this model's forward() (views of engine buffers)")
        if self.family == "c4":
            r = rois if torch.is_tensor(rois) else torch.cat(tuple(rois), 0)
            r = r.reshape(-1, r.shape[-1])[:, -4:].to(eng.device).float()        # detector.py:100-101 (preprocess_rois)
            n = r.size(0)
            mr = eng.buffer("mask_rois")
            if n > mr.size(0):
                raise RuntimeError("mask_head: %d RoIs exceed the engine capacity %d" % (n, mr.size(0)))
            mr.zero_()
            mr[:n, 1:5] = r
            eng.run(None, 1.0, ST_MASK_ROI_FEAT, ST_MASK_OUT)
            return eng.buffer("masks_full")[:n]
        # per-level lists -> original order (detector.py:103-106)
        lv, parts = [], []
        for i, r in enumerate(rois):
            if r is None or len(r) == 0:
                continue
            r = r.to(eng.device).float()
            if r.size(1) == 5:
                r = r[:, 1:5]
            parts.append(r)
            lv.append(torch.full((r.size(0),), i, dtype=torch.int32, device=eng.device))
        cat, lvl = torch.cat(parts, 0), torch.cat(lv, 0)
        if roi_original_idx is not None:
            idx = roi_original_idx.to(eng.device).long()
            cat, lvl = cat[idx], lvl[idx]
        n = cat.size(0)
        mr, ml = eng.buffer("mask_rois"), eng.buffer("mask_levels")
        if n > mr.size(0):
            raise RuntimeError("mask_head: %d RoIs exceed the engine capacity %d" % (n, mr.size(0)))
        mr.zero_(); ml.zero_()
        mr[:n, 1:5] = cat
        ml[:n] = lvl
        eng.run(None, 1.0, ST_MASK_ROI_FEAT, ST_MASK_OUT)
        return eng.buffer("masks_full")[:n]

    # ------------------------------------------------------------------ fused batched path
    def detect(self, images, scaling_factor=1.0, with_masks=None):
        """Fused path: images [B,3,H,W] -> dict of padded per-image detections (boxes [B,cap,4], scores, classes, counts,
        masks [B,cap,28,28] of the detected class).  No host synchronisation inside.
        `images` may live in (pinned) HOST memory: the upload then goes through two device staging buffers on a copy stream, so the
        H2D copy of call i+1 overlaps the compute of call i.  The returned tensors are views of engine buffers: read them (e.g. an
        asynchronous copy to pinned memory on the current stream) before the next detect() on the same input shape."""
        if not self.use_rpn_head:
            raise RuntimeError("detect() is the fused RPN path; Fast R-CNN configurations go through forward(image, rois)")
        eng = self.engine_for(images.size(0), images.size(2), images.size(3))
        eng.last_scaling_factor = float(scaling_factor)
        eng.set_original_size(0, 0)          # clip to the network input / scaling_factor (a previous postprocess_output may have set an image size)
        with_masks = self.use_mask_head if with_masks is None else with_masks
        last = ST_MASK_OUT if with_masks else ST_DETECT
        if not images.is_cuda:
            images = self._upload(eng, images)
            st = eng._stage_state
            # host input = fixed device staging buffers: the ~110 launches of the step are captured once per (buffer, scaling factor, stage
            # range) in a CUDA graph (second call on; the first one runs eagerly and warms every kernel up) and replayed afterwards
            key = (st["pending"], float(scaling_factor), last)
            g = st["graphs"].get(key)
            if g is None and st["seen"].get(key, 0) >= 1 and self.capture_graphs:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    eng.run(images, float(scaling_factor), ST_TRUNK, last)
                st["graphs"][key] = g
            st["seen"][key] = st["seen"].get(key, 0) + 1
            if g is not None:
                g.replay()
            else:
                eng.run(images, float(scaling_factor), ST_TRUNK, last)
            st["free"][st["pending"]].record(torch.cuda.current_stream(eng.device))     # the staging buffer may be overwritten after this run
            st["pending"] = None
        else:
            eng.run(images.contiguous().float(), float(scaling_factor), ST_TRUNK, last)
        B, cap = images.size(0), eng.cfg.det_cap
        # "range_flag" (int32 [1]) is non-zero if an activation left the fp16 range of the default kind::f16 convolutions: read it together
        # with the results (no extra synchronisation here), or call engine_owning(out['boxes']).check_range()
        out = {"boxes": eng.buffer("det_boxes"), "scores": eng.buffer("det_scores"), "classes": eng.buffer("det_classes"),
               "counts": eng.buffer("det_counts"), "roi_idx": eng.buffer("det_roi_idx"), "range_flag": eng.buffer("range_flag")}
        if with_masks:
            m = eng.buffer("masks")
            out["masks"] = m.view(B, cap, m.shape[-2], m.shape[-1])
        return out

    def _upload(self, eng, host_images):
        """Host -> device through two staging buffers and a dedicated copy stream (2-deep pipeline across successive detect() calls)."""
        st = getattr(eng, "_stage_state", None)
        if st is None:
            with torch.cuda.device(eng.device):
                st = {"buf": [torch.empty((eng.cfg.batch, 3, eng.cfg.height, eng.cfg.width), dtype=torch.float32, device=eng.device) for _ in range(2)],
                      "up": [torch.cuda.Event() for _ in range(2)], "free": [torch.cuda.Event() for _ in range(2)],
                      "stream": torch.cuda.Stream(device=eng.device), "i": 0, "pending": None, "graphs": {}, "seen": {}}
            eng._stage_state = st
        b = st["i"] % 2
        st["i"] += 1
        cur = torch.cuda.current_stream(eng.device)
        with torch.cuda.stream(st["stream"]):
            st["stream"].wait_event(st["free"][b])              # no-op until the event has been recorded once
            st["buf"][b].copy_(host_images, non_blocking=True)
            st["up"][b].record(st["stream"])
        cur.wait_event(st["up"][b])
        st["pending"] = b
        return st["buf"][b]
