"""Writes tests/golden/coco_eval_golden.npz: the synthetic case of tests/coco_eval_cases.py and what the reference's own pycocotools
(oracle/build_cocoapi.sh) computes on it -- COCOeval precision / recall / scores / stats for 'bbox' and 'segm' after the notebooks'
results-file conversion, the IoU matrices of sampled (image, category) pairs, and every GT mask as COCO.annToRLE gives it
(frPyObjects + merge), as its compressed string.
    python tests/golden/make_coco_eval_golden.py"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import coco_eval_cases as cc  # noqa: E402
from oracle import cocoapi  # noqa: E402


def main(seed=0):
    mods = cocoapi.load()
    mask = mods[2]
    enc = lambda m: mask.encode(np.asfortranarray(m[:, :, None]))[0]['counts'].decode()   # noqa: E731
    ds, boxes, segms = cc.make_case(seed, encode=enc)
    case = dict(dataset=ds, all_boxes=[[b.tolist() if len(b) else [] for b in c] for c in boxes], all_segms=segms)
    out = dict(case=np.frombuffer(json.dumps(case).encode(), np.uint8))
    for t in ('bbox', 'segm'):
        E = cc.oracle_eval(mods, ds, boxes, segms, t)
        out[t + '_precision'], out[t + '_recall'], out[t + '_scores'] = E.eval['precision'], E.eval['recall'], E.eval['scores']
        out[t + '_stats'] = np.array(E.stats, np.float64)
        keys = sorted(k for k, v in E.ious.items() if len(v))
        pick = [keys[i] for i in np.linspace(0, len(keys) - 1, min(24, len(keys))).astype(int)]
        out[t + '_iou_keys'] = np.array(pick, np.int64).reshape(-1, 2)
        out[t + '_iou_shapes'] = np.array([E.ious[k].shape for k in pick], np.int64).reshape(-1, 2)
        out[t + '_iou_values'] = np.concatenate([np.asarray(E.ious[k], np.float64).reshape(-1) for k in pick])
        if t == 'segm':
            gt = E.cocoGt
            rles = {str(a['id']): gt.annToRLE(a)['counts'] for a in ds['annotations']}
            rles = {k: (v.decode() if isinstance(v, bytes) else v) for k, v in rles.items()}
            out['gt_rles'] = np.frombuffer(json.dumps(rles).encode(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "coco_eval_golden.npz"), **out)
    print("wrote coco_eval_golden.npz: bbox AP %.4f, segm AP %.4f" % (out['bbox_stats'][0], out['segm_stats'][0]))


if __name__ == "__main__":
    main()
