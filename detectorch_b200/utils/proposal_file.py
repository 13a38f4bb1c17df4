"""Detectron proposals pickle: what JsonDataset._add_proposals_from_file (lib/data/json_dataset.py:237-266) reads -- a dict of
'boxes' (float32 [n, 4] per image, original-image x1 y1 x2 y2), 'scores' (float32 [n]) and 'ids' (the COCO image ids), one entry per
image of the dataset.  The reader sorts the entries by id and pairs them with the roidb's images in sorted-id order, so every image of
the dataset needs exactly one entry.  A file written here feeds eval_fast_FPN.ipynb's proposal_file= and detect(proposals=).

    props = model.propose_images(ims)                                  # [(boxes, scores)] in the order of image_ids
    write_proposals_file("rpn_proposals.pkl", image_ids, props)
"""
import pickle

import numpy as np


def write_proposals_file(path, image_ids, proposals):
    """image_ids: one COCO image id per entry; proposals: one (boxes [n, 4], scores [n]) per entry (propose_images output).  The entries
    are written in ascending id order.  Raises ValueError on mismatched lengths, repeated ids or malformed arrays."""
    ids = [int(i) for i in image_ids]
    proposals = list(proposals)
    if len(ids) != len(proposals):
        raise ValueError("write_proposals_file: %d image ids for %d proposal sets" % (len(ids), len(proposals)))
    if len(set(ids)) != len(ids):
        raise ValueError("write_proposals_file: repeated image id")
    boxes, scores = [], []
    for i, p in zip(ids, proposals):
        if not isinstance(p, (tuple, list)) or len(p) != 2:
            raise ValueError("write_proposals_file: image %d: expected a (boxes, scores) pair" % i)
        b, s = np.asarray(p[0], np.float32), np.asarray(p[1], np.float32)
        if b.ndim != 2 or b.shape[1] != 4 or s.shape != (b.shape[0],):
            raise ValueError("write_proposals_file: image %d: boxes must be [n, 4] and scores [n]" % i)
        boxes.append(np.ascontiguousarray(b))
        scores.append(np.ascontiguousarray(s))
    order = np.argsort(np.array(ids, np.int64), kind='stable')
    data = {'boxes': [boxes[k] for k in order], 'scores': [scores[k] for k in order], 'ids': [ids[k] for k in order]}
    with open(path, 'wb') as f:
        pickle.dump(data, f, protocol=pickle.HIGHEST_PROTOCOL)
