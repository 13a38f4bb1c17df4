"""Writes proposal_recall_golden.npz with the reference's own evaluate_box_proposals (lib/utils/json_dataset_evaluator.py:238-320) on
its compiled cython_bbox.bbox_overlaps (oracle/cython_bbox.py), for the cases of tests/proposal_recall_cases.py.
Run from the repository root: python tests/golden/make_proposal_recall_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    from oracle import cython_bbox
    import proposal_recall_cases as cases
    jde, _ = cython_bbox.load()
    out = {}
    names = []
    for k, (name, roidb, area, limit, thr) in enumerate(cases.edge_cases()):
        r = jde.evaluate_box_proposals(None, roidb, thresholds=None if thr is None else thr.copy(), area=area, limit=limit)
        names.append(name)
        out["%s/recalls" % name] = r['recalls']
        out["%s/gt_overlaps" % name] = r['gt_overlaps']
        out["%s/ar" % name] = np.float64(r['ar'])
        out["%s/num_pos" % name] = np.int64(r['num_pos'])
        out["%s/thresholds" % name] = np.asarray(r['thresholds'])
    out["names"] = np.array(names)
    path = os.path.join(ROOT, "tests", "golden", "proposal_recall_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(names), "cases")


if __name__ == "__main__":
    main()
