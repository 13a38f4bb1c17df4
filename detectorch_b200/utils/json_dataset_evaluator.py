"""evaluate_boxes / evaluate_masks of the reference's lib/utils/json_dataset_evaluator.py (:40-64, :128-146) on the device: the same
signatures and the same COCOeval numbers (coco_eval.evaluate), without writing, reloading or keeping a results file.  A notebook
switches with one import line:
    from detectorch_b200.utils.json_dataset_evaluator import evaluate_boxes, evaluate_masks
json_dataset.COCO.dataset supplies the ground truth (built on the device once per json_dataset, kept on it); its classes /
category_to_id_map give the json category id of each contiguous class, as _write_coco_*_results_file uses them.
evaluate_box_proposals (:238-320) is the proposal recall of coco_eval.box_proposal_recall, one (area, limit) combination.
_write_coco_bbox_results_file / _write_coco_segms_results_file (:67-190) write the reference's results json, byte for byte, with
coco_eval.write_results (for test-dev, whose evaluation returns None, the file is the only output).
_do_detection_eval / _do_segmentation_eval (:116-125, :193-202) evaluate a results file, parsed on the device (coco_eval.load_results):
    E = _do_segmentation_eval(json_dataset, "segmentations_results.json", output_dir)"""
import logging
import os

import numpy as np

from . import coco_eval

logger = logging.getLogger(__name__)


def _ground_truth(json_dataset):
    gt = getattr(json_dataset, "_device_coco_gt", None)
    if gt is None:
        gt = coco_eval.CocoGroundTruth(json_dataset.COCO.dataset)
        json_dataset._device_coco_gt = gt
    return gt


def _category_ids(json_dataset):
    return [json_dataset.category_to_id_map[c] for c in json_dataset.classes if c != '__background__']


def _evaluate(json_dataset, all_boxes, all_segms, iou_type):
    # Only do evaluation on non-test sets (annotations are undisclosed on test), as the reference
    if json_dataset.name.find('test') != -1:
        return None
    E = coco_eval.evaluate(_ground_truth(json_dataset), all_boxes, iou_type, all_segms, category_ids=_category_ids(json_dataset))
    _log_detection_eval_metrics(E)
    return E


def evaluate_masks(json_dataset, all_boxes, all_segms, output_dir, use_salt=True, cleanup=False):
    """-> the evaluation ('segm'): .eval['precision' | 'recall' | 'scores'], .stats, .params.  output_dir / use_salt / cleanup are
    accepted for the reference's signature; nothing is written."""
    return _evaluate(json_dataset, all_boxes, all_segms, 'segm')


def evaluate_boxes(json_dataset, all_boxes, output_dir, use_salt=True, cleanup=False):
    """-> the evaluation ('bbox'), as evaluate_masks."""
    return _evaluate(json_dataset, all_boxes, None, 'bbox')


def _results_ground_truth(json_dataset):
    """The images (json_dataset.COCO.getImgIds(), sorted) and categories the results files are written for; no annotations."""
    cats = list(dict.fromkeys(_category_ids(json_dataset)))
    return coco_eval.CocoGroundTruth({'images': [{'id': i, 'height': 1, 'width': 1} for i in sorted(json_dataset.COCO.getImgIds())],
                                      'categories': [{'id': c} for c in cats]})


def _write_coco_segms_results_file(json_dataset, all_boxes, all_segms, res_file):
    """The reference's segm results json (all_boxes / all_segms [class][image], or a DeviceResults with all_segms None), byte for
    byte; a non-finite box or score raises ValueError (see coco_eval.write_results)."""
    logger.info('Writing segmentation results json to: {}'.format(os.path.abspath(res_file)))
    coco_eval.write_results(_results_ground_truth(json_dataset), all_boxes, 'segm', res_file, all_segms,
                            category_ids=_category_ids(json_dataset))


def _write_coco_bbox_results_file(json_dataset, all_boxes, res_file):
    """The reference's bbox results json, as _write_coco_segms_results_file."""
    logger.info('Writing bbox results json to: {}'.format(os.path.abspath(res_file)))
    coco_eval.write_results(_results_ground_truth(json_dataset), all_boxes, 'bbox', res_file, category_ids=_category_ids(json_dataset))


def _do_file_eval(json_dataset, res_file, iou_type):
    gt = _ground_truth(json_dataset)
    E = coco_eval.evaluate(gt, coco_eval.load_results(gt, str(res_file)), iou_type)
    _log_detection_eval_metrics(E)
    return E


def _do_segmentation_eval(json_dataset, res_file, output_dir):
    """COCOeval(json_dataset.COCO, json_dataset.COCO.loadRes(res_file), 'segm') after evaluate() + accumulate(), logged -> the
    evaluation (coco_eval.load_results + evaluate).  output_dir is accepted for the reference's signature; nothing is written (the
    reference pickles the COCOeval object there)."""
    return _do_file_eval(json_dataset, res_file, 'segm')


def _do_detection_eval(json_dataset, res_file, output_dir):
    """The 'bbox' evaluation of a results file, as _do_segmentation_eval."""
    return _do_file_eval(json_dataset, res_file, 'bbox')


def _log_detection_eval_metrics(E):
    ind_lo = np.where(np.isclose(E.params.iouThrs, 0.5))[0][0]
    ind_hi = np.where(np.isclose(E.params.iouThrs, 0.95))[0][0]
    precision = E.eval['precision'][ind_lo:(ind_hi + 1), :, :, 0, 2]
    ap = np.mean(precision[precision > -1]) if np.any(precision > -1) else -1
    logger.info('~~~~ Mean and per-category AP @ IoU=[0.50,0.95] ~~~~')
    logger.info('{:.1f}'.format(100 * ap))
    E.summarize()


def evaluate_box_proposals(json_dataset, roidb, thresholds=None, area='all', limit=None):
    """Detectron's proposal recall (AR over IoU thresholds for one area range and proposal limit) -> {'ar', 'recalls', 'thresholds',
    'gt_overlaps', 'num_pos'}, equal to the reference's; the greedy matching runs on the device.  An unknown area raises ValueError."""
    if area not in coco_eval.PROPOSAL_AREAS:
        raise ValueError('Unknown area range: {}'.format(area))
    return coco_eval.box_proposal_recall(roidb, [area], [limit], thresholds)[(area, limit)]
