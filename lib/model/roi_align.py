"""Overlay of lib/model/roi_align.py: RoIAlignFunction / RoIAlign / preprocess_rois over the sm_90a kernel."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from detectorch_b200.model.roi_align import RoIAlignFunction, RoIAlign, preprocess_rois  # noqa: E402,F401
