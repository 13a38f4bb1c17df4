"""Overlay for notebooks that do `sys.path.insert(0, "lib/")` + `from model.detector import detector`
(eval_mask_FPN.ipynb cell 1): resolves to the H100 engine-backed mirror."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from detectorch_b200.model.detector import detector  # noqa: E402,F401
