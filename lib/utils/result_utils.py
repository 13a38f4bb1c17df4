"""Overlay of lib/utils/result_utils.py for notebooks that do `import utils.result_utils as result_utils` (eval_*.ipynb cell 1): every name
the notebooks use -- empty_results (cell 9), postprocess_output / segm_results / extend_results (cell 10), to_np -- resolves to the H100
mirror (postprocess_output and segm_results run on the device)."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from detectorch_b200.utils.result_utils import (empty_results, extend_results, postprocess_output, segm_results,  # noqa: E402,F401
                                                to_np)
