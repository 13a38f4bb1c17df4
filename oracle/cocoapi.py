"""The reference's vendored pycocotools, built by oracle/build_cocoapi.sh into oracle/_ref/pycocotools, imported with the shims it
needs on Python 3.12 / numpy 2 -- applied to its modules only, nothing process-wide:
  * coco.py imports matplotlib (plotting only): stub modules are registered when matplotlib itself is not importable;
  * coco.py's loadRes names `unicode`: the module gets unicode = str;
  * cocoeval.py uses np.float and passes a float count to np.linspace: the module sees a numpy whose float is float and whose
    linspace takes int(num)."""
import importlib
import os
import sys
import types

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, "_ref")
_mods = None


def available():
    d = os.path.join(REF_DIR, "pycocotools")
    return os.path.isdir(d) and any(f.startswith("_mask") and f.endswith(".so") for f in os.listdir(d))


def build():
    import subprocess
    subprocess.check_call(["bash", os.path.join(_HERE, "build_cocoapi.sh")], stdout=subprocess.DEVNULL)


def load():
    """-> (COCO, COCOeval, mask module) of the built reference pycocotools; ImportError when it is not built."""
    global _mods
    if _mods is not None:
        return _mods
    if not available():
        raise ImportError("reference pycocotools not built under %s (oracle/build_cocoapi.sh)" % REF_DIR)
    try:
        import matplotlib.pyplot  # noqa: F401
    except ImportError:
        for m in ("matplotlib", "matplotlib.pyplot", "matplotlib.collections", "matplotlib.patches"):
            sys.modules.setdefault(m, types.ModuleType(m))
        sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
        sys.modules["matplotlib.collections"].PatchCollection = None
        sys.modules["matplotlib.patches"].Polygon = None
    if REF_DIR not in sys.path:
        sys.path.insert(0, REF_DIR)
    coco = importlib.import_module("pycocotools.coco")
    coco.unicode = str
    cocoeval = importlib.import_module("pycocotools.cocoeval")
    shim = types.ModuleType("numpy")
    shim.__dict__.update(np.__dict__)
    shim.float = float
    shim.linspace = lambda start, stop, num=50, **kw: np.linspace(start, stop, int(num), **kw)
    cocoeval.np = shim
    mask = importlib.import_module("pycocotools.mask")
    _mods = (coco.COCO, cocoeval.COCOeval, mask)
    return _mods
