#!/usr/bin/env bash
# Builds the reference's vendored pycocotools (lib/cocoapi: coco.py, cocoeval.py, mask.py, _mask.pyx + common/maskApi.c) from where it
# lies under $REF (read-only) into oracle/_ref/pycocotools/ (git-ignored), offline, with Cython.  Nothing is copied into the repo: the
# sources are copied to a temp dir, where _mask.pyx gets its one numpy-2 token (np.NPY_OWNDATA -> np.NPY_ARRAY_OWNDATA).  The Python
# 3 / numpy 2 shims the modules need at import time are applied by oracle/cocoapi.py, not by editing them.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=$HERE/_ref/pycocotools
API=$REF/lib/cocoapi
if [ ! -d "$API/PythonAPI/pycocotools" ]; then echo "build_cocoapi: $API not present - using prebuilt $OUT"; exit 0; fi
if ! python -c "import Cython" 2>/dev/null; then echo "build_cocoapi: Cython not importable - pycocotools oracle not built"; exit 0; fi
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
# the same layout as lib/cocoapi: _mask.pyx names its C source as ../common/maskApi.c
mkdir -p "$TMP/PythonAPI/pycocotools" "$TMP/common"
cp "$API/common/maskApi.c" "$API/common/maskApi.h" "$TMP/common/"
cp "$API/PythonAPI/pycocotools/"*.py "$TMP/PythonAPI/pycocotools/"
sed -e 's/np\.NPY_OWNDATA/np.NPY_ARRAY_OWNDATA/g' "$API/PythonAPI/pycocotools/_mask.pyx" > "$TMP/PythonAPI/pycocotools/_mask.pyx"
cat > "$TMP/PythonAPI/setup.py" <<'PY'
from setuptools import setup, Extension
from Cython.Build import cythonize
import numpy as np
setup(ext_modules=cythonize([Extension("pycocotools._mask", ["pycocotools/_mask.pyx"],
                                       include_dirs=[np.get_include(), "../common"],
                                       extra_compile_args=["-Wno-cpp", "-Wno-unused-function", "-std=c99"])],
                            language_level=3, quiet=True))
PY
(cd "$TMP/PythonAPI" && python setup.py -q build_ext --inplace >/dev/null 2>&1)
rm -rf "$OUT"
mkdir -p "$OUT"
cp "$TMP/PythonAPI/pycocotools/"*.py "$TMP/PythonAPI/pycocotools/"_mask*.so "$OUT/"
ls "$OUT"
