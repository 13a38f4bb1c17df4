#!/usr/bin/env bash
# pre-commit check: the library must build for sm_90a and the CPU suite must pass
set -e
cd "$(dirname "$0")/.."
python -m detectorch_b200.build --force > /dev/null
python -m pytest tests -x -q -m "not gpu" 2>&1 | tail -2
