"""Host checks of the device results-file reader's inputs: the generated power-of-five table entry for entry against Python
integers, and the case corpus of tests/results_file_cases.py against json.loads."""
import json
import math
import os
import re

import results_file_cases as rc

from detectorch_b200 import build


def _parse_table(text):
    body = lambda name: re.search(r"#define %s \{\\\n(.*?)\}" % name, text, re.S).group(1)
    words = [int(w, 16) for w in re.findall(r"0x([0-9a-f]{16})ull", body("DT_POW5_T"))]
    shifts = [int(v) for v in re.findall(r"-?\d+", body("DT_POW5_S"))]
    return words, shifts


def test_pow5_table_matches_python_integers():
    words, shifts = _parse_table(build.pow5_table())
    qs = range(build.P5_MIN, build.P5_MAX + 1)
    assert len(words) == 2 * len(qs) and len(shifts) == len(qs)
    for n, q in enumerate(qs):
        t = (words[2 * n] << 64) | words[2 * n + 1]
        s = shifts[n]
        assert 2 ** 127 <= t < 2 ** 128
        # t = floor(5^q 2^s): t <= 5^q 2^s < t + 1, in integers on whichever side is fractional
        num, den = (5 ** q, 1) if q >= 0 else (1, 5 ** -q)
        num, den = (num << s, den) if s >= 0 else (num, den << -s)
        assert t * den <= num < (t + 1) * den, q


def test_pow5_table_is_what_build_writes():
    build.write_pow10_table()
    with open(build.POW5) as f:
        assert f.read() == build.pow5_table()


def test_malformed_corpus_is_rejected_by_json():
    for text in rc.MALFORMED:
        try:
            json.loads(rc.encode(text))
        except ValueError:
            continue
        raise AssertionError("json.loads accepts %r" % text[:80])


def test_not_array_corpus_is_json_but_not_an_array_of_objects():
    for text in rc.NOT_ARRAY:
        v = json.loads(text)
        assert not (isinstance(v, list) and all(isinstance(r, dict) for r in v)), text


def test_extra_refusals_are_json_with_nan_or_non_ascii():
    for text in rc.EXTRA:
        data = rc.encode(text)
        json.loads(data)                                  # accepted by json.loads ...
        nan = re.search(r"NaN|Infinity", text) is not None
        assert nan or max(data) >= 0x80, text             # ... and refused for a documented reason


def test_variants_read_back_as_the_records():
    recs = [{"image_id": 3, "category_id": 2, "bbox": [1.5, 2.0, 3.25, 4.0], "score": 0.75,
             "segmentation": {"size": [4, 5], "counts": "0\\1/2"}}, {"image_id": 1, "category_id": 7, "bbox": [0, 1e-5, 2, 3], "score": 1}]
    for name, data in rc.variants(recs, 0):
        got = json.loads(data)
        strip = [{k: v for k, v in r.items() if k not in ("note", "zz")} for r in got]
        assert strip == recs, name
    assert json.loads(rc.duplicate_keys(recs)) == recs
    assert json.loads(rc.escaped_counts(recs)) == recs


def test_numbers_are_json_numbers():
    nums = rc.numbers(1, 3000)
    assert len(nums) == 3000
    vals = json.loads("[" + ", ".join(nums) + "]")
    assert all(isinstance(v, (int, float)) and math.isfinite(float(v)) for v in vals)
