"""Cases of the device reader of COCO results files (coco_eval.load_results): a corpus of malformed JSON, re-serialisations of a
results list that json.loads reads back to the same records, and decimal numbers that exercise every path of a correctly rounded
conversion (the exact big-integer decisions included)."""
import json
import math
import random
import struct
from decimal import Decimal, localcontext

BASE = '{"image_id": 1, "category_id": 1, "bbox": [1.5, 2, 3, 4], "score": 0.5}'


def _rec(**kw):
    d = {"image_id": "1", "category_id": "1", "bbox": "[1.5, 2, 3, 4]", "score": "0.5"}
    d.update(kw)
    return "{" + ", ".join('"%s": %s' % (k, v) for k, v in d.items() if v is not None) + "}"


# text json.loads rejects (each must also be refused by load_results)
MALFORMED = [
    "", " ", "[", "]", "[" + BASE, "[" + BASE + ",]", "[," + BASE + "]", "[" + BASE + " " + BASE + "]", "[" + BASE + "] x",
    "[" + BASE + "][]", "[" + BASE + "]]", "[[" + BASE + "]", "[{]", "[{}}]", "[" + BASE[:-1] + "]",
    "[" + BASE[:-1] + ",}]", "[" + BASE.replace(":", "", 1) + "]", "[" + BASE.replace('"image_id"', "image_id") + "]",
    "[" + BASE.replace('"image_id"', "'image_id'") + "]", "[" + _rec(score="01") + "]", "[" + _rec(score="00.5") + "]",
    "[" + _rec(score="+1") + "]", "[" + _rec(score=".5") + "]", "[" + _rec(score="1.") + "]", "[" + _rec(score="1e") + "]",
    "[" + _rec(score="1e+") + "]", "[" + _rec(score="-") + "]", "[" + _rec(score="--1") + "]", "[" + _rec(score="0x10") + "]",
    "[" + _rec(score="1.5.5") + "]", "[" + _rec(score="1 2") + "]", "[" + _rec(score="True") + "]", "[" + _rec(score="nul") + "]",
    "[" + _rec(score="") + "]", "[" + _rec(extra='"a\tb"') + "]", "[" + _rec(extra='"a\\x"') + "]", "[" + _rec(extra='"\\u12"') + "]",
    "[" + _rec(extra='"\\u12g4"') + "]", "[" + _rec(extra='"abc') + "]", "[" + _rec(extra="[1, 2}") + "]", "[" + _rec(extra="{]") + "]",
    "[" + _rec(extra='{"a" 1}') + "]", "[" + _rec(extra='{"a": }') + "]", "[" + _rec(extra="[1,]") + "]", "[" + _rec(extra='{1: 2}') + "]",
    "[" + _rec(extra='"\n"') + "]", "[" + _rec(extra="tru") + "]", "[" + _rec(extra="[[[[]]]") + "]", "[" + BASE + "\x0c]",
    "[" + _rec(extra="[" * 70 + "]" * 69) + "]",
]
# JSON, but not an array of objects (loadRes asserts a list; its records are dicts)
NOT_ARRAY = [BASE, "{}", '"[]"', "1", "[1]", "[[]]", "[null]", "[" + BASE + ", 2]", '["x"]']
# valid for json.loads, refused by load_results: NaN / Infinity literals and bytes >= 0x80 (json.dump writes neither)
EXTRA = [
    "[" + _rec(score="NaN") + "]", "[" + _rec(score="Infinity") + "]", "[" + _rec(score="-Infinity") + "]",
    "[" + _rec(extra="NaN") + "]", "[" + _rec(extra='"café"') + "]", "﻿[" + BASE + "]",
]


def encode(text):
    return text.encode("utf-8")


def variants(records, seed):
    """(name, bytes) re-serialisations of `records` that json.loads reads back as the same list (records shuffled: as the list
    given with them)."""
    rng = random.Random(seed)
    out = [("indent", json.dumps(records, indent=2)), ("tabs", json.dumps(records, indent="\t")),
           ("crlf", json.dumps(records, indent=1).replace("\n", "\r\n")), ("compact", json.dumps(records, separators=(",", ":")))]
    shuffled_keys = [dict(rng.sample(list(r.items()), len(r))) for r in records]
    out.append(("keys shuffled", json.dumps(shuffled_keys)))
    extra = []
    for n, r in enumerate(records):
        r = dict(r)
        r["note"] = 'a \\"quoted\\" {brace] é'.encode("ascii", "backslashreplace").decode() if n % 3 == 0 else [1, {"x": [[], {}]}, "]"]
        r["zz"] = {"deep": [[[{"k": "v"}]]], "t": True, "f": False, "n": None, "num": -1.5e-3}
        extra.append(r)
    out.append(("extra keys", json.dumps(extra)))
    return [(n, t.encode()) for n, t in out]


def duplicate_keys(records):
    """Text with a first, overridden occurrence of every key loadRes reads (json.loads keeps the last)."""
    dup = {"image_id": "-5", "category_id": "123456", "score": '"x"', "bbox": "[1]", "segmentation": "[[1, 2]]"}
    parts = []
    for r in records:
        first = "".join('"%s": %s, ' % (k, v) for k, v in dup.items() if k in r)
        parts.append("{" + first + json.dumps(r)[1:])
    return ("[" + ", ".join(parts) + "]").encode()


def escaped_counts(records):
    """Every RLE string with its characters \\u-escaped in turn (and '/' as '\\/' where it occurs)."""
    out = []
    for r in records:
        body = json.dumps(r)
        seg = r.get("segmentation")
        if isinstance(seg, dict) and isinstance(seg.get("counts"), str):
            c = seg["counts"]
            enc = json.dumps(c)[1:-1]
            esc = "".join("\\u%04x" % ord(ch) if i % 2 == 0 else "\\/" if ch == "/" else json.dumps(ch)[1:-1] for i, ch in enumerate(c))
            body = body.replace('"' + enc + '"', '"' + esc + '"', 1)
        out.append(body)
    return ("[" + ", ".join(out) + "]").encode()


def number_forms(v):
    """Other spellings of the float v (json.loads gives v for each)."""
    r = repr(v)
    out = [r]
    if math.isfinite(v) and v == int(v) and abs(v) < 1e15:
        out += [str(int(v)), "%de0" % int(v), "%dE+00" % int(v)]
    m, e = ("%.17e" % v).split("e")
    out.append("%sE%d" % (m, int(e)))
    return [x for x in out if float(x) == v]


def _bits(x):
    return struct.unpack("<q", struct.pack("<d", x))[0]


def _from_bits(b):
    return struct.unpack("<d", struct.pack("<q", b))[0]


def _halfway(b):
    """The exact decimal of the midpoint of the positive double of bits b and the next one up."""
    with localcontext() as ctx:
        ctx.prec = 2000
        return (Decimal(_from_bits(b)) + Decimal(_from_bits(b + 1))) / 2


def numbers(seed, n):
    """n JSON number texts: repr of random finite doubles and those cut to 15 / 16 digits; 1-40 digit mantissas with exponents -350 ..
    310; exact halfway points (normal and subnormal) written in full and one unit in the last digit either side; the edge cases;
    integers of up to 309 digits and 400-digit mantissas below the overflow bound; exponents written with 30 digits."""
    rng = random.Random(seed)
    out = ["2.2250738585072011e-308", "4.9e-324", "2.4703282292062328e-324", "2.4703282292062327e-324", "1e-400", "-1e-400",
           "1.7976931348623158e308", "1.7976931348623157e308", "-0", "-0.0", "0", "0.0", "-0e5", "1e-324", "5e-324", "2.5e-324",
           "9007199254740993", "9007199254740992.5", "123456789012345678901234567890", "0." + "0" * 400 + "1e400",
           "1" + "0" * 308, "17976931348623157" + "0" * 292]
    while len(out) < n:
        kind = rng.randrange(7)
        if kind == 0:
            while True:
                v = _from_bits(rng.getrandbits(64) - (1 << 63))
                if math.isfinite(v):
                    break
            out += [repr(v), "%.15g" % v, "%.16g" % v]
        elif kind == 1:
            d = str(rng.randrange(1, 10)) + "".join(str(rng.randrange(10)) for _ in range(rng.randrange(40)))
            e = rng.randrange(-350, 311)
            t = ("-" if rng.random() < .3 else "") + (d[0] + "." + d[1:] if len(d) > 1 and rng.random() < .5 else d) + "e%d" % e
            try:
                if math.isfinite(float(t)):
                    out.append(t)
            except OverflowError:
                pass
        elif kind in (2, 3):
            b = rng.randrange(1, 1 << 52) if kind == 2 else rng.randrange(1 << 52, (0x7fe << 52))
            h = _halfway(b)
            unit = Decimal(1).scaleb(h.as_tuple().exponent)
            for x in (h, h - unit, h + unit):
                out.append(format(x, "f") if abs(x.adjusted()) < 40 else str(x))
        elif kind == 4:
            nd = rng.randrange(290, 310)
            out.append(str(rng.randrange(10 ** (nd - 1), min(10 ** nd, int(1.7976931348623157e308)))))
        elif kind == 5:
            d = str(rng.randrange(1, 10)) + "".join(str(rng.randrange(10)) for _ in range(399))
            out.append(d + "e%d" % rng.randrange(-700, -92))
        else:
            m = "%d.%d" % (rng.randrange(1, 10), rng.randrange(10 ** 6))
            e = rng.randrange(-320, 300)
            out.append(m + "e" + ("-" if e < 0 else "+") + str(abs(e)).zfill(30))
    return out[:n]
