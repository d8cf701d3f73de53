"""The plan of dgx_groupby_uid / dgx_dev_groupby_uid (dgx_api.cu gb_plan, gb_front, gb_back, gb_sort) restated in
Python: the key widths, the radix passes and the launch count of one call.  Its constants are read from the CUDA
sources and the statements it restates are matched as text, so a rewrite fails loudly here instead of drifting.
"""
from __future__ import annotations

import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the groupby plan model (tests/groupby_plan.py)")
    return m


def _body(name, text):
    return _one(r"(?s)static \w+ " + name + r"\(.*?\n\}\n", text, name).group(0)


def read_constants(api: str | None = None, kern: str | None = None) -> dict:
    api = _src("dgx_api.cu") if api is None else api
    kern = _src("groupby_kernel.cuh") if kern is None else kern
    m = _one(r"constexpr int GB_NT = (\d+), GB_VT = (\d+), GB_TILE = GB_NT \* GB_VT;", kern, "the radix tile")
    K = {"GB_NT": int(m.group(1)), "GB_VT": int(m.group(2))}
    m = _one(r"constexpr int GB_RADIX = (\d+), GB_DIGIT_BITS = (\d+);", kern, "the radix digit")
    K["RADIX"], K["DIGIT_BITS"] = int(m.group(1)), int(m.group(2))
    if K["RADIX"] != 1 << K["DIGIT_BITS"]:
        raise ValueError("GB_RADIX is not 2^GB_DIGIT_BITS")
    plan = _body("gb_plan", api)
    for stmt in (r"g\.b_p = gb_bits\(npar - 1\);", r"g\.b_d = gb_bits\(ndest \? ndest - 1 : 0\);",
                 r"g\.b_s = gb_bits\(nrows\);",
                 r"g\.p1 = \(g\.b_p \+ g\.b_d \+ GB_DIGIT_BITS - 1\) / GB_DIGIT_BITS;",
                 r"g\.p2 = \(g\.b_p \+ g\.b_s \+ GB_DIGIT_BITS - 1\) / GB_DIGIT_BITS;"):
        _one(stmt, plan, "gb_plan")
    sort = _body("gb_sort", api)
    if sort.count("<<<") != 3:
        raise ValueError("gb_sort's launches changed: restate them in the groupby plan model")
    K["SORT_PER_PASS"] = int(_one(r"count_launches\(l, (\d+) \* \(int\)passes\);", sort, "gb_sort's count").group(1))
    front, back = _body("gb_front", api), _body("gb_back", api)
    K["FRONT"] = int(_one(r"count_launches\(l, (\d+)\);", front, "gb_front's count").group(1))
    K["BACK"] = int(_one(r"count_launches\(l, (\d+)\);", back, "gb_back's count").group(1))
    if front.count("<<<") != K["FRONT"] or back.count("<<<") != K["BACK"]:
        raise ValueError("the launches of gb_front / gb_back do not match their counts")
    if back.count("gb_sort(") != 2:
        raise ValueError("gb_back's sorts changed: restate them in the groupby plan model")
    return K


K = read_constants()


def bits(x: int) -> int:
    return int(x).bit_length()


def plan(nrows: int, ndest: int, npar: int) -> dict:
    b_p, b_d, b_s = bits(npar - 1), bits(ndest - 1 if ndest else 0), bits(nrows)
    d = K["DIGIT_BITS"]
    return {"b_p": b_p, "b_d": b_d, "b_s": b_s, "p1": -(-(b_p + b_d) // d), "p2": -(-(b_p + b_s) // d)}


def launches(nrows: int, ndest: int, npar: int, nvalues: int, npvalues: int, nedges: int, device_form=False) -> int:
    """Kernel launches of one call.  The host form launches nothing for npar == 0 or when there is no row value or no
    parent value, and only the front (checks, pairs, edge scan) when no edge remains; the device form launches nothing
    for npar, nrows, v_cap or par_cap of 0 (nvalues / npvalues stand for the caps there)."""
    if npar == 0 or nvalues == 0 or npvalues == 0 or (device_form and nrows == 0):
        return 0
    if nedges == 0 and not device_form:
        return K["FRONT"]
    p = plan(nrows, ndest, npar)
    return K["FRONT"] + K["BACK"] + K["SORT_PER_PASS"] * (p["p1"] + p["p2"])
