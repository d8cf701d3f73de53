"""The launch plan of dgx_var_propagate / dgx_var_level_agg and their device forms (dgx_api.cu vv_run, vv_passes,
la_run) restated in Python.  Its constants are read from the CUDA sources and the statements it restates are matched
as text, so a rewrite fails loudly here instead of drifting.
"""
from __future__ import annotations

import os
import re

from groupby_plan import K as GB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the value-variable plan model (tests/valvar_plan.py)")
    return m


def _body(name, text):
    return _one(r"(?s)static \w+ " + name + r"\(.*?\n\}\n", text, name).group(0)


def read_constants(api: str | None = None, kern: str | None = None) -> dict:
    if api is None:
        with open(os.path.join(CSRC, "dgx_api.cu")) as f:
            api = f.read()
    if kern is None:
        with open(os.path.join(CSRC, "valvar_kernel.cuh")) as f:
            kern = f.read()
    K = {"RANGE_BITS": int(_one(r"constexpr int VV_RANGES = 4, VV_RANGE_BITS = (\d+);", kern, "the range bits").group(1))}
    _one(r"return \(gb_bits\(ndest \? ndest - 1 : 0\) \+ VV_RANGE_BITS \+ GB_DIGIT_BITS - 1\) / GB_DIGIT_BITS;",
         _body("vv_passes", api), "vv_passes")
    run = _body("vv_run", api)
    per = [int(x) for x in re.findall(r"count_launches\(l, (\d+)\);", run)]
    if len(per) != 1 or run.count("<<<") != per[0] or run.count("gb_sort(") != 1:
        raise ValueError("vv_run's launches changed: restate them in the value-variable plan model")
    K["LEVEL"] = per[0]
    la = _body("la_run", api)
    agg = [int(x) for x in re.findall(r"count_launches\(l, (\d+)\);", la)]
    if len(agg) != 1 or la.count("<<<") != agg[0]:
        raise ValueError("la_run's launches changed: restate them in the value-variable plan model")
    K["AGG"] = agg[0]
    K["SORT_PER_PASS"] = GB["SORT_PER_PASS"]
    K["DIGIT_BITS"] = GB["DIGIT_BITS"]
    return K


K = read_constants()


def passes(ndest: int) -> int:
    b_d = int(ndest - 1 if ndest else 0).bit_length()
    return -(-(b_d + K["RANGE_BITS"]) // K["DIGIT_BITS"])


def propagate_launches(n: int, ndests) -> int:
    """Kernel launches of one propagation: nothing for an empty map, else per level the fixed kernels and the radix
    sort's passes over rank << 2 | range.  Rows, values and the map's size do not enter."""
    if n == 0:
        return 0
    return sum(K["LEVEL"] + K["SORT_PER_PASS"] * passes(d) for d in ndests)


def level_agg_launches(n: int, nrows: int, values: int) -> int:
    """4 launches whatever the sizes, none when the map, the rows or the values are empty."""
    return 0 if n == 0 or nrows == 0 or values == 0 else K["AGG"]
