"""The launch plan of dgx_recurse_filter / dgx_dev_recurse_filter (dgx_api.cu rc_step) restated in Python.  Its
constants are read from the CUDA sources and the statements it restates are matched as text, so a rewrite fails loudly
here instead of drifting.
"""
from __future__ import annotations

import os
import re

from merge_geometry import tree_launches
from merge_matrix_geometry import K as XM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the recurse plan model (tests/recurse_plan.py)")
    return m


def read_constants(api: str | None = None) -> dict:
    api = _src("dgx_api.cu") if api is None else api
    body = _one(r"(?s)static int rc_step\(.*?\n\}\n", api, "rc_step").group(0)
    counts = [int(x) for x in re.findall(r"count_launches\(l, (\d+)\);", body)]
    if len(counts) != 2 or body.count("<<<") != sum(counts) or body.count("merge_matrix_impl(") != 1:
        raise ValueError("rc_step's launches changed: restate them in the recurse plan model")
    _one(r"rc_insert_kernel<<<stride_grid\(\), 256, 0, l->stream>>>\(P\);", body, "the insert grid")
    dev = _one(r"(?s)extern \"C\" int dgx_dev_recurse_filter\(.*?\n\}\n", api, "dgx_dev_recurse_filter").group(0)
    _one(r"if \(nrows == 0 \|\| v_cap == 0\) \{", dev, "the device form's empty step")
    host = _one(r"(?s)extern \"C\" int dgx_recurse_filter\(.*?\n\}\n", api, "dgx_recurse_filter").group(0)
    _one(r"if \(m == 0\) \{", host, "the host form's empty step")
    return {"FRONT": counts[0], "BACK": counts[1], "MERGE": XM["LAUNCHES"], "XM_T": XM["XM_T"]}


K = read_constants()


def launches(nrows: int, v_cap: int) -> int:
    """Kernel launches of one step: none without a row or a value (v_cap is v_off[nrows] for the host form), else the
    front, the matrix merge with its sample tree of max(1, ceil(log2 ceil(v_cap / XM_T))) levels, and the back.  Row
    count, kept count and set size do not enter."""
    if nrows == 0 or v_cap == 0:
        return 0
    return K["FRONT"] + K["MERGE"] + tree_launches(-(-v_cap // K["XM_T"])) + K["BACK"]
