"""The launch plan of dgx_math_eval / dgx_dev_math_eval (dgx_api.cu mt_run) restated in Python.  Its constants are read
from the CUDA sources and the statements it restates are matched as text, so a rewrite fails loudly here instead of
drifting.
"""
from __future__ import annotations

import os
import re

from merge_geometry import tree_launches
from merge_matrix_geometry import K as XM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the math plan model (tests/math_plan.py)")
    return m


def read_constants(api: str | None = None) -> dict:
    if api is None:
        with open(os.path.join(CSRC, "dgx_api.cu")) as f:
            api = f.read()
    body = _one(r"(?s)static int mt_run\(.*?\n\}\n", api, "mt_run").group(0)
    counts = [int(x) for x in re.findall(r"count_launches\(l, (\d+)\);", body)]
    if len(counts) != 2 or body.count("<<<") != sum(counts) or body.count("merge_matrix_impl(") != 1:
        raise ValueError("mt_run's launches changed: restate them in the math plan model")
    _one(r"merge_matrix_impl\(l, [^;]*, nl, cap,", body, "the key-union merge over the leaves' total room")
    return {"FRONT": counts[0], "BACK": counts[1], "MERGE": XM["LAUNCHES"], "XM_T": XM["XM_T"]}


K = read_constants()


def launches(cap: int) -> int:
    """Kernel launches of one call, cap the leaves' total room (the sum of their n): check, plan and gather, the key
    union's matrix merge with its sample tree when any leaf has room, then eval, scan, finish and write.  Neither the
    program's size nor the entry counts enter."""
    merge = K["MERGE"] + tree_launches(-(-cap // K["XM_T"])) if cap else 0
    return K["FRONT"] + merge + K["BACK"]
