"""The launch plan of dgx_path_expand / dgx_dev_path_expand (dgx_api.cu ps_level) restated in Python.  Its constants
are read from the CUDA sources and the statements it restates are matched as text, so a rewrite fails loudly here
instead of drifting.
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
        raise ValueError(f"{what} changed: restate it in the shortest-path plan model (tests/shortest_plan.py)")
    return m


def read_constants(api: str | None = None) -> dict:
    if api is None:
        with open(os.path.join(CSRC, "dgx_api.cu")) as f:
            api = f.read()
    body = _one(r"(?s)static int ps_level\(.*?\n\}\n", api, "ps_level").group(0)
    counts = [int(x) for x in re.findall(r"count_launches\(l, (\d+)\);", body)]
    if len(counts) != 2 or body.count("<<<") != sum(counts) or body.count("merge_matrix_impl(") != 2:
        raise ValueError("ps_level's launches changed: restate them in the shortest-path plan model")
    _one(r"merge_matrix_impl\(l, U\(P\.nv\), U\(P\.nv_off\), rc1, vc,", body, "the new-node merge (max(1, v_cap))")
    _one(r"merge_matrix_impl\(l, U\(P\.es\), U\(P\.es_off\), nsg, rc1,", body, "the expanded merge (max(1, rows))")
    _one(r"ps_insert_kernel<<<stride_grid\(\), 256, 0, l->stream>>>\(P\);", body, "the insert grid")
    res = _one(r"(?s)extern \"C\" int dgx_path_result\(.*?\n\}\n", api, "dgx_path_result").group(0)
    walk = len(re.findall(r"count_launches\(l, (\d+)\);", res))
    return {"FRONT": counts[0], "BACK": counts[1], "MERGE": XM["LAUNCHES"], "XM_T": XM["XM_T"], "WALK": walk}


K = read_constants()


def launches(rows: int, values: int) -> int:
    """Kernel launches of one level (rows and values are src_off[nsg] and v_off[rows] for the host form, src_cap and
    v_cap for the device form): the front, two matrix merges with sample trees of max(1, ceil(log2 ceil(n / XM_T)))
    levels for n = max(1, values) and max(1, rows), and the back.  The sg count, dest count and set sizes do not
    enter."""
    m = K["MERGE"] + tree_launches(-(-max(values, 1) // K["XM_T"]))
    e = K["MERGE"] + tree_launches(-(-max(rows, 1) // K["XM_T"]))
    return K["FRONT"] + m + e + K["BACK"]
