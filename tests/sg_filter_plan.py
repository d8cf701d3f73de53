"""The launch plan of dgx_sg_filter / dgx_dev_sg_filter (dgx_api.cu sf_run) restated in Python.  The statements it
restates are matched as text in the CUDA sources, so a rewrite fails loudly here instead of drifting.
"""
from __future__ import annotations

import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
HDR = os.path.join(ROOT, "include", "dgx.h")


def _src(path):
    with open(path) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the @filter plan model (tests/sg_filter_plan.py)")
    return m


def read_constants(api: str | None = None, hdr: str | None = None) -> dict:
    """{"LAUNCHES": launches of a call with a D0 slot, "MAX_NODES", "MAX_LEAVES", "MAX_DEPTH": the tree limits}."""
    api = _src(os.path.join(CSRC, "dgx_api.cu")) if api is None else api
    hdr = _src(HDR) if hdr is None else hdr
    body = _one(r"(?s)static int sf_run\(.*?\n\}\n", api, "sf_run").group(0)
    n = int(_one(r"count_launches\(l, (\d+)\);", body, "sf_run's launch count").group(1))
    # every scan( call is one scan_u64_kernel launch, whose own <<< sits in the scan lambda
    counted = body.count("<<<") - 1 + body.count("scan(")
    if counted != n:
        raise ValueError("sf_run's launches changed: restate them in the @filter plan model")
    for k in ("sf_check_kernel", "sf_eval_kernel", "cc_filter_kernel", "cc_page_kernel", "cc_compact_kernel",
              "sf_mark_kernel", "sf_out_kernel"):
        _one(k + "<<<", body, f"sf_run's {k}")
    for fn, empty in (("dgx_sg_filter", "n0 == 0"), ("dgx_dev_sg_filter", "d0_cap == 0")):
        _one(r"(?s)extern \"C\" int %s\(.*?if \(%s\) \{" % (fn, re.escape(empty)), api, f"{fn}'s empty call")
    lim = {k: int(_one(r"#define DGX_SGF_%s (\d+)" % k, hdr, f"DGX_SGF_{k}").group(1))
           for k in ("MAX_NODES", "MAX_LEAVES", "MAX_DEPTH")}
    return {"LAUNCHES": n, **lim}


K = read_constants()


def launches(d0_slots: int) -> int:
    """Kernel launches of one call: none when D0 has no slot (n0 in the host form, d0_cap in the device form), else a
    constant: rows, values, leaves and tree size do not enter."""
    return 0 if d0_slots == 0 else K["LAUNCHES"]
