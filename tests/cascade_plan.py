"""The launch plan of dgx_cascade / dgx_dev_cascade (dgx_api.cu cc_run) restated in Python.  The statements it restates
are matched as text in the CUDA sources, so a rewrite fails loudly here instead of drifting.
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
        raise ValueError(f"{what} changed: restate it in the cascade plan model (tests/cascade_plan.py)")
    return m


def read_constants(api: str | None = None) -> dict:
    """{"A": launches once a call, "B": launches a level with work, "MAX_DEPTH": levels}."""
    api = _src("dgx_api.cu") if api is None else api
    body = _one(r"(?s)static int cc_run\(.*?\n\}\n", api, "cc_run").group(0)
    m = _one(r"count_launches\(l, (\d+) \+ (\d+) \* \(int\)D\);", body, "cc_run's launch count")
    a, b = int(m.group(1)), int(m.group(2))
    loop = _one(r"(?s)for \(uint64_t i = 0; i < D; \+\+i\) \{(\n        CcLevel L = .*?)\n    \}\n", body,
                "the level loop").group(1)
    per_level = loop.count("<<<") + loop.count("scan(")
    # every scan( call is one scan_u64_kernel launch, whose own <<< sits in the scan lambda
    once = body.count("<<<") - 1 - loop.count("<<<") + body.count("scan(") - loop.count("scan(")
    if per_level != b or once != a:
        raise ValueError("cc_run's launches changed: restate them in the cascade plan model")
    depth = int(_one(r"constexpr uint32_t kCcMaxDepth = (\d+);", api, "the depth limit").group(1))
    for fn in ("dgx_cascade", "dgx_dev_cascade"):
        _one(r"(?s)extern \"C\" int %s\(.*?if \((T\.level\.empty\(\)|m == 0 && nd == 0)\) \{" % fn, api,
             f"{fn}'s empty call")
    return {"A": a, "B": b, "MAX_DEPTH": depth}


K = read_constants()


def launches(levels_with_work: int) -> int:
    """Kernel launches of one call: none without a level holding a dest value or a value slot, else A + B per such
    level.  Node, row and value counts do not enter."""
    return 0 if levels_with_work == 0 else K["A"] + K["B"] * levels_with_work
