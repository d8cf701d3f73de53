"""The published answers of the reference's order-by-value-variable tests (tests/golden/var_order_common.json, built by
tests/golden/make_var_order_golden.py) as cases for the restatement, the formula and both library forms."""
from __future__ import annotations

import json
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "var_order_common.json")


def cases():
    """[(label, (map, desc, dest, rows, count, offset), want)]: want is (rows, dest) or "nil" for Go's error."""
    with open(PATH) as fh:
        data = json.load(fh)
    out = []
    for c in data["cases"]:
        m = None if c["keys"] is None else (np.array(c["keys"], np.uint64), np.array(c["vals"], np.int64))
        case = (m, c["desc"], np.array(c["dest"], np.uint64), [np.array(r, np.uint64) for r in c["rows"]], c["count"],
                c["offset"])
        want = "nil" if "error" in c else (c["want_rows"], c["want_dest"])
        out.append((c["label"], case, want))
    return out


def check(got_rows, got_dest, want) -> bool:
    return [list(map(int, r)) for r in got_rows] == want[0] and list(map(int, got_dest)) == want[1]
