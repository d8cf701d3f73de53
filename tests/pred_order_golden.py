"""The published answers of tests/golden/pred_order_common.json as calls: each case's column, built from the
query/common_test.go values the fixture copied, and its (col, desc, dest, rows, count, offset)."""
from __future__ import annotations

import datetime as dt
import json
import os

import numpy as np

from dgraph_b200 import algo

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pred_order_common.json")
TYPE = {"int": algo.VAL_INT64, "float": algo.VAL_FLOAT64, "datetime": algo.VAL_DATETIME, "string": algo.VAL_STRING}


def _value(t, s):
    if t == "int":
        return int(s)
    if t == "float":
        return float(s)
    if t == "datetime":  # the fixture's dates are UTC days
        d = dt.datetime.fromisoformat(s).replace(tzinfo=dt.timezone.utc)
        return (int(d.timestamp()), 0)
    return s.encode()


def cases():
    """[(label, case, want uids)]."""
    with open(PATH) as f:
        fx = json.load(f)
    out = []
    for c in fx["cases"]:
        row = np.asarray(c["row"], np.uint64)
        col = algo.ValColumn(TYPE[c["type"]], row, [[_value(c["type"], c["values"][str(int(u))])] for u in row])
        case = (col, c["desc"], row, [row], c["count"], c["offset"])
        out.append((c["test"], case, np.asarray(c["want"], np.uint64)))
    return out
