"""The published compare-function answers of tests/golden/compare_common.json as calls: the columns built from the
copied triples, the arguments converted to the schema type, and for the index path the rows Go reads, built here with
the tokenizers' rules (float: int64(f); year: the value's UTC year) and getInequalityTokens' key walk (ge / gt:
the index keys from the argument's token up; le / lt: from it down; between: the keys between the two tokens; eq: one
row per argument's token).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import datetime as _dt
import json
import math
import os
import re

import numpy as np

from dgraph_b200 import algo

_HERE = os.path.dirname(os.path.abspath(__file__))
TYPES = {"int": algo.VAL_INT64, "float": algo.VAL_FLOAT64, "bool": algo.VAL_BOOL, "datetime": algo.VAL_DATETIME,
         "string": algo.VAL_STRING}
_EPOCH = _dt.datetime(1970, 1, 1, tzinfo=_dt.timezone.utc)


def load():
    with open(os.path.join(_HERE, "golden", "compare_common.json")) as f:
        return json.load(f)


def parse_time(s: str):
    """Go's datetime parsing of these literals: a year, a date, or an RFC 3339 time with its zone -> (sec, nsec)."""
    if re.fullmatch(r"\d{4}", s):
        s += "-01-01"
    if "T" not in s:
        s += "T00:00:00+00:00"
    d = _dt.datetime.fromisoformat(s.replace("Z", "+00:00"))
    delta = d - _EPOCH
    return delta.days * 86400 + delta.seconds, delta.microseconds * 1000


def parse(typ: str, s: str):
    if typ == "int":
        return int(s)
    if typ == "float":
        return float(s)
    if typ == "bool":
        return s == "true"
    if typ == "datetime":
        return parse_time(s)
    return s.encode()


def column(G, pred):
    """The predicate's ValColumn: every uid with a triple, its values in triple order."""
    typ = G["schema"][pred]
    vals = {}
    for u, v in G["triples"][pred]:
        vals.setdefault(u, []).append(parse(typ, v))
    uids = sorted(vals)
    return algo.ValColumn(TYPES[typ], uids, [vals[u] for u in uids]), uids, [vals[u] for u in uids]


def token(tokenizer, v):
    if tokenizer == "float":
        return int(math.trunc(v))
    return (_EPOCH + _dt.timedelta(seconds=v[0])).year


def value_case(G, c):
    col, _, _ = column(G, c["pred"])
    typ = G["schema"][c["pred"]]
    return col, c["op"], [parse(typ, a) for a in c["args"]], np.asarray(c["cands"], np.uint64)


def index_case(G, c):
    """(col, op, args, rows, row_arg) of handleCompareFunction for the case."""
    col, uids, values = column(G, c["pred"])
    typ = G["schema"][c["pred"]]
    args = [parse(typ, a) for a in c["args"]]
    tk = c["tokenizer"]
    index = {}
    for u, vs in zip(uids, values):
        for v in vs:
            index.setdefault(token(tk, v), set()).add(u)
    keys = sorted(index)
    ta = [token(tk, a) for a in args]
    op = c["op"]
    if op == "eq":
        sel = ta
    elif op in ("ge", "gt"):
        sel = [k for k in keys if k >= ta[0]]
    elif op in ("le", "lt"):
        sel = [k for k in reversed(keys) if k <= ta[0]]
    else:
        sel = [k for k in keys if ta[0] <= k <= ta[1]]
    rows = [np.asarray(sorted(index.get(k, ())), np.uint64) for k in sel]
    if op == "eq":
        ra = algo.CompareRowArgs("eq", len(rows), len(args))
    else:
        ra = algo.CompareRowArgs(op, len(rows), 1, bool(sel) and sel[0] == ta[0])
    return col, op, args, rows, ra


def merged(rows):
    return np.unique(np.concatenate(rows)).astype(np.uint64) if rows and sum(len(r) for r in rows) else \
        np.zeros(0, np.uint64)
