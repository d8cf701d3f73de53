"""Generates tests/golden/pred_order_common.json.  Run in the authoring container only (reads the reference's tests,
which do not exist on the GPU box):

    python tests/golden/make_pred_order_golden.py

The fixture holds the published answers of the reference's query tests that order one node by one predicate, copied,
never computed here, with the query/common_test.go triples they read.  It scans every query*_test.go for two shapes:
  - a child block `friend(orderasc|orderdesc: P[, first: n][, offset: n])` of `me(func: uid(0x01))`, with no filter,
    facets or language on it: the row is uid 1's friend edges;
  - a root `me(func: anyofterms(name, "..."), orderasc|orderdesc: P[, first / offset])`: the row is the uids whose name
    holds one of the terms.
A case is kept only when P is a scalar int, float, datetime or string predicate, every uid of the row has one value of
P and no two values are equal.  There Go's indexed and unindexed sorts agree, so the published answer is also
sortWithoutIndex's.  count is the node's first, or 1000 where the query sets none (the query layer's default
before processSort).  Each answer is kept as the published JSON and as its uids: the row uid whose triples hold every
field the test prints.  The script prints how many tests it scanned, how many matched a shape and how many qualify.
"""
import json
import os
import re

REF = "/root/reference"
QDIR = os.path.join(REF, "query")
common = open(os.path.join(QDIR, "common_test.go")).read()
TYPES = {"int": "int", "float": "float", "datetime": "datetime", "string": "string"}


def schema_type(p, sortable=True):
    """The predicate's type; for a sort key (sortable) None when it is absent, a list or language-tagged."""
    m = re.search(r"^%s\s*:\s*(\[?)(\w+)([^\n]*)" % re.escape(p), common, re.M)
    if not m or (sortable and (m.group(1) or "@lang" in m.group(3))):
        return None
    return TYPES.get(m.group(2).lower())


def triples(p):
    return [(int(u), v) for u, v in re.findall(r'^\s*<(\d+)> <%s> "([^"]*)" \.' % re.escape(p), common, re.M)]


def same(t, field_val, triple_val):
    if t in ("int", "float"):
        return float(field_val) == float(triple_val)
    if t == "datetime":
        return str(field_val).startswith(triple_val)
    return field_val == triple_val


def key(t, v):
    return float(v) if t in ("int", "float") else v  # datetimes as ISO dates order as strings


def uids_of(items, row):
    out = []
    for it in items:
        hit = [u for u in row if all(schema_type(k, False) and any(x == u and same(schema_type(k, False), val, tv)
                                                              for x, tv in triples(k)) for k, val in it.items())]
        assert len(hit) == 1, (it, hit)
        out.append(hit[0])
    return out


CHILD = re.compile(r"me\(func:\s*uid\(0x0?1\)\)\s*\{[^{}]*?friend\((orderasc|orderdesc):\s*(\w+)\s*"
                   r"((?:,\s*(?:first|offset):\s*-?\d+\s*)*)\)\s*\{([^{}]*)\}")
ROOT = re.compile(r"me\(func:\s*anyofterms\(name,\s*\"([^\"]*)\"\),\s*(orderasc|orderdesc):\s*(\w+)\s*"
                  r"((?:,\s*(?:first|offset):\s*-?\d+\s*)*)\)\s*\{([^{}]*)\}")
friends = [int(v) for v in re.findall(r"^\s*<1> <friend> <(\d+)> \.", common, re.M)]
names = triples("name")

scanned, matched, cases = 0, 0, []
for fn in sorted(f for f in os.listdir(QDIR) if re.match(r"query\d*_test\.go$", f)):
    src = open(os.path.join(QDIR, fn)).read()
    for m in re.finditer(r"^func (Test\w+)\(t \*testing\.T\) \{\n(.*?)^\}\n", src, re.M | re.S):
        scanned += 1
        name, body = m.group(1), m.group(2)
        strs = re.findall(r"`([^`]*)`", body)
        for i, q in enumerate(strs):
            c, r = CHILD.search(q), ROOT.search(q)
            if not (c or r) or q.count("order") != 1 or "@" in q:
                continue
            res = next((s for s in strs[i + 1:] if '"data"' in s), None)
            if res is None:
                continue
            if c:
                order, pred, page, row = c.group(1), c.group(2), c.group(3), sorted(friends)
            else:
                terms = r.group(1).lower().split()
                row = sorted({u for u, v in names if set(v.lower().split()) & set(terms)})
                order, pred, page = r.group(2), r.group(3), r.group(4)
            matched += 1
            t = schema_type(pred)
            vals = {}
            for u, v in triples(pred):
                vals.setdefault(u, []).append(v)
            ok = t is not None and all(len(vals.get(u, [])) == 1 for u in row) and \
                len({key(t, vals[u][0]) for u in row}) == len(row)
            if not ok:
                continue
            first = re.search(r"first:\s*(-?\d+)", page)
            offset = re.search(r"offset:\s*(-?\d+)", page)
            data = json.loads(res)["data"]["me"]
            items = data[0].get("friend", []) if c else data
            cases.append({"test": name, "query": " ".join(q.split()), "pred": pred, "type": t,
                          "desc": order == "orderdesc", "row": row,
                          "count": int(first.group(1)) if first else 1000, "offset": int(offset.group(1)) if offset else 0,
                          "values": {str(u): vals[u][0] for u in row}, "published": " ".join(res.split()),
                          "want": uids_of(items, row)})
print(f"scanned {scanned} tests, {matched} queries of the two shapes, {len(cases)} qualify: "
      + ", ".join(sorted({c['test'] for c in cases})))
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "pred_order_common.json"), "w") as f:
    json.dump({"cases": cases}, f, indent=1)
    f.write("\n")
