"""Generates tests/golden/compare_common.json.  Run in the authoring container only (reads the reference's tests, which
do not exist on the GPU box):

    python tests/golden/make_compare_golden.py

The fixture holds the published answers of the reference's compare-function tests, copied, never computed here, with
the query/common_test.go triples and schema types they read.  Each answer is kept as the published JSON and as its
uids: a `uid` field where the test prints one, otherwise the candidate whose triples hold every field the test prints.
  - TestFilterNonIndexedPredicate (query/query0_test.go): the 21 root cases over uid(1, 2, 3, 4), string, int,
    datetime, float and bool, on the value path.
  - TestEqFilterWithoutIndex and TestBetweenWithoutIndex's first case: @filter over type(CarModel), 0xc8-0xca.
  - TestBetweenFloat: the `salary` float index (rows 0 and last filtered) and the `average` float list.
  - TestDateTimeQuery's year-index cases: le(dob, ...) with and without a zone, and graduation (a list) between / eq /
    lt / gt at root.
Left out:
  - TestFilterNonIndexedPredicate's `friend @filter(ge(survival_rate, 1.6))`: its candidates are uid 1's friend edges,
    which other query tests mutate in the shared cluster;
  - TestBetweenWithoutIndex's `newfriend @filter(...)` case: its child rows are newfriend edges this fixture does not
    copy;
  - TestDateTimeQuery's created_at / updated_at cases: they order by the value (orderdesc) or read facets and
    `updated_at|modified_at` aliases, which is not the comparison these calls make, and its `gt(age, 15) @filter(...)`
    cases: their candidates come from the int index of `age`, which other tests mutate.
"""
import json
import os
import re

REF = "/root/reference"
common = open(os.path.join(REF, "query", "common_test.go")).read()
q0 = open(os.path.join(REF, "query", "query0_test.go")).read()

PREDS = {"noindex_name": "string", "noindex_age": "int", "noindex_dob": "datetime", "noindex_alive": "bool",
         "noindex_salary": "float", "year": "int", "make": "string", "model": "string", "salary": "float",
         "average": "float", "dob": "datetime", "graduation": "datetime"}
for p, t in PREDS.items():  # the schema types the tests read
    m = re.search(r"^%s\s*:\s*(\[?)(\w+)" % re.escape(p), common, re.M)
    assert m and m.group(2).lower() == t, (p, m and m.group(2))
triples = {p: [[int(u), v] for u, v in re.findall(r'^\s*<(\d+)> <%s> "([^"]*)" \.' % re.escape(p), common, re.M)]
           for p in PREDS}
assert triples["noindex_age"] == [[1, "21"], [2, "22"], [3, "23"], [4, "24"]]
assert sorted(u for u, _ in triples["graduation"]) == [1, 31, 31]

FN = re.compile(r"\b(eq|le|lt|ge|gt|between)\((\w+),\s*([^)]*)\)")


def body_of(name):
    b = q0[q0.index(f"func {name}(t *testing.T)"):]
    return b[:b.index("\nfunc ", 1)]


def same(pred, field_val, triple_val):
    t = PREDS[pred]
    if t in ("int", "float"):
        return float(field_val) == float(triple_val)
    if t == "datetime":
        return str(field_val).startswith(triple_val)
    if t == "bool":
        return field_val == (triple_val == "true")
    return field_val == triple_val


def uids_of(result, cands):
    items = next(iter(json.loads(result)["data"].values()))
    out = []
    for it in items:
        if "uid" in it:
            out.append(int(it["uid"], 16))
            continue
        hit = [c for c in cands if all(any(u == c and same(k, v, tv) for u, tv in triples[k]) for k, v in it.items())]
        assert len(hit) == 1, (it, hit)
        out.append(hit[0])
    return sorted(out)


def cases_of(name, path, cands, keep=lambda q: True):
    strs = re.findall(r"`([^`]*)`", body_of(name))
    res = []
    for i, q in enumerate(strs):
        m = FN.search(q)
        if not m or not keep(q):
            continue
        r = next(s for s in strs[i + 1:] if '"data"' in s)
        args = [a.strip().strip('"') for a in m.group(3).split(",")]
        res.append({"test": name, "query": " ".join(q.split()), "op": m.group(1), "pred": m.group(2), "args": args,
                    "path": path, "cands": cands, "published": " ".join(r.split()), "want": uids_of(r, cands or
                                                                                                       [u for u, _ in triples[m.group(2)]])})
    return res


cases = cases_of("TestFilterNonIndexedPredicate", "value", [1, 2, 3, 4], lambda q: "func: uid(1, 2, 3, 4)" in q)
assert len(cases) == 21
cases += cases_of("TestEqFilterWithoutIndex", "value", [200, 201, 202])
cases += cases_of("TestBetweenWithoutIndex", "value", [200, 201, 202], lambda q: "CarModel" in q)
cases += cases_of("TestBetweenFloat", "index", None)
cases += cases_of("TestDateTimeQuery", "index", None,
                  lambda q: re.search(r"func: (le|lt|gt|eq|between)\((dob|graduation),", q) is not None)
assert len(cases) == 21 + 1 + 1 + 5 + 8, len(cases)
for c in cases:
    if c["path"] == "index":
        c["tokenizer"] = "float" if PREDS[c["pred"]] == "float" else "year"

fixture = {"schema": {p: PREDS[p] for p in PREDS}, "list": ["average", "graduation"], "triples": triples,
           "cases": cases}
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "compare_common.json"), "w") as f:
    json.dump(fixture, f, indent=1)
    f.write("\n")
