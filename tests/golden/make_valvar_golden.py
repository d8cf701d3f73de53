"""Generates tests/golden/valvar_common.json.  Run in the authoring container only (reads the reference's query
tests, which do not exist on the GPU box):

    python tests/golden/make_valvar_golden.py

The fixture holds the triples of query/common_test.go that the value-variable tests read -- the `path` edges with
their `weight` facets, `friend`, `follow`, `age` and `name` -- and the answers the reference's tests publish for
TestLevelBasedFacetVarAggSum, TestLevelBasedFacetVarSum, TestLevelBasedSumMix1, TestLevelBasedFacetVarSum1,
TestLevelBasedFacetVarSum2, TestQueryVarValAggMinMax, TestQueryVarValAggNestedFunc (min / max), TestMultiLevelAgg and
TestMultiLevelAgg1, as uid -> value.  The answers are copied from the tests' expected JSON, never computed here.
"""
import json
import os
import re

REF = "/root/reference/query"
src = open(os.path.join(REF, "common_test.go")).read()

edges = {p: [] for p in ("path", "friend", "follow")}
for f, p, t, facets in re.findall(r"<(\d+)> <(path|friend|follow)> <(\d+)>\s*(\([^)]*\))?\s*\.", src):
    w = re.search(r"\bweight = ([0-9.]+)", facets or "")
    edges[p].append([int(f), int(t)] + ([float(w.group(1))] if p == "path" and w else [None] if p == "path" else []))
ages = {int(u): int(a) for u, a in re.findall(r'<(\d+)> <age> "(\d+)" \.', src)}
names = {int(u): n for u, n in re.findall(r'<(\d+)> <name> "([^"]*)" \.', src)}

# The published answers (uid -> value), from the expected JSON of each test.
want = {
    "TestLevelBasedFacetVarAggSum": {"sumw": {"1000": 0.7999999999999999}},
    "TestLevelBasedFacetVarSum": {"L4": {"1003": 3.9, "1002": 1.2000000000000002}},
    "TestLevelBasedSumMix1": {"L2": {"24": 38.2, "31": 38.1}},
    "TestLevelBasedFacetVarSum1": {"L3": {"1003": 2.9, "1002": 0.2}},
    "TestLevelBasedFacetVarSum2": {"L4": {"1001": 2.9, "1003": 0.8}},
    "TestQueryVarValAggMinMax": {"n": {"23": 38, "1": 15, "31": 15}, "s": {"23": 38, "1": 19, "31": 15}},
    "TestQueryVarValAggNestedFunc": {"n": {"31": 15, "1": 15, "23": 38}, "s": {"31": 15, "1": 19, "23": 38}},
    "TestMultiLevelAgg": {"sum(val(s))": {"1": 2, "23": 5, "31": 0}},
    "TestMultiLevelAgg1": {"ss": {"31": 0, "1": 2, "23": 5}},
}
# anyofterms(name, "Michonne Andrea Rick") and its lower-case form match these uids
terms = {"michonne", "andrea", "rick"}
matched = sorted(u for u, n in names.items() if terms & set(n.lower().split()))
out = {"source": "query/common_test.go triples and the expected JSON of the tests named in `want`",
       "edges": edges, "age": {str(u): a for u, a in sorted(ages.items())},
       "anyofterms_michonne_andrea_rick": matched, "want": want}
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "valvar_common.json"), "w") as f:
    json.dump(out, f, indent=1)
print("valvar_common.json:", {p: len(e) for p, e in edges.items()}, "ages", len(ages), "matched", matched)
