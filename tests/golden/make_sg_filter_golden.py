"""Generates tests/golden/sg_filter_common.json.  Run in the authoring container only (reads the reference's query
tests, which do not exist on the GPU box):

    python tests/golden/make_sg_filter_golden.py

The fixture holds the triples of query/common_test.go that the @filter tests read -- `name` (untagged values only),
`friend` and `school` -- the term rows their anyofterms() leaves and roots read, and the answers the reference's tests
publish for TestUidFunctionInFilter, TestUidFunctionInFilter2, TestUidFunctionInFilter4, TestUidInFunction,
TestUidInFunction1, TestUidInFunction2, TestCountAtRootWithAlias4, TestHasFuncAtRootFilter,
TestToFastJSONFilterOrFirst, TestToFastJSONFilterOrOffset and TestToFastJSONFilterOrCount.

Term rows: anyofterms(name, "a b") reads the `name` term index, whose tokens are the lower-cased words of each untagged
name (tok.TermTokenizer: unicode word split, lower case).  For the ASCII names these tests meet that is a whitespace
split and str.lower(); a row is every uid one of whose words is one of the query's words, ascending.

The answers are copied from the tests' expected JSON, never computed here: names in result order, a list of names per
parent row (empty where the JSON has no `friend` key), or the published count.
"""
import json
import os
import re

REF = "/root/reference/query"
src = open(os.path.join(REF, "common_test.go")).read()

edges = {p: [[int(f), int(t)] for f, t in re.findall(r"<(\d+)> <%s> <(\d+)>\s*\." % p, src)]
         for p in ("friend", "school")}
names = {int(u): n for u, n in re.findall(r'<(\d+)> <name> "([^"\\]*)" \.', src)}


def term_row(query):
    words = set(query.lower().split())
    return sorted(u for u, n in names.items() if words & set(n.lower().split()))


QUERIES = ["Michonne Andrea", "Michonne Rick Daryl", "Andrea", "Glenn SomethingElse", "Daryl", "Glenn Rhee",
           "Daryl Dixon", "Andrea Rhee"]

# The published answers, from the expected JSON of each test.
want = {
    "TestUidFunctionInFilter": {"names": ["Michonne", "Glenn Rhee"]},
    "TestUidFunctionInFilter2": {"rows": [["Rick Grimes"], ["Michonne"], [], [], []]},
    "TestUidFunctionInFilter4": {"names": ["Andrea With no friends"]},
    "TestUidInFunction": {"names": ["Michonne"]},
    "TestUidInFunction1": {"names": ["Michonne", "Glenn Rhee"]},
    "TestUidInFunction2": {"rows": [["Glenn Rhee", "Daryl Dixon"], ["Michonne"], []]},
    "TestCountAtRootWithAlias4": {"count": 2},
    "TestHasFuncAtRootFilter": {"names": ["Michonne", "Rick Grimes"]},
    "TestToFastJSONFilterOrFirst": {"rows": [["Glenn Rhee", "Daryl Dixon"]]},
    "TestToFastJSONFilterOrOffset": {"rows": [["Daryl Dixon", "Andrea"]]},
    "TestToFastJSONFilterOrCount": {"counts": [2], "rows": [["Andrea"]]},
}
out = {"source": "query/common_test.go triples and the expected JSON of the tests named in `want`",
       "terms": "anyofterms rows: uids whose untagged name, lower-cased and split on whitespace, shares a word with the "
                "query's words",
       "names": {str(u): n for u, n in sorted(names.items())}, "edges": edges,
       "anyofterms": {q: term_row(q) for q in QUERIES}, "want": want}
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "sg_filter_common.json"), "w") as f:
    json.dump(out, f, indent=1)
print("sg_filter_common.json:", {p: len(e) for p, e in edges.items()}, "names", len(names),
      {q: r for q, r in out["anyofterms"].items()})
