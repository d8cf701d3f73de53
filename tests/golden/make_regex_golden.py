"""Generates tests/golden/regex_common.json.  Run in the authoring container only (reads the reference's tests, which
do not exist on the GPU box):

    python tests/golden/make_regex_golden.py

The fixture holds the published answers of the reference's regexp() value tests, copied, never computed here:
TestFilterRegex6 to TestFilterRegex13 (query/query3_test.go), each `pattern @filter(regexp(value, /.../))` under
uid(0x1234), over the 24 `value` strings common_test.go gives the `pattern` children 0x2000, 0x2001, ... in order.
The filter's UidList is those 24 uids; each answer is kept as the values the test prints, mapped to their uids.
Left out:
  - TestFilterRegex1-5 and the `regexp(dob ...)` case (`friend @filter(regexp(...))`): their candidates are friend
    edges and values other query tests mutate in the shared cluster;
  - TestFilterRegex14 (`/pattern/x`) and the empty-pattern case: errors raised before any value is tested;
  - the `name@ru` cases (TestFilterRegex15/16): language-tagged values, which this fixture's untagged column does not hold;
  - the `has(...)` and `regexp(name, ...)` root-function cases (TestRegexInFilterNoDataOnRoot,
    TestRegexInFilterIndexedPredOnRoot, TestMultiRegexInFilter*, TestRegexFuncWithAfter) and query4's `King*` cases:
    their candidates depend on other tests' mutations of `name`, `full_name`, `firstName` and `make`.
"""
import json
import os
import re

REF = "/root/reference"
common = open(os.path.join(REF, "query", "common_test.go")).read()
m = re.search(r'patterns := \[\]string\{(.*?)\}', common, re.S)
values = re.findall(r'"([^"]*)"', m.group(1))
assert len(values) == 24 and 'nextId := uint64(0x2000)' in common
uid_of = {v: 0x2000 + i for i, v in enumerate(values)}

q3 = open(os.path.join(REF, "query", "query3_test.go")).read()
cases = []
for n in range(6, 14):
    body = q3[q3.index(f"func TestFilterRegex{n}(t *testing.T)"):]
    body = body[:body.index("\n}\n")]
    pm = re.search(r'regexp\(value, /(.*)/(i?)\)\)', body)
    want = re.findall(r'\{"value":\s*"([^"]*)"\}', body)
    if n == 13:
        assert '{"data": {"me": []}}' in body
    cases.append({"test": f"TestFilterRegex{n}", "pattern": pm.group(1), "fold": pm.group(2) == "i",
                  "want": sorted(uid_of[v] for v in want)})
assert [len(c["want"]) for c in cases] == [2, 2, 3, 3, 2, 2, 2, 0]

fixture = {"value": [[uid_of[v], v] for v in values], "cases": cases}
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "regex_common.json"), "w") as f:
    json.dump(fixture, f, indent=1)
    f.write("\n")
