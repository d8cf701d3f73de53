"""Generates tests/golden/var_order_common.json.  Run in the authoring container only (reads the reference's query
tests, which do not exist on the GPU box):

    python tests/golden/make_var_order_golden.py

The fixture holds, for each reference test that orders a root by an int value variable, the root's DestUIDs and uid
matrix, the variable's map and the published order:
  TestMultiCountSort            f as var(anyofterms(name, "michonne rick andrea")) { n as count(friend) },
                                orderasc: val(n): a tie at count 1, kept in uid order
  TestQueryVarValAggMinMax      sum as math(n + s) of min / max of the friends' ages, orderdesc: val(sum)
  TestQueryVarValAggMinMaxSelf  sum as math(n + a + s), orderasc: val(sum)
  TestQueryVarValAggMul         mul as math(n * s) over uid 1's friends, orderdesc: val(mul): a three-way tie at 0
  TestMultiLevelAgg1            ss as sum(val(s)), uid(ss), orderasc: val(ss)
  TestUseVariableBeforeDefinitionError  orderasc: val(avgAge) before avgAge is defined: Go's nil-map error
Uids, names and the friend edges come from query/common_test.go.  The map of TestMultiCountSort is count(friend) from
the edges (the answer publishes the same counts); the other maps are the val() columns of the published answers (val(n)
+ val(s) for TestQueryVarValAggMinMax), keyed by the names' uids, the unnamed entry of uid 1's friends being 101.  The
expected order is the answer's names, never computed here.
"""
import json
import os
import re

REF = "/root/reference/query"
src = open(os.path.join(REF, "common_test.go")).read()
friend = [(int(f), int(t)) for f, t in re.findall(r"<(\d+)> <friend> <(\d+)>\s*\.", src)]
names = {int(u): n for u, n in re.findall(r'<(\d+)> <name> "([^"\\]*)" \.', src)}
uid_of = {}
for u, n in sorted(names.items()):
    uid_of.setdefault(n, u)


def term_row(query):
    words = set(query.lower().split())
    return sorted(u for u, n in names.items() if words & set(n.lower().split()))


def test_src(name):
    for f in ("query0_test.go", "query1_test.go", "query3_test.go"):
        s = open(os.path.join(REF, f)).read()
        m = re.search(r"func %s\(t \*testing\.T\) \{(.*?)\n\}\n" % name, s, re.S)
        if m:
            return m.group(1)
    raise KeyError(name)


def answer(name):
    return json.loads(re.search(r"`(\{\"data\".*?)`", test_src(name), re.S).group(1))["data"]


friends_of_1 = sorted(t for f, t in friend if f == 1)
cases = []


def add(label, desc, dest, keys, vals, order, rows=None):
    dest = sorted(dest)
    cases.append({"label": label, "desc": desc, "dest": dest, "rows": rows or [dest], "keys": keys, "vals": vals,
                  "count": 0, "offset": 0, "want_rows": [order], "want_dest": sorted(order)})


# TestMultiCountSort
f = term_row("michonne rick andrea")
cnt = {u: sum(1 for a, _ in friend if a == u) for u in f}
ans = answer("TestMultiCountSort")["countorder"]
assert [cnt[uid_of[e["name"]]] for e in ans] == [e["count(friend)"] for e in ans]
add("TestMultiCountSort", False, f, f, [cnt[u] for u in f], [uid_of[e["name"]] for e in ans])

# TestQueryVarValAggMinMax / TestQueryVarValAggMinMaxSelf
f = term_row("Michonne Andrea Rick")
ans = answer("TestQueryVarValAggMinMax")["me"]
m = {uid_of[e["name"]]: e["val(n)"] + e["val(s)"] for e in ans}
add("TestQueryVarValAggMinMax", True, f, sorted(m), [m[u] for u in sorted(m)], [uid_of[e["name"]] for e in ans])
ans = answer("TestQueryVarValAggMinMaxSelf")["me"]
m = {uid_of[e["name"]]: e["val(sum)"] for e in ans}
add("TestQueryVarValAggMinMaxSelf", False, f, sorted(m), [m[u] for u in sorted(m)], [uid_of[e["name"]] for e in ans])

# TestQueryVarValAggMul: the unnamed friend of uid 1 is the one uid without a name
ans = answer("TestQueryVarValAggMul")["me"]
unnamed = [u for u in friends_of_1 if u not in names]
assert len(unnamed) == 1
order = [uid_of[e["name"]] if "name" in e else unnamed[0] for e in ans]
m = dict(zip(order, [e["val(mul)"] for e in ans]))
add("TestQueryVarValAggMul", True, friends_of_1, sorted(m), [m[u] for u in sorted(m)], order)

# TestMultiLevelAgg1: the root is uid(ss)
ans = answer("TestMultiLevelAgg1")["sumorder"]
m = {uid_of[e["name"]]: e["val(ss)"] for e in ans}
add("TestMultiLevelAgg1", False, sorted(m), sorted(m), [m[u] for u in sorted(m)], [uid_of[e["name"]] for e in ans])

# TestUseVariableBeforeDefinitionError
assert "used before definition" in test_src("TestUseVariableBeforeDefinitionError")
d = term_row("Michonne Daryl Andrea")
cases.append({"label": "TestUseVariableBeforeDefinitionError", "desc": False, "dest": d, "rows": [d], "keys": None,
              "vals": None, "count": 0, "offset": 0, "error": "used before definition"})

out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "var_order_common.json")
with open(out, "w") as fh:
    json.dump({"source": "query/common_test.go and query/query{0,1,3}_test.go", "cases": cases}, fh, indent=1)
    fh.write("\n")
print(out, len(cases))
