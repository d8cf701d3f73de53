"""Generates tests/golden/match_common.json.  Run in the authoring container only (reads the reference's tests, which
do not exist on the GPU box):

    python tests/golden/make_match_golden.py

The fixture holds the published answers of the reference's match() tests, copied, never computed here:
  TestDistance (worker/match_test.go)        ten levenshteinDistance results
  TestMatchFuncWithAfterWithValidUid         match(name, Ali, 5), after: 0x2710 -> 0x2712, 0x2714
  TestMatchFuncWithAfterWithLastUid          match(name, Ali, 5), after: 0x2714 -> nothing
  TestMatchingWithPagination (match case)    match(tweet-d, "aaaaaa", 3), first: 1 -> the uid whose tweet-d is "aaabcd"
and the untagged `name` and `tweet-d` triples of query/common_test.go those queries read, as (uid, value bytes in hex).
The trigram rows are built from the triples by the tests (byte trigrams, tok.TrigramTokenizer).
Left out: `has(name) @filter(match(name, "", 8))` (count 39).  has(name) and the untagged values it reads are those of
the shared test cluster after the other query tests' mutations, which common_test.go alone does not state.
"""
import json
import os
import re

REF = "/root/reference"
src = open(os.path.join(REF, "query", "common_test.go")).read()


def unquote(s: str) -> bytes:
    return json.loads('"' + s + '"').encode()


def triples(pred):
    out = {}
    for u, v in re.findall(r'<(\d+)> <' + re.escape(pred) + r'> "((?:[^"\\]|\\.)*)" \.', src):
        out.setdefault(int(u), unquote(v))  # untagged only: a tagged triple has @lang before the dot
    return sorted(out.items())


dist_src = open(os.path.join(REF, "worker", "match_test.go")).read()
distance = [[a, b, int(d)] for d, a, b in re.findall(r'require.Equal\(t, (\d+), levenshteinDistance\("([^"]*)", "([^"]*)"\)\)',
                                                     dist_src)]
assert len(distance) == 10

q1 = open(os.path.join(REF, "query", "query1_test.go")).read()
assert '"uid": "0x2712"}, {"name": "Alice", "uid": "0x2714"}' in q1 and 'match(name, Ali, 5), after: 0x2714' in q1
q0 = open(os.path.join(REF, "query", "query0_test.go")).read()
assert 'match(tweet-d, "aaaaaa", 3), first:1' in q0 and '{"tweet-d":"aaabcd"}' in q0
tweet_d = triples("tweet-d")
aaabcd = [u for u, v in tweet_d if v == b"aaabcd"]
assert len(aaabcd) == 1

fixture = {
    "distance": distance,
    "triples": {p: [[u, v.hex()] for u, v in triples(p)] for p in ("name", "tweet-d")},
    "cases": [
        {"test": "TestMatchFuncWithAfterWithValidUid", "pred": "name", "query": "Ali", "max": 5, "after": 0x2710,
         "first": 0, "want": [0x2712, 0x2714]},
        {"test": "TestMatchFuncWithAfterWithLastUid", "pred": "name", "query": "Ali", "max": 5, "after": 0x2714,
         "first": 0, "want": []},
        {"test": "TestMatchingWithPagination", "pred": "tweet-d", "query": "aaaaaa", "max": 3, "after": 0,
         "first": 1, "want": aaabcd},
    ],
}
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "match_common.json"), "w") as f:
    json.dump(fixture, f, indent=1)
    f.write("\n")
