"""Every environment variable libdgx reads is documented in INTEGRATION.md section 4, and every one documented there is
read: a knob that nothing reads tells an operator they can tune what cannot be tuned.  The library also has one build
configuration plus the instrumented `make prof` build, so no other DGX_* macro selects code."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")


def sources():
    for p in sorted(glob.glob(os.path.join(CSRC, "*"))):
        if p.endswith((".cu", ".cuh", ".hpp", ".h")):
            yield p, open(p).read()


def documented_knobs():
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = re.search(r"^## 4\..*?(?=^## )", doc, flags=re.S | re.M)
    assert sec, "INTEGRATION.md has no section 4"
    return set(re.findall(r"^\| `(DGX_[A-Z0-9_]+)", sec.group(0), flags=re.M))


def test_documented_knobs_are_the_ones_read():
    read = {n for _, src in sources() for n in re.findall(r'getenv\(\s*"(DGX_[A-Z0-9_]+)"', src)}
    assert read, "no getenv found under dgraph_b200/csrc"
    assert documented_knobs() == read


def test_only_profiling_macro_selects_code():
    tested = set()
    for path, src in sources():
        for expr in re.findall(r"^\s*#\s*(?:if|ifdef|ifndef|elif)\b(.*)$", src, flags=re.M):
            tested |= set(re.findall(r"\bDGX_[A-Z0-9_]+", expr))
    assert tested == {"DGX_PIPE_PROF"}
