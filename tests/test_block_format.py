"""The UidPack block format is read in one place: decode_kernel.cuh's helpers (gv_walk_block, warp_mbar_init,
warp_window_load, warp_tag_walk, expand_block) serve every kernel that reads a pack.  A second copy of the
group-varint walk or of the warp's block expansion would have to be fixed separately whenever the format handling
changes (a corrupt tag's clamp, the 64-bit running sum), so these checks keep such copies from coming back."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")


def sources():
    for p in sorted(glob.glob(os.path.join(CSRC, "*"))):
        if p.endswith((".cu", ".cuh", ".hpp", ".h")):
            yield os.path.basename(p), open(p).read()


def count(pattern):
    return {name: len(re.findall(pattern, src)) for name, src in sources() if re.search(pattern, src)}


def test_group_varint_value_assembled_once():
    # `v |= (u32)d[k] << (8 * k)`: one little-endian value of 1..4 bytes, whatever the loop variable is called
    assert count(r"\bd\[(\w+)\]\s*<<\s*\(\s*8\s*\*\s*\1\s*\)") == {"decode_kernel.cuh": 1}


def test_block_expansion_once():
    assert count(r"__funnelshift_r\(\s*w0\s*,\s*w1\b") == {"decode_kernel.cuh": 1}


def test_warp_mbarrier_set_up_in_one_helper():
    calls = {}
    for name, src in sources():
        src = re.sub(r"\bvoid\s+mbar_init\s*\(", "", src)  # the definition
        helper = re.search(r"\bvoid\s+warp_mbar_init\s*\(.*?\n}\n", src, flags=re.S)
        if helper:
            assert re.search(r"\bmbar_init\s*\(", helper.group(0)), "warp_mbar_init no longer sets up the barrier"
            src = src.replace(helper.group(0), "")
        n = len(re.findall(r"\bmbar_init\s*\(", src))
        if n:
            calls[name] = n
    assert set(calls) == {"filter_pipe.cuh"}, calls
