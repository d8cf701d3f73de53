"""The launch plan of dgx_var_order / dgx_dev_var_order (dgx_api.cu vo_run) restated in Python.  The statements it
restates are matched as text in the CUDA sources, so a rewrite fails loudly here instead of drifting.
"""
from __future__ import annotations

import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")


def _src(path):
    with open(path) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the order-by-variable plan model (tests/var_order_plan.py)")
    return m


def read_constants(api: str | None = None, kern: str | None = None) -> dict:
    """{"FIXED": launches besides the radix passes, "KEY_PASSES": passes of the order-key sort, "DIGIT_BITS",
    "CTA_MIN": the longest tier-2 row a single thread sorts, "MAX_INSERTION"}."""
    api = _src(os.path.join(CSRC, "dgx_api.cu")) if api is None else api
    kern = _src(os.path.join(CSRC, "var_order_kernel.cuh")) if kern is None else kern
    body = _one(r"(?s)static int vo_run\(.*?\n\}\n", api, "vo_run").group(0)
    counted = [int(x) for x in re.findall(r"count_launches\(l, (\d+)\);", body)]
    if len(counted) != 2:
        raise ValueError("vo_run's launch counts changed: restate them in the order-by-variable plan model")
    # every scan( call is one scan_u64_kernel launch, whose own <<< sits in the scan lambda; the two gb_sort calls
    # count their own passes
    direct = body.count("<<<") - 1 + body.count("scan(P.")
    if direct != sum(counted):
        raise ValueError("vo_run's launches changed: restate them in the order-by-variable plan model")
    for k in ("vo_check_kernel", "vo_gather_kernel", "vo_compact_kernel", "vo_rowkey_kernel", "vo_tier_kernel",
              "vo_rows_kernel", "vo_cta_kernel", "vo_write_kernel", "vo_dest_kernel"):
        _one(k + "<<<", body, f"vo_run's {k}")
    if body.count("gb_sort(") != 2:
        raise ValueError("vo_run's radix sorts changed: restate them in the order-by-variable plan model")
    _one(r"gb_sort\(l, tiles, P\.bad, P\.words \+ VO_W_H, ek, ep, P\.words \+ VO_W_W, VO_KEY_PASSES,", body,
         "the order-key sort")
    _one(r"gb_sort\(l, tiles, P\.bad, P\.words \+ VO_W_H, rk, rp, P\.words \+ VO_W_W, pr,", body, "the row sort")
    _one(r"return \(gb_bits\(nrows \? nrows - 1 : 0\) \+ GB_DIGIT_BITS - 1\) / GB_DIGIT_BITS;", api,
         "vo_row_passes")
    for fn in ("dgx_var_order", "dgx_dev_var_order"):
        _one(r"(?s)extern \"C\" int %s\(.*?if \(ndest == 0 \|\| nrows == 0\) \{" % fn, api, f"{fn}'s empty call")
    c = {k: int(_one(r"constexpr \w+ VO_%s = (\d+);" % k, kern, f"VO_{k}").group(1))
         for k in ("KEY_PASSES", "CTA_MIN", "MAX_INSERTION")}
    gb = _src(os.path.join(CSRC, "groupby_kernel.cuh"))
    digit = int(_one(r"GB_DIGIT_BITS = (\d+)", gb, "GB_DIGIT_BITS").group(1))
    return {"FIXED": sum(counted), "DIGIT_BITS": digit, **c}


K = read_constants()


def row_passes(nrows: int) -> int:
    b = (nrows - 1).bit_length() if nrows > 1 else 0
    return (b + K["DIGIT_BITS"] - 1) // K["DIGIT_BITS"]


def launches(ndest: int, nrows: int) -> int:
    """Kernel launches of one call: none without a dest value or a row (ndest is the dest room in the device form),
    else the fixed kernels and 3 per radix pass: KEY_PASSES for the order key and row_passes(nrows) for the row.  The
    values, ties, map size and the rows' tiers do not enter."""
    if ndest == 0 or nrows == 0:
        return 0
    return K["FIXED"] + 3 * (K["KEY_PASSES"] + row_passes(nrows))
