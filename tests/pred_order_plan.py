"""Launch plan of orderasc / orderdesc by a predicate (dgx_pred_order, dgx_api.cu po_run): the launches before the
key sort, the key sort's passes, the row sort's passes and the launches after, set by the column type and nrows alone.
"""
from __future__ import annotations

from dgraph_b200 import algo

K = {"FRONT": 6,          # fz_lookup, po_check, po_gather, 2 scans, po_compact
     "KEY_PASSES": 8,     # the 64-bit key (int64, float64, string prefix; a datetime's seconds)
     "NS_PASSES": 4,      # a datetime's nanoseconds, then one re-key launch
     "BACK": 8,           # po_rekey (rows), po_tier, po_rows, vo_cta, scan, po_write, scan, vo_dest
     "DIGIT_BITS": 8}


def row_passes(nrows: int) -> int:
    """P_r = ceil(bits(nrows - 1) / 8)."""
    b = max(nrows - 1, 0).bit_length()
    return (b + K["DIGIT_BITS"] - 1) // K["DIGIT_BITS"]


def launches(typ: int, nrows: int) -> int:
    """Kernel launches of one call with nrows > 0 and dest not empty."""
    key = 3 * K["KEY_PASSES"] + (3 * K["NS_PASSES"] + 1 if typ == algo.VAL_DATETIME else 0)
    return K["FRONT"] + key + K["BACK"] + 3 * row_passes(nrows)
