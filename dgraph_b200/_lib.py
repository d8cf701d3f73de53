"""ctypes loader for libdgx.so (the sm_90a CUDA library behind include/dgx.h).

There is deliberately NO fallback: if the shared library is missing or CUDA is
unavailable, every product entry point raises.  Build with `make` or
`python -c "import __graft_entry__ as g; g.build()"`.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("DGX_LIB") or os.path.join(_HERE, "libdgx.so")  # DGX_LIB: try an experimental build

DGX_OK = 0
DGX_ERR_ARG, DGX_ERR_CAP = -3, -4
STATUS_NAMES = {0: "DGX_OK", -1: "DGX_ERR_CUDA", -2: "DGX_ERR_OOM", -3: "DGX_ERR_ARG", -4: "DGX_ERR_CAP", -5: "DGX_ERR_NODEV"}
OP_INTERSECT, OP_DIFFERENCE = 0, 1


class DgxError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{STATUS_NAMES.get(code, code)}: {msg}")
        self.code = code


class PackView(C.Structure):
    """dgx_pack_view (include/dgx.h)."""
    _fields_ = [
        ("block_size", C.c_uint32),
        ("nblocks", C.c_size_t),
        ("base", C.c_void_p),
        ("num_uids", C.c_void_p),
        ("delta_off", C.c_void_p),
        ("deltas", C.c_void_p),
    ]


class PackRef(C.Structure):
    """dgx_pack_ref (include/dgx.h): a pack plus the (key, version) that names it in the HBM cache."""
    _fields_ = [("pack", C.POINTER(PackView)), ("key", C.c_uint64), ("version", C.c_uint64)]


class QueryTree(C.Structure):
    """dgx_query_tree (include/dgx.h): a cindex.Query tree as CSR arrays, node 0 the root."""
    _fields_ = [("nnodes", C.c_size_t), ("op", C.c_void_p), ("leaf_off", C.c_void_p), ("leaf_idx", C.c_void_p),
                ("sub_off", C.c_void_p), ("sub_idx", C.c_void_p)]


class CascadeTree(C.Structure):
    """dgx_cascade_tree (include/dgx.h): a forest of subgraph nodes in pre-order."""
    _fields_ = [("nnodes", C.c_size_t), ("parent", C.c_void_p), ("flags", C.c_void_p), ("first", C.c_void_p),
                ("offset", C.c_void_p), ("counts_len", C.c_void_p)]


class CascadeNode(C.Structure):
    """dgx_cascade_node (include/dgx.h): one node's device arrays for dgx_dev_cascade."""
    _fields_ = [("v", C.c_void_p), ("v_off", C.c_void_p), ("nrows", C.c_size_t), ("v_cap", C.c_size_t),
                ("dest", C.c_void_p), ("ndest", C.c_size_t), ("has_val", C.c_void_p), ("nhas", C.c_size_t)]


class PathLevel(C.Structure):
    """dgx_path_level (include/dgx.h): one shortest-path expansion level, nsg sgs in exec order as CSR arrays."""
    _fields_ = [("nsg", C.c_size_t), ("attr", C.c_void_p), ("src_off", C.c_void_p), ("src", C.c_void_p),
                ("v_off", C.c_void_p), ("v", C.c_void_p), ("dest_off", C.c_void_p), ("dest", C.c_void_p)]


class PathStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("edges", "discovered", "to_level")]


class VarLevel(C.Structure):
    """dgx_var_level (include/dgx.h): one node of a value variable's path, its SrcUIDs, uid matrix and DestUIDs."""
    _fields_ = [("src", C.c_void_p), ("v_off", C.c_void_p), ("v", C.c_void_p), ("dest", C.c_void_p),
                ("nrows", C.c_size_t), ("v_cap", C.c_size_t), ("ndest", C.c_size_t)]


class MathNode(C.Structure):
    """dgx_math_node (include/dgx.h): one node of a math() program in post-order."""
    _fields_ = [("op", C.c_uint8), ("const_tag", C.c_uint8), ("child", C.c_uint16 * 3), ("leaf", C.c_uint32),
                ("const_word", C.c_uint64)]


class MathLeaf(C.Structure):
    """dgx_math_leaf (include/dgx.h): one variable's map, per-entry tags or one type, and the nil bit."""
    _fields_ = [("key", C.c_void_p), ("word", C.c_void_p), ("tag", C.c_void_p), ("d_len", C.c_void_p),
                ("n", C.c_size_t), ("type", C.c_int), ("nil", C.c_int)]


class StrColumn(C.Structure):
    """dgx_str_column (include/dgx.h): a predicate's string values, uid i owning values val_off[i] .. val_off[i+1) and
    value j the bytes byte_off[j] .. byte_off[j+1)."""
    _fields_ = [("uid", C.c_void_p), ("val_off", C.c_void_p), ("byte_off", C.c_void_p), ("bytes", C.c_void_p),
                ("n", C.c_size_t), ("nvals", C.c_size_t), ("nbytes", C.c_size_t)]


class ValColumn(C.Structure):
    """dgx_val_column (include/dgx.h): a predicate's values converted to one type, uid i owning values val_off[i] ..
    val_off[i+1), as words (and nanoseconds) or, for DGX_VAL_STRING, a referenced StrColumn; an optional bad byte per
    value."""
    _fields_ = [("type", C.c_int), ("uid", C.c_void_p), ("val_off", C.c_void_p), ("word", C.c_void_p),
                ("nsec", C.c_void_p), ("bad", C.c_void_p), ("str", C.POINTER(StrColumn)), ("n", C.c_size_t),
                ("nvals", C.c_size_t)]


class ValArgs(C.Structure):
    """dgx_val_args (include/dgx.h): a compare function's arguments, words (and nanoseconds) or string byte ranges."""
    _fields_ = [("word", C.c_void_p), ("nsec", C.c_void_p), ("bytes", C.c_void_p), ("byte_off", C.c_void_p),
                ("n", C.c_size_t)]


class SgFilterTree(C.Structure):
    """dgx_sg_filter_tree (include/dgx.h): a subgraph's @filter tree, node 0 the root, parents below their children."""
    _fields_ = [("nnodes", C.c_size_t), ("op", C.c_void_p), ("parent", C.c_void_p), ("leaf", C.c_void_p)]


class SgFilterLeaf(C.Structure):
    """dgx_sg_filter_leaf (include/dgx.h): a LIST leaf's uids, or a COUNT leaf's counts / offsets and comparison."""
    _fields_ = [("kind", C.c_int), ("cmp", C.c_int), ("threshold", C.c_int64), ("uids", C.c_void_p), ("n", C.c_size_t),
                ("d_len", C.c_void_p), ("counts", C.c_void_p), ("off", C.c_void_p)]


class CacheStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("hits", "misses", "evictions", "bytes", "entries", "max_bytes")]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("calls", "uids_in", "uids_out", "h2d_bytes", "d2h_bytes", "kernel_launches")]


# every symbol include/dgx.h declares: name -> (restype, argtypes)
_vp, _sz, _u64, _int = C.c_void_p, C.c_size_t, C.c_uint64, C.c_int
_szp = C.POINTER(C.c_size_t)
SYMBOLS = {
    "dgx_init": (_int, [_int]),
    "dgx_shutdown": (None, []),
    "dgx_last_error": (C.c_char_p, []),
    "dgx_describe": (_int, [C.c_char_p, _sz]),
    "dgx_host_alloc": (_vp, [_sz]),
    "dgx_host_free": (None, [_vp]),
    "dgx_get_stats": (None, [C.POINTER(Stats)]),
    "dgx_intersect2": (_int, [_vp, _sz, _vp, _sz, _vp, _sz, _szp]),
    "dgx_intersect_sorted": (_int, [_vp, _vp, _sz, _vp, _sz, _szp]),
    "dgx_merge_sorted": (_int, [_vp, _vp, _sz, _vp, _sz, _szp]),
    "dgx_difference": (_int, [_vp, _sz, _vp, _sz, _vp, _sz, _szp]),
    "dgx_intersect_batch": (_int, [_vp, _vp, _vp, _vp, _sz, _vp, _vp, _sz]),
    "dgx_decode": (_int, [C.POINTER(PackView), _u64, _vp, _sz, _szp]),
    "dgx_decode_intersect_sorted": (_int, [C.POINTER(PackView), _u64, _vp, _vp, _sz, _vp, _sz, _szp]),
    "dgx_intersect_compressed": (_int, [C.POINTER(PackView), _u64, _vp, _sz, _vp, _sz, _szp]),
    "dgx_intersect_sorted_packed": (_int, [C.POINTER(PackRef), _sz, _vp, _sz, _szp]),
    "dgx_intersect_compressed_ref": (_int, [C.POINTER(PackRef), _u64, _vp, _sz, _vp, _sz, _szp]),
    "dgx_intersect_compressed_rows": (_int, [C.POINTER(PackRef), _sz, _u64, _vp, _sz, _vp, _vp, _sz]),
    "dgx_intersect_compressed_matrix": (_int, [C.POINTER(PackRef), _vp, _vp, _sz, _vp, _vp, _sz]),
    "dgx_merge_sorted_matrix": (_int, [_vp, _vp, _sz, _vp, _sz, _szp]),
    "dgx_list_uids_rows": (_int, [C.POINTER(PackRef), _vp, _sz, _vp, _vp, _vp, _u64, _vp, _sz, _vp, _vp, _sz]),
    "dgx_list_uids_unfiltered_rows": (_int, [C.POINTER(PackRef), _sz, _vp, _vp, _vp, _u64, C.c_int32, _vp, _vp, _sz]),
    "dgx_list_count_rows": (_int, [C.POINTER(PackRef), _sz, _vp, _vp, _vp, _u64, _vp]),
    "dgx_decode_to_buffer_rows": (_int, [C.POINTER(PackRef), _sz, _vp, _vp, _sz]),
    "dgx_encode_from_buffer_rows": (_int, [_vp, _vp, _sz, C.c_uint32, _vp, _sz, _vp, _vp, _vp]),
    "dgx_trigram_query": (_int, [C.POINTER(QueryTree), C.POINTER(PackRef), _sz, _vp, _vp, _vp, _vp, _vp, _sz, _u64, _vp, _sz, _szp]),
    "dgx_reach_create": (_int, [_vp, _vp, _sz, C.POINTER(_vp)]),
    "dgx_reach_destroy": (None, [_vp]),
    "dgx_reach_size": (_int, [_vp, _szp]),
    "dgx_reach_export": (_int, [_vp, _vp, _vp, _sz, _szp]),
    "dgx_recurse_filter": (_int, [_vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _sz, _szp]),
    "dgx_var_propagate": (_int, [_int, _vp, _vp, _sz, C.POINTER(VarLevel), _sz, _vp, _vp, _sz, _szp]),
    "dgx_var_level_agg": (_int, [_int, _int, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _vp, _vp, _sz, _szp]),
    "dgx_math_eval": (_int, [C.POINTER(MathNode), _sz, C.POINTER(MathLeaf), _sz, _vp, _sz, _vp, _vp, _vp, _sz, _vp]),
    "dgx_path_create": (_int, [_u64, _u64, C.POINTER(_vp)]),
    "dgx_path_destroy": (None, [_vp]),
    "dgx_path_expand": (_int, [_vp, C.POINTER(PathLevel), _vp, _vp, _sz, C.POINTER(PathStats)]),
    "dgx_path_result": (_int, [_vp, _vp, _vp, _sz, _szp]),
    "dgx_cascade": (_int, [C.POINTER(CascadeTree), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _sz]),
    "dgx_sg_filter": (_int, [C.POINTER(SgFilterTree), C.POINTER(SgFilterLeaf), _sz, _vp, _sz, _vp, _vp, _sz, C.c_int32,
                             C.c_int32, _vp, _sz, _szp, _vp, _vp, _sz, _vp]),
    "dgx_match": (_int, [C.POINTER(PackRef), _sz, _vp, _vp, _vp, _vp, _vp, _sz, _u64, _vp, _sz, C.POINTER(StrColumn), _vp,
                         _sz, C.c_int64, _vp, _sz, _szp]),
    "dgx_regex_compile": (_int, [_vp, _sz, _int, C.POINTER(_vp)]),
    "dgx_regex_free": (None, [_vp]),
    "dgx_regex_tables": (_int, [_vp, _szp, _szp, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp)]),
    "dgx_regex_match": (_int, [C.POINTER(PackRef), _sz, _vp, _vp, _vp, _vp, _vp, _sz, _u64, _vp, _sz,
                               C.POINTER(StrColumn), _vp, _vp, _sz, _szp]),
    "dgx_compare_uids": (_int, [_int, C.POINTER(ValArgs), C.POINTER(ValColumn), _vp, _sz, _vp, _sz, _szp, _vp]),
    "dgx_compare_rows": (_int, [_int, C.POINTER(ValArgs), C.POINTER(ValColumn), _vp, _vp, _sz, _vp, _vp, _vp, _sz]),
    "dgx_var_order": (_int, [C.POINTER(MathLeaf), _int, _vp, _sz, _vp, _vp, _sz, C.c_int32, C.c_int32, _vp, _vp, _sz,
                             _vp, _sz, _szp]),
    "dgx_pred_order": (_int, [C.POINTER(ValColumn), _int, _vp, _sz, _vp, _vp, _sz, C.c_int32, C.c_int32, _vp, _vp,
                              _sz, _vp, _sz, _szp]),
    "dgx_groupby_uid": (_int, [_vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _vp, _sz, _vp, _sz, _szp, _szp]),
    "dgx_pack_seek": (_int, [C.POINTER(PackView), _int, _u64, _int, _sz, _vp, _sz, _szp, _szp]),
    "dgx_encode_bound": (None, [_sz, C.c_uint32, _szp, _szp]),
    "dgx_encode": (_int, [_vp, _sz, C.c_uint32, _vp, _vp, _vp, _vp, _szp, _szp, C.POINTER(PackView)]),
    "dgx_intersect_packed": (_int, [C.POINTER(PackRef), C.POINTER(PackRef), C.c_uint32, _vp, _vp, _vp, _vp, _szp, _szp, C.POINTER(PackView)]),
    "dgx_difference_packed": (_int, [C.POINTER(PackRef), C.POINTER(PackRef), C.c_uint32, _vp, _vp, _vp, _vp, _szp, _szp, C.POINTER(PackView)]),
    "dgx_intersect_sorted_packed_out": (_int, [C.POINTER(PackRef), _sz, C.c_uint32, _vp, _vp, _vp, _vp, _szp, _szp, C.POINTER(PackView)]),
    "dgx_merge_sorted_packed": (_int, [C.POINTER(PackRef), _sz, C.c_uint32, _vp, _vp, _vp, _vp, _szp, _szp, C.POINTER(PackView)]),
    "dgx_pack_image_size": (_sz, [_sz, _sz]),
    "dgx_pack_image_view": (_int, [_vp, C.c_uint32, _sz, _sz, C.POINTER(PackView)]),
    "dgx_cache_configure": (_int, [_sz]),
    "dgx_cache_clear": (None, []),
    "dgx_cache_get_stats": (None, [C.POINTER(CacheStats)]),
    "dgx_index_of_batch": (_int, [_vp, _sz, _vp, _sz, _vp]),
    "dgx_intersect_batch_shared": (_int, [_vp, _vp, _sz, _vp, _sz, _vp, _vp, _sz]),
    "dgx_lane_create": (_vp, [_int, _vp]),
    "dgx_lane_destroy": (None, [_vp]),
    "dgx_lane_sync": (_int, [_vp]),
    "dgx_lane_stream": (_vp, [_vp]),
    "dgx_lane_set_resident_inputs": (_int, [_vp, _int]),
    "dgx_lane_launches": (_u64, [_vp]),
    "dgx_dev_alloc": (_vp, [_sz]),
    "dgx_dev_free": (None, [_vp]),
    "dgx_memcpy_h2d": (_int, [_vp, _vp, _vp, _sz]),
    "dgx_memcpy_d2h": (_int, [_vp, _vp, _vp, _sz]),
    "dgx_dev_filter_batch": (_int, [_vp, _int, _vp, _vp, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_merge_sorted": (_int, [_vp, _vp, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_pack_upload": (_int, [_vp, C.POINTER(PackView), C.POINTER(_vp)]),
    "dgx_dev_pack_free": (None, [_vp]),
    "dgx_dev_pack_exact_len": (_sz, [_vp]),
    "dgx_dev_pack_bytes": (_sz, [_vp]),
    "dgx_dev_decode": (_int, [_vp, _vp, _u64, _vp, _sz, _vp]),
    "dgx_dev_intersect_compressed_rows": (_int, [_vp, _vp, _sz, _u64, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_intersect_compressed_matrix": (_int, [_vp, _vp, _vp, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_decode_to_buffer_rows": (_int, [_vp, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_encode_from_buffer_rows": (_int, [_vp, _vp, _vp, _sz, C.c_uint32, _vp, _sz, _vp, _vp, _vp]),
    "dgx_dev_merge_sorted_matrix": (_int, [_vp, _vp, _vp, _sz, _sz, _vp, _sz, _vp]),
    "dgx_dev_list_uids_rows": (_int, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _u64, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_list_uids_unfiltered_rows": (_int, [_vp, _vp, _sz, _vp, _vp, _vp, _u64, C.c_int32, _vp, _sz, _vp]),
    "dgx_dev_list_count_rows": (_int, [_vp, _vp, _sz, _vp, _vp, _vp, _u64, _vp]),
    "dgx_dev_trigram_query": (_int, [_vp, C.POINTER(QueryTree), _vp, _sz, _vp, _vp, _vp, _vp, _vp, _sz, _u64, _vp, _sz, _vp]),
    "dgx_dev_recurse_filter": (_int, [_vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_var_propagate": (_int, [_vp, _int, _vp, _vp, _sz, C.POINTER(VarLevel), _sz, _vp, _vp, _sz, _vp]),
    "dgx_dev_var_level_agg": (_int, [_vp, _int, _int, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _sz, _vp, _vp, _sz, _vp]),
    "dgx_dev_math_eval": (_int, [_vp, C.POINTER(MathNode), _sz, C.POINTER(MathLeaf), _sz, _vp, _sz, _vp, _vp, _vp, _sz,
                                 _vp]),
    "dgx_dev_path_expand": (_int, [_vp, _vp, C.POINTER(PathLevel), _sz, _sz, _sz, _vp, _vp, _sz, _vp]),
    "dgx_dev_cascade": (_int, [_vp, C.POINTER(CascadeTree), C.POINTER(CascadeNode), _vp, _vp, _sz, _vp, _vp, _sz, _vp]),
    "dgx_dev_sg_filter": (_int, [_vp, C.POINTER(SgFilterTree), C.POINTER(SgFilterLeaf), _sz, _vp, _sz, _vp, _vp, _vp,
                                 _sz, _sz, C.c_int32, C.c_int32, _vp, _sz, _vp, _vp, _vp, _sz, _vp]),
    "dgx_dev_match": (_int, [_vp, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _sz, _u64, _int, _vp, _sz, _vp,
                             C.POINTER(StrColumn), _vp, _sz, C.c_int64, _vp, _sz, _vp]),
    "dgx_dev_regex_match": (_int, [_vp, _vp, _sz, _vp, _vp, _vp, _vp, _vp, _sz, _u64, _int, _vp, _sz, _vp,
                                   C.POINTER(StrColumn), _vp, _vp, _sz, _vp]),
    "dgx_dev_compare_uids": (_int, [_vp, _int, C.POINTER(ValArgs), C.POINTER(ValColumn), _vp, _sz, _vp, _vp, _sz,
                                    _vp, _vp]),
    "dgx_dev_compare_rows": (_int, [_vp, _int, C.POINTER(ValArgs), C.POINTER(ValColumn), _vp, _vp, _sz, _sz, _vp,
                                    _vp, _vp, _sz]),
    "dgx_dev_var_order": (_int, [_vp, C.POINTER(MathLeaf), _int, _vp, _sz, _vp, _vp, _vp, _sz, _sz, C.c_int32,
                                 C.c_int32, _vp, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_pred_order": (_int, [_vp, C.POINTER(ValColumn), _int, _vp, _sz, _vp, _vp, _vp, _sz, _sz, C.c_int32,
                                  C.c_int32, _vp, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_groupby_uid": (_int, [_vp, _vp, _sz, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _sz, _sz, _sz, _vp, _vp, _vp, _sz, _vp, _sz, _vp]),
    "dgx_merge_matrix_overflows": (_u64, [_vp]),
    "dgx_filter_tail_queries": (_u64, [_vp]),
    "dgx_wire_posting_list_pack": (_int, [_vp, _sz, C.POINTER(_vp), _szp]),
    "dgx_wire_pack_measure": (_int, [_vp, _sz, _szp, _szp]),
    "dgx_wire_pack_parse": (_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _sz, C.POINTER(PackView)]),
    "dgx_wire_list_header": (_sz, [_sz, _vp]),
    "dgx_wire_uid_matrix": (_int, [_vp, _vp, _sz, _vp, _sz, _szp]),
    "dgx_wire_list_decode": (_int, [_vp, _sz, _vp, _sz, _szp]),
}

_lib = None


def load() -> C.CDLL:
    """dlopen libdgx.so and bind every exported symbol.  Raises if the library is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(
            f"{SO_PATH} not found: the CUDA extension is not built. "
            "Run `make` (or __graft_entry__.build()); there is no CPU fallback."
        )
    lib = C.CDLL(SO_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != DGX_OK:
        raise DgxError(rc, load().dgx_last_error().decode("utf-8", "replace"))


def describe() -> str:
    buf = C.create_string_buffer(512)
    check(load().dgx_describe(buf, 512))
    return buf.value.decode()


def stats() -> dict:
    s = Stats()
    load().dgx_get_stats(C.byref(s))
    return {n: getattr(s, n) for n, _ in Stats._fields_}
