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
    "dgx_dev_merge_sorted_matrix": (_int, [_vp, _vp, _vp, _sz, _sz, _vp, _sz, _vp]),
    "dgx_dev_list_uids_rows": (_int, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _u64, _vp, _sz, _vp, _sz, _vp]),
    "dgx_dev_list_uids_unfiltered_rows": (_int, [_vp, _vp, _sz, _vp, _vp, _vp, _u64, C.c_int32, _vp, _sz, _vp]),
    "dgx_dev_list_count_rows": (_int, [_vp, _vp, _sz, _vp, _vp, _vp, _u64, _vp]),
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
