"""dgraph_b200: H100-native (sm_90a CUDA) posting-list set operations and
UidPack decode -- the drop-in for dgraph's algo/ + codec/ hot path.

The product is dgraph_b200/libdgx.so behind include/dgx.h; the modules here are
the host-side mirror of the reference's Go API used by the parity tests:

    from dgraph_b200 import algo, codec, pb
    o = pb.List(); algo.IntersectWith(pb.List(u), pb.List(v), o)
"""
from . import _lib, pb  # noqa: F401
from . import algo, codec  # noqa: F401

__all__ = ["algo", "codec", "pb", "_lib"]
