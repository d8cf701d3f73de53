"""Per-kernel device times of C17b's hub level (tools/bench_ops.py c17_rows: C13's matrix as one propagation level,
its most popular destination 999 736 in-edges), int and float maps, by torch.profiler over 5 resident calls each.

    python tools/prof_valvar_hub.py --out valvar_hub_prof.json
"""
import argparse
import ctypes as C, json, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); args = ap.parse_args()
import gen_groupby as gg
from dgraph_b200 import _lib
lib = _lib.load(); _lib.check(lib.dgx_init(0))
st = torch.cuda.Stream(); torch.cuda.set_stream(st)
lane = lib.dgx_lane_create(0, C.c_void_p(st.cuda_stream))
src, v, v_off, dest = gg.c13_rows(np.random.default_rng(13))
rng = np.random.default_rng(18)
up = lambda x: torch.from_numpy(np.concatenate([np.ascontiguousarray(x, np.uint64), np.zeros(1, np.uint64)]).view(np.int64)).cuda()
dl = [up(x) for x in (src, v, v_off, dest)]
arr = (_lib.VarLevel * 1)(_lib.VarLevel(dl[0].data_ptr(), dl[2].data_ptr(), dl[1].data_ptr(), dl[3].data_ptr(), src.size, int(v_off[-1]), dest.size))
out = {"device": torch.cuda.get_device_name(0)}
import subprocess
out["power"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
for typ, name in ((1, "int"), (2, "float")):
    pk = np.sort(rng.choice(src, int(src.size * 0.9), replace=False))
    pv = rng.integers(-1000, 1000, pk.size) if typ == 1 else rng.normal(0, 1e3, pk.size)
    dk, dv = up(pk), up(np.ascontiguousarray(pv).view(np.uint64))
    ok, ov = (torch.empty(dest.size + 1, dtype=torch.int64, device="cuda") for _ in range(2))
    dn = torch.empty(1, dtype=torch.int64, device="cuda")
    call = lambda: _lib.check(lib.dgx_dev_var_propagate(lane, typ, dk.data_ptr(), dv.data_ptr(), pk.size, arr, 1, ok.data_ptr(), ov.data_ptr(), dest.size, dn.data_ptr()))
    for _ in range(2): call()
    _lib.check(lib.dgx_lane_sync(lane))
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5): call()
        _lib.check(lib.dgx_lane_sync(lane))
    k = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0):
            t = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            if t: k[e.key[:60]] = round(t / 5 / 1000, 4)
    out[name] = dict(sorted(k.items(), key=lambda x: -x[1]))
json.dump(out, open(args.out, "w"), indent=1)
print(json.dumps(out, indent=1))
lib.dgx_lane_destroy(lane)
