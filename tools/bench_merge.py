#!/usr/bin/env python
"""MergeSorted alone (BASELINE config 5: k=64 lists, lengths ~ 1/rank, 1e8 UIDs in total) on one H100, device-resident,
CUDA-event timed, checked against torch.unique.  tools/bench_ops.py holds the same row; this script exists to iterate
on the merge kernels without paying for the other configs.  --dense adds a densely allocated variant (gaps 1..3)."""
import argparse, json, os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_ops import Lane, zipf_gaps_gpu, thin_gpu, timeit, DEV, peak_gbs   # noqa: E402


def one(L, lists, label, peak, reps):
    tot = sum(t.numel() for t in lists)
    out = torch.empty(tot + 8, dtype=torch.int64, device=DEV)
    out_len = torch.zeros(1, dtype=torch.int64, device=DEV)
    ms, _ = timeit(lambda: L.merge(lists, out, out_len), warm=2, reps=reps)
    L.sync()
    nm = int(out_len.item())
    want = torch.unique(torch.cat(lists))
    ok = bool(nm == want.numel() and torch.equal(out[:nm], want))
    gb = 8 * (tot + nm) / 1e9
    return {"case": label, "ms": round(ms, 4), "in": tot, "out": nm, "GBps": round(gb / ms * 1e3, 1),
            "frac": round(gb / ms * 1e3 / peak, 4), "check": ok}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--scale", type=int, default=1, help="divide sizes by this")
    ap.add_argument("--dense", action="store_true")
    a = ap.parse_args()
    gen = torch.Generator(device=DEV); gen.manual_seed(5)
    L = Lane()
    peak = peak_gbs()[0]
    total = 100_000_000 // a.scale
    master = zipf_gaps_gpu(2 * total, gen)
    w = 1.0 / np.arange(1, 65)
    lens = (w / w.sum() * total).astype(np.int64)
    lists = [thin_gpu(master, float(l) / master.numel(), gen) for l in lens]
    print(json.dumps(one(L, lists, "C5 zipf-gap", peak, a.reps)), flush=True)
    if a.dense:
        g = torch.randint(1, 4, (2 * total,), device=DEV, generator=gen, dtype=torch.int64)
        master = torch.cumsum(g, 0) + (1 << 40)
        lists = [thin_gpu(master, float(l) / master.numel(), gen) for l in lens]
        print(json.dumps(one(L, lists, "C5 dense (gaps 1..3)", peak, a.reps)), flush=True)
        eq = [thin_gpu(master, 1.0 / 128, gen) for _ in range(64)]
        print(json.dumps(one(L, eq, "64 equal lists", peak, a.reps)), flush=True)


if __name__ == "__main__":
    main()
