#!/usr/bin/env python
"""Per-operation device-resident benchmarks of libdgx on one H100 (BASELINE configs C1-C5).

Complements bench.py (which times the headline config C2): every row reports CUDA-event
time, input UIDs/s, algorithmic GB/s (SURVEY.md 8d formulas) and the fraction of the
measured HBM peak, plus a correctness check computed independently on the GPU with torch
(sort/unique/isin) or against the original list.  Output: one JSON document on stdout /
--out.

    python tools/bench_ops.py [--out gpurun_out/ops.json] [--small]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from dgraph_b200 import _lib  # noqa: E402

DEV = torch.device("cuda", 0)


def peak_gbs():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        return float(json.load(open(p))["hbm_gbs"]), "measured"
    return 3350.0, "H100 SXM data sheet"


def zipf_gaps_gpu(n, gen, a=1.5, clip=1 << 20):
    """Zipf-like gap list on the GPU: gap = min(floor(u^(-1/(a-1))), clip), uid = cumsum(gap)."""
    u = torch.rand(n, device=DEV, generator=gen, dtype=torch.float64).clamp_(min=1e-12)
    g = torch.clamp(torch.floor(u.pow(-1.0 / (a - 1.0))), max=float(clip)).to(torch.int64)
    return torch.cumsum(g, 0)


def thin_gpu(master, p, gen):
    return master[torch.rand(master.numel(), device=DEV, generator=gen) < p].contiguous()


class Lane:
    def __init__(self, lib=None, handle=None):
        self.lib = lib or _lib.load()
        if handle is not None:   # bench.py's lane (already bound to torch's current stream)
            self.h = handle
            return
        _lib.check(self.lib.dgx_init(0))
        self.stream = torch.cuda.Stream(device=DEV)
        torch.cuda.set_stream(self.stream)
        self.h = self.lib.dgx_lane_create(0, C.c_void_p(self.stream.cuda_stream))
        assert self.h

    def sync(self):
        _lib.check(self.lib.dgx_lane_sync(self.h))

    def filter_batch(self, op, lists, k_off, out, out_off):
        self.prepared(op, lists, k_off, out, out_off)()

    def prepared(self, op, lists, k_off, out, out_off):
        """The descriptor tables are marshalled ONCE (20 000 data_ptr() calls take milliseconds of Python): the
        returned closure is what gets timed -- one C-ABI call."""
        n = len(lists)
        ptrs = (C.c_void_p * n)(*[t.data_ptr() for t in lists])
        lens = (C.c_size_t * n)(*[t.numel() for t in lists])
        koff = (C.c_size_t * len(k_off))(*k_off)
        nq, po, cap, poff = len(k_off) - 1, C.c_void_p(out.data_ptr()), out.numel(), C.c_void_p(out_off.data_ptr())

        def call():
            _lib.check(self.lib.dgx_dev_filter_batch(self.h, op, ptrs, lens, koff, nq, po, cap, poff))
        return call

    def merge(self, lists, out, out_len):
        n = len(lists)
        ptrs = (C.c_void_p * n)(*[t.data_ptr() for t in lists])
        lens = (C.c_size_t * n)(*[t.numel() for t in lists])
        _lib.check(self.lib.dgx_dev_merge_sorted(self.h, ptrs, lens, n, C.c_void_p(out.data_ptr()), out.numel(),
                                                 C.c_void_p(out_len.data_ptr())))


def timeit(fn, warm=3, reps=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    evs[0].record()
    for i in range(reps):
        fn()
        evs[i + 1].record()
    torch.cuda.synchronize()
    ts = [evs[i].elapsed_time(evs[i + 1]) for i in range(reps)]
    return float(np.median(ts)), ts


QUIET = False


def row(name, cfg, ms, uids_in, algo_bytes, ok, extra=None):
    peak, src = peak_gbs()
    gbs = algo_bytes / (ms * 1e-3) / 1e9
    r = {"op": name, "config": cfg, "ms": ms, "uids_in": int(uids_in), "uids_per_s": uids_in / (ms * 1e-3),
         "algorithmic_bytes": int(algo_bytes), "algorithmic_GBps": gbs, "frac_of_hbm_peak": gbs / peak,
         "peak_GBps": peak, "peak_source": src, "check": ok}
    if extra:
        r.update(extra)
    if not QUIET:
        print(json.dumps(r), flush=True)
    return r


def quick_rows(lib, lane, dev, peak):
    """bench.py's `ops` key: one compact line per BASELINE config other than the headline, full sizes,
    device-resident, CUDA events, independent torch check; no CPU legs (bench.py has its own)."""
    global DEV, QUIET
    DEV, QUIET = dev, True
    rows = run(Lane(lib, lane), 1, quick=True)
    return [{"op": r["op"], "config": r["config"], "ms": round(r["ms"], 4), "uids_per_s": r["uids_per_s"],
             "algorithmic_GBps": round(r["algorithmic_GBps"], 1), "frac_of_hbm_peak": round(r["algorithmic_GBps"] / peak, 4),
             "check": r["check"]} for r in rows]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true", help="1/10 sizes (quick functional pass)")
    ap.add_argument("--c6-only", action="store_true", help="only the C6 handleUidPostings rows")
    ap.add_argument("--c7-only", action="store_true", help="only the C7 sort-bucket rows")
    ap.add_argument("--c8-only", action="store_true", help="only the C8 DestUIDs (MergeSorted of a uid matrix) rows")
    ap.add_argument("--c9-only", action="store_true", help="only the C9 List.Uids rows with mutable layers")
    ap.add_argument("--c10-only", action="store_true", help="only the C10 unfiltered List.Uids and count rows")
    ap.add_argument("--c11-only", action="store_true", help="only the C11 backup / restore codec rows")
    ap.add_argument("--c12-only", action="store_true", help="only the C12 regexp() trigram query rows")
    ap.add_argument("--c13-only", action="store_true", help="only the C13 @groupby over a uid predicate rows")
    ap.add_argument("--c14-only", action="store_true", help="only the C14 @recurse filter rows")
    ap.add_argument("--c15-only", action="store_true", help="only the C15 @cascade rows")
    ap.add_argument("--c16-only", action="store_true", help="only the C16 shortest() rows")
    ap.add_argument("--c17-only", action="store_true", help="only the C17 value-variable rows")
    ap.add_argument("--c18-only", action="store_true", help="only the C18 math() rows")
    ap.add_argument("--c19-only", action="store_true", help="only the C19 @filter and first / offset rows")
    ap.add_argument("--c20-only", action="store_true", help="only the C20 orderasc / orderdesc by a value variable rows")
    ap.add_argument("--c21-only", action="store_true", help="only the C21 match() rows")
    ap.add_argument("--c23-only", action="store_true", help="only the C23 compare function rows")
    ap.add_argument("--c24-only", action="store_true", help="only the C24 orderasc / orderdesc by a predicate rows")
    args = ap.parse_args()
    if args.c6_only:
        rows = c6_rows(Lane())
    elif args.c7_only:
        rows = c7_rows(Lane())
    elif args.c8_only:
        rows = c8_rows(Lane())
    elif args.c9_only:
        rows = c9_rows(Lane())
    elif args.c10_only:
        rows = c10_rows(Lane())
    elif args.c11_only:
        rows = c11_rows(Lane())
    elif args.c12_only:
        rows = c12_rows(Lane())
    elif args.c13_only:
        rows = c13_rows(Lane())
    elif args.c14_only:
        rows = c14_rows(Lane())
    elif args.c15_only:
        rows = c15_rows(Lane())
    elif args.c16_only:
        rows = c16_rows(Lane())
    elif args.c17_only:
        rows = c17_rows(Lane())
    elif args.c18_only:
        rows = c18_rows(Lane())
    elif args.c19_only:
        rows = c19_rows(Lane())
    elif args.c20_only:
        rows = c20_rows(Lane())
    elif args.c21_only:
        rows = c21_rows(Lane())
    elif args.c23_only:
        rows = c23_rows(Lane())
    elif args.c24_only:
        rows = c24_rows(Lane())
    else:
        rows = run(Lane(), 10 if args.small else 1, quick=False)
    if args.c6_only or args.c7_only or args.c8_only or args.c9_only or args.c10_only or args.c11_only or args.c12_only or args.c13_only or args.c14_only or args.c15_only or args.c16_only or args.c17_only or args.c18_only or args.c19_only or args.c20_only or args.c21_only or args.c23_only or args.c24_only:  # the card and its power limit, read in the same run as the numbers
        import subprocess

        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
        rows = {"device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": q, "rows": rows}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


def run(L, S, quick):
    import gen as hostgen

    small = S > 1
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1234)
    rows = []

    # ---- C1: 2-way IntersectWith, 2 x 1e5 uniform in [0, 1e7): single call latency + batched x2048
    n1 = 100_000
    pairs = []
    for i in range((512 if quick else 2048) // S):
        a = torch.unique(torch.randint(0, 10_000_000, (int(n1 * 1.02),), device=DEV, generator=gen))[:n1].contiguous()
        b = torch.unique(torch.randint(0, 10_000_000, (int(n1 * 1.02),), device=DEV, generator=gen))[:n1].contiguous()
        pairs.append((a, b))
    out = torch.empty(n1 * len(pairs) + 8, dtype=torch.int64, device=DEV)
    off = torch.zeros(len(pairs) + 1, dtype=torch.int64, device=DEV)
    a, b = pairs[0]
    ms, _ = timeit(L.prepared(0, [a, b], [0, 2], out, off), reps=50)
    L.sync()
    nout = int(off[1].item())
    want = a[torch.isin(a, b, assume_unique=True)]
    ok = bool(torch.equal(out[:nout], want))
    rows.append(row("IntersectWith", "C1: 2 x 1e5 uniform unique in [0,1e7), one call (launch-latency bound, L2 resident)",
                    ms, 2 * n1, 8 * (2 * n1 + nout), ok, {"out": nout}))
    lists, koff = [], [0]
    for a, b in pairs:
        lists += [a, b]
        koff.append(len(lists))
    ms, _ = timeit(L.prepared(0, lists, koff, out, off))
    L.sync()
    offc = off.cpu().numpy()
    ok = True
    for i in (0, len(pairs) // 2, len(pairs) - 1):
        a, b = pairs[i]
        ok = ok and bool(torch.equal(out[offc[i]:offc[i + 1]], a[torch.isin(a, b, assume_unique=True)]))
    tot = sum(a.numel() + b.numel() for a, b in pairs)
    rows.append(row("IntersectWith (batch)", f"C1 x {len(pairs)} pairs in one launch", ms, tot, 8 * (tot + int(offc[-1])), ok))
    del pairs, lists

    # ---- C2 dense variant: k=8, thinnings p=0.9 of a 1.11e6 master, 16 queries
    Q = 16 // (4 if small else 1)
    lists, koff, wants = [], [0], []
    for q in range(Q):
        master = zipf_gaps_gpu(1_110_000, gen)
        ql = [thin_gpu(master, 0.9, gen) for _ in range(8)]
        lists += ql
        koff.append(len(lists))
    cap = sum(min(t.numel() for t in lists[koff[q]:koff[q + 1]]) for q in range(Q))
    out = torch.empty(cap + 8, dtype=torch.int64, device=DEV)
    off = torch.zeros(Q + 1, dtype=torch.int64, device=DEV)
    ms, _ = timeit(L.prepared(0, lists, koff, out, off))
    L.sync()
    offc = off.cpu().numpy()
    w = lists[0]
    for t in lists[1:8]:
        w = w[torch.isin(w, t, assume_unique=True)]
    ok = bool(torch.equal(out[offc[0]:offc[1]], w))
    tot = sum(t.numel() for t in lists)
    rows.append(row("IntersectSorted (dense)", f"C2 variant: k=8 thinnings p=0.9 of a 1.11e6 Zipf master, {Q} queries per launch",
                    ms, tot, 8 * (tot + int(offc[-1])), ok, {"out": int(offc[-1])}))
    del lists

    # ---- C4 (single GPU share): batched 2-way, sizes ~ power law alpha=2 on [1e4, 1e6]
    npairs = 10_000 // S  # the whole 10k-pair batch on one GPU (~7.7 GB of lists)
    rng = np.random.default_rng(401)
    u = rng.random(npairs)
    sizes = np.minimum((1e4 / (1 - u * (1 - 1e4 / 1e6))).astype(np.int64), 1_000_000)
    lists, koff = [], [0]
    for sz in sizes:
        master = zipf_gaps_gpu(int(sz) * 2, gen)
        lists += [thin_gpu(master, 0.5, gen), thin_gpu(master, 0.5, gen)]
        koff.append(len(lists))
    cap = sum(min(lists[2 * i].numel(), lists[2 * i + 1].numel()) for i in range(npairs))
    out = torch.empty(cap + 8, dtype=torch.int64, device=DEV)
    off = torch.zeros(npairs + 1, dtype=torch.int64, device=DEV)
    ms, _ = timeit(L.prepared(0, lists, koff, out, off), reps=5)
    L.sync()
    offc = off.cpu().numpy()
    ok = True
    for i in (0, npairs // 3, npairs - 1):
        a, b = lists[2 * i], lists[2 * i + 1]
        ok = ok and bool(torch.equal(out[offc[i]:offc[i + 1]], a[torch.isin(a, b, assume_unique=True)]))
    tot = sum(t.numel() for t in lists)
    rows.append(row("IntersectWith (batch, skewed sizes)", f"C4: {npairs} pairs in one launch, sizes ~ power law alpha=2 on [1e4,1e6], thinnings p=0.5",
                    ms, tot, 8 * (tot + int(offc[-1])), ok, {"total_uids": tot}))
    del lists, out

    # ---- C5: MergeSorted k=64, total 1e8 (lengths ~ 1/rank), then Difference with a 1e7 list
    total = 100_000_000 // S
    master = zipf_gaps_gpu(2 * total, gen)
    w = 1.0 / np.arange(1, 65)
    lens = (w / w.sum() * total).astype(np.int64)
    lists = [thin_gpu(master, float(l) / master.numel(), gen) for l in lens]
    tot = sum(t.numel() for t in lists)
    out = torch.empty(tot + 8, dtype=torch.int64, device=DEV)
    out_len = torch.zeros(1, dtype=torch.int64, device=DEV)
    ms, _ = timeit(lambda: L.merge(lists, out, out_len), warm=2, reps=5)
    L.sync()
    nm = int(out_len.item())
    want = torch.unique(torch.cat(lists))
    ok = bool(nm == want.numel() and torch.equal(out[:nm], want))
    del want
    rows.append(row("MergeSorted", f"C5: k=64 lists, lengths ~ 1/rank, total {tot} UIDs (thinnings of a {master.numel()} master); single-pass multiway merge (merge_multi.cuh + merge_tile32.cuh)",
                    ms, tot, 8 * (tot + nm), ok, {"out": nm}))
    dlist = thin_gpu(master, 10_000_000 / S / master.numel(), gen)
    merged = out[:nm].clone()
    dout = torch.empty(nm + 8, dtype=torch.int64, device=DEV)
    doff = torch.zeros(2, dtype=torch.int64, device=DEV)
    ms, _ = timeit(L.prepared(1, [merged, dlist], [0, 2], dout, doff), warm=2, reps=5)
    L.sync()
    nd = int(doff[1].item())
    want = merged[~torch.isin(merged, dlist, assume_unique=True)]
    ok = bool(nd == want.numel() and torch.equal(dout[:nd], want))
    rows.append(row("Difference", f"C5: merged ({nm}) minus a {dlist.numel()}-UID list", ms, nm + dlist.numel(),
                    8 * (nm + dlist.numel() + nd), ok, {"out": nd}))
    del lists, out, merged, dout, want, master

    # ---- C3: codec.Decode of a 1e8-UID pack (BlockSize 256), then IntersectSorted with 1e7 and 1e6 lists
    n3 = 100_000_000 // S
    master = zipf_gaps_gpu(n3, gen)
    host = master.cpu().numpy().view(np.uint64)

    class _P:  # the pack's arrays (numpy generator, tests/gen.py; byte-identical to the oracle's Encode)
        pass
    pack = _P()
    _, pack.base, pack.num_uids, pack.delta_off, pack.deltas = hostgen.encode_pack_np_parallel(host, 256, threads=min(32, os.cpu_count() or 1))
    pack.nblocks = pack.base.size
    view = _lib.PackView()
    base, num, doff_, deltas = pack.base, pack.num_uids, pack.delta_off, pack.deltas
    view.block_size, view.nblocks = 256, pack.nblocks
    view.base, view.num_uids, view.delta_off, view.deltas = base.ctypes.data, num.ctypes.data, doff_.ctypes.data, deltas.ctypes.data
    pk = C.c_void_p()
    _lib.check(L.lib.dgx_dev_pack_upload(L.h, C.byref(view), C.byref(pk)))
    pack_bytes = int(deltas.size + 12 * pack.nblocks)
    out = torch.empty(n3 + 8, dtype=torch.int64, device=DEV)
    out_len = torch.zeros(1, dtype=torch.int64, device=DEV)

    def dec():
        _lib.check(L.lib.dgx_dev_decode(L.h, pk, 0, C.c_void_p(out.data_ptr()), n3, C.c_void_p(out_len.data_ptr())))

    ms, _ = timeit(dec, warm=2, reps=5)
    L.sync()
    ok = bool(int(out_len.item()) == n3 and torch.equal(out[:n3], master))
    extra = {"pack_bytes": pack_bytes}
    if not quick:
        from oracle import pyoracle as orc   # CPU comparison leg only

        sample = host[: min(n3, 20_000_000)]
        t0 = time.perf_counter()
        spack = orc.encode(sample, 256)
        t_enc = time.perf_counter() - t0
        t1 = time.perf_counter()
        orc.decode(spack, 0)
        t_dec_cpu = time.perf_counter() - t1
        extra.update({"cpu_oracle_decode_uids_per_s": sample.size / t_dec_cpu, "cpu_oracle_encode_uids_per_s": sample.size / t_enc})
    rows.append(row("codec.Decode", f"C3: {n3}-UID pack, BlockSize 256, {pack.nblocks} blocks, {deltas.size / n3:.3f} delta bytes/UID",
                    ms, n3, pack_bytes + 8 * n3, ok, extra))
    l1 = thin_gpu(master, 0.1, gen)
    l2 = thin_gpu(master, 0.01, gen)
    decoded = out[:n3]
    iout = torch.empty(l2.numel() + 8, dtype=torch.int64, device=DEV)
    ioff = torch.zeros(2, dtype=torch.int64, device=DEV)
    ms_i, _ = timeit(L.prepared(0, [decoded, l1, l2], [0, 3], iout, ioff), warm=2, reps=5)
    L.sync()
    ni = int(ioff[1].item())
    want = l2[torch.isin(l2, l1, assume_unique=True)]
    ok = bool(ni == want.numel() and torch.equal(iout[:ni], want))
    tot = n3 + l1.numel() + l2.numel()
    rows.append(row("IntersectSorted after Decode", f"C3: [decoded {n3}, {l1.numel()}, {l2.numel()}] (driven from the shortest list; long lists are probed, not streamed)",
                    ms_i, tot, 8 * (tot + ni), ok, {"out": ni, "note": "algorithmic bytes count every list once; the kernel reads far fewer"}))
    rows.append(row("Decode + IntersectSorted (pipeline)", "C3 end to end on device: decode to HBM, then intersect",
                    ms + ms_i, tot, pack_bytes + 8 * n3 + 8 * (tot + ni), ok))
    L.lib.dgx_dev_pack_free(pk)
    if quick:
        return rows

    # ---- C3 end to end through the host-pointer C ABI: the pack crosses PCIe COMPRESSED ---------
    # (dgx_decode_intersect_sorted: H2D of the pack + the two lists, decode and intersect on the
    # device, D2H of the result) against the CPU oracle doing codec.Decode + algo.IntersectSorted.
    h1 = l1.cpu().numpy().view(np.uint64)
    h2 = l2.cpu().numpy().view(np.uint64)
    hp = (C.c_void_p * 2)(h1.ctypes.data, h2.ctypes.data)
    hl = (C.c_size_t * 2)(h1.size, h2.size)
    hout = np.empty(h2.size, dtype=np.uint64)
    hn = C.c_size_t(0)

    def e2e():
        _lib.check(L.lib.dgx_decode_intersect_sorted(C.byref(view), 0, hp, hl, 2, hout.ctypes.data_as(C.c_void_p),
                                                      hout.size, C.byref(hn)))

    e2e()
    t0 = time.perf_counter()
    for _ in range(3):
        e2e()
    t_e2e = (time.perf_counter() - t0) / 3
    ok = bool(hn.value == ni and np.array_equal(hout[: hn.value], iout[:ni].cpu().numpy().view(np.uint64)))
    t1 = time.perf_counter()
    dec_cpu = orc.decode(spack, 0)          # the 2e7-UID sample pack, scaled below
    t_dec = (time.perf_counter() - t1) * (n3 / sample.size)
    t1 = time.perf_counter()
    orc.intersect_sorted([host, h1, h2])
    t_int = time.perf_counter() - t1
    r = row("Decode + IntersectSorted (host pointers, e2e)",
            "C3 through dgx_decode_intersect_sorted: pack (compressed) and lists cross PCIe, result comes back",
            t_e2e * 1e3, tot, pack_bytes + 8 * (l1.numel() + l2.numel()) + 8 * ni, ok,
            {"h2d_bytes": pack_bytes + 8 * (h1.size + h2.size), "cpu_oracle_ms": (t_dec + t_int) * 1e3,
             "cpu_oracle_decode_ms": t_dec * 1e3, "cpu_oracle_intersect_ms": t_int * 1e3,
             "speedup_vs_cpu_1thread": (t_dec + t_int) / t_e2e,
             "note": "algorithmic bytes here = bytes that cross PCIe; the CPU figure is the single-threaded oracle (decode scaled from a 2e7-UID sample)"})
    rows.append(r)
    # same call with every input in pinned host memory (dgx_host_alloc): PCIe at DMA speed
    def pin(a):
        ptr = L.lib.dgx_host_alloc(max(a.nbytes, 16))
        C.memmove(ptr, a.ctypes.data, a.nbytes)
        return ptr
    pview = _lib.PackView()
    pview.block_size, pview.nblocks = 256, pack.nblocks
    pins = [pin(base), pin(num), pin(doff_), pin(deltas), pin(h1), pin(h2)]
    pview.base, pview.num_uids, pview.delta_off, pview.deltas = pins[0], pins[1], pins[2], pins[3]
    php = (C.c_void_p * 2)(pins[4], pins[5])

    def e2e_pinned():
        _lib.check(L.lib.dgx_decode_intersect_sorted(C.byref(pview), 0, php, hl, 2, hout.ctypes.data_as(C.c_void_p),
                                                      hout.size, C.byref(hn)))

    e2e_pinned()
    t0 = time.perf_counter()
    for _ in range(3):
        e2e_pinned()
    t_pin = (time.perf_counter() - t0) / 3
    ok = bool(hn.value == ni and np.array_equal(hout[: hn.value], iout[:ni].cpu().numpy().view(np.uint64)))
    rows.append(row("Decode + IntersectSorted (pinned host pointers, e2e)", "as above, inputs in dgx_host_alloc memory",
                    t_pin * 1e3, tot, pack_bytes + 8 * (l1.numel() + l2.numel()) + 8 * ni, ok,
                    {"speedup_vs_cpu_1thread": (t_dec + t_int) / t_pin, "cpu_oracle_ms": (t_dec + t_int) * 1e3}))
    for ptr in pins:
        L.lib.dgx_host_free(ptr)
    rows += c6_rows(L)
    rows += c7_rows(L)
    rows += c8_rows(L)
    rows += c9_rows(L)
    return rows


def c6_rows(L, threads: int = 4):
    """C6 "handleUidPostings": one task's 10 000 posting lists (UidPacks, BlockSize 256) each intersected with the same
    v from the same afterUID (worker/task.go:783-987 -> algo.IntersectCompressedWith).  Five legs on the same inputs,
    each checked row by row against the oracle: (1) dgx_dev_intersect_compressed_rows on resident packs (CUDA events),
    (2) the host form with named packs in steady state, (3) the host form with anonymous packs flattened back to back
    into one pinned buffer (every pack crosses PCIe each step), (4) dgx_intersect_compressed_ref per row from
    `threads` host threads, (5) the oracle row loop on one thread and on every host thread."""
    from concurrent.futures import ThreadPoolExecutor

    import gen_rows
    from oracle import pyoracle as orc

    lib = L.lib
    master, rows_u, v = gen_rows.c6_inputs()
    nrows, m = len(rows_u), v.size
    ops = [orc.encode(r, 256) for r in rows_u]
    arrs = [(op.base, op.num_uids, op.delta_off, op.deltas) for op in ops]
    exact = sum(r.size for r in rows_u)
    del rows_u
    # flat images of all packs back to back in one pinned buffer (what the shim's flatten writes)
    sizes = [lib.dgx_pack_image_size(a[0].size, a[3].size) for a in arrs]
    blob = lib.dgx_host_alloc(sum(sizes) + 64)
    assert blob
    views, o = [], 0
    for (base, num, doff, deltas), sz in zip(arrs, sizes):
        pv = _lib.PackView()
        _lib.check(lib.dgx_pack_image_view(C.c_void_p(blob + o), 256, base.size, deltas.size, C.byref(pv)))
        C.memmove(pv.base, base.ctypes.data, base.nbytes)
        C.memmove(pv.delta_off, doff.ctypes.data, doff.nbytes)
        C.memmove(pv.num_uids, num.ctypes.data, num.nbytes)
        C.memmove(pv.deltas, deltas.ctypes.data, deltas.nbytes)
        views.append(pv)
        o += sz

    def refs_of(named: bool):
        refs = (_lib.PackRef * nrows)()
        for i in range(nrows):
            refs[i].pack = C.pointer(views[i])
            refs[i].key, refs[i].version = ((900_000 + i) if named else 0), 1
        return refs

    named, anon = refs_of(True), refs_of(False)
    hv = np.ascontiguousarray(v)
    cap = sum(min(m, int(a[1].sum(dtype=np.uint64))) for a in arrs)
    hout = np.empty(max(cap, 1), np.uint64)
    hoff = np.zeros(nrows + 1, np.uint64)

    def host_rows(refs, after):
        _lib.check(lib.dgx_intersect_compressed_rows(refs, nrows, after, hv.ctypes.data_as(C.c_void_p), m,
                                                      hout.ctypes.data_as(C.c_void_p), hoff.ctypes.data_as(C.c_void_p), cap))

    def wall(fn, reps):
        fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps * 1e3

    # device-resident packs for leg 1
    handles = []
    for pv in views:
        h = C.c_void_p()
        _lib.check(lib.dgx_dev_pack_upload(L.h, C.byref(pv), C.byref(h)))
        handles.append(h)
    tab = (C.c_void_p * nrows)(*[h.value for h in handles])
    d_v = torch.from_numpy(hv.view(np.int64)).to(DEV)
    d_out = torch.empty(cap + 8, dtype=torch.int64, device=DEV)
    d_off = torch.zeros(nrows + 1, dtype=torch.int64, device=DEV)
    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(16 << 30))
    out_rows = []
    try:
        for after in (0, int(master[master.size // 2])):
            t0 = time.perf_counter()
            want = [orc.intersect_compressed_with(op, after, v) for op in ops]
            t_orc1 = time.perf_counter() - t0
            ncpu = os.cpu_count() or 1
            t0 = time.perf_counter()
            with ThreadPoolExecutor(max_workers=ncpu) as ex:   # ctypes releases the GIL
                list(ex.map(lambda op: orc.intersect_compressed_with(op, after, v), ops))
            t_orcn = time.perf_counter() - t0
            want_off = np.concatenate([[0], np.cumsum([w.size for w in want])]).astype(np.uint64)
            want_all = np.concatenate(want) if want_off[-1] else np.zeros(0, np.uint64)
            nout = int(want_off[-1])
            abytes = gen_rows.algorithmic_bytes([(a[0], a[2]) for a in arrs], after, hv, nout)

            def same(out, off):
                return bool(np.array_equal(off, want_off) and np.array_equal(out[:nout], want_all))

            def dev():
                _lib.check(lib.dgx_dev_intersect_compressed_rows(L.h, tab, nrows, after, C.c_void_p(d_v.data_ptr()), m,
                                                                 C.c_void_p(d_out.data_ptr()), cap, C.c_void_p(d_off.data_ptr())))
            ms1, _ = timeit(dev, warm=3, reps=10)
            L.sync()
            ok1 = same(d_out[:nout].cpu().numpy().view(np.uint64), d_off.cpu().numpy().view(np.uint64))
            ms2 = wall(lambda: host_rows(named, after), 5)
            ok2 = same(hout, hoff)
            hoff[:] = 0
            ms3 = wall(lambda: host_rows(anon, after), 5)
            ok3 = same(hout, hoff)
            single_out = [np.empty(max(min(m, int(a[1].sum(dtype=np.uint64))), 1), np.uint64) for a in arrs]
            single_n = [C.c_size_t(0) for _ in range(nrows)]

            def one(i):
                _lib.check(lib.dgx_intersect_compressed_ref(C.byref(named[i]), after, hv.ctypes.data_as(C.c_void_p), m,
                                                            single_out[i].ctypes.data_as(C.c_void_p), single_out[i].size,
                                                            C.byref(single_n[i])))

            def per_row():
                with ThreadPoolExecutor(max_workers=threads) as ex:
                    list(ex.map(one, range(nrows)))
            ms4 = wall(per_row, 2)
            ok4 = all(np.array_equal(single_out[i][: single_n[i].value], want[i]) for i in range(nrows))
            cfg = (f"C6 handleUidPostings: {nrows} UidPacks (BlockSize 256, sizes ~ power law alpha=2 on [1e3,1e6], samples of a "
                   f"2e7 Zipf-gap master, {exact} UIDs) each ∩ one v ({m} UIDs, thinning p=0.05), afterUID={after}")
            uids_in = exact + m
            extra = {"rows": nrows, "out": nout, "after": after,
                     "bytes_note": "algorithmic bytes count every v element inside a touched block's range once per row; "
                                   "slices longer than 4x the block are probed by binary search, so the kernel reads far "
                                   "fewer and the GB/s figure is not an HBM rate"}
            for name, ms, ok, note in (
                ("IntersectCompressedWithRows (device, resident packs)", ms1, ok1, "dgx_dev_intersect_compressed_rows, CUDA events"),
                ("IntersectCompressedWithRows (host, named packs, cache hits)", ms2, ok2, "dgx_intersect_compressed_rows, wall clock incl. D2H"),
                ("IntersectCompressedWithRows (host, anonymous packs over PCIe)", ms3, ok3, "one pinned flat-image buffer per step, wall clock"),
                (f"IntersectCompressedWith per row ({threads} host threads)", ms4, ok4, "dgx_intersect_compressed_ref per row, named packs, wall clock"),
                ("oracle row loop (1 thread)", t_orc1 * 1e3, True, "algo.IntersectCompressedWith restated in C, one row after another"),
                (f"oracle row loop ({ncpu} threads)", t_orcn * 1e3, True, "same, rows spread over every host thread"),
            ):
                out_rows.append(row(name, cfg, ms, uids_in, abytes, ok, dict(extra, rows_per_s=nrows / (ms * 1e-3), note=note)))
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_cache_clear()
        lib.dgx_host_free(C.c_void_p(blob))
    return out_rows


def c7_rows(L, threads: int = 4):
    """C7 "sort buckets": one uid matrix of 10 000 rows (sizes ~ power law alpha=2 on [10, 1e4]) intersected with each
    of three index-bucket packs (BlockSize 256: 1e6, 1e4 and 100 uids), the intersectBucket loop of an indexed sort
    (worker/sort.go:605-700 -> algo.IntersectCompressedWith(pack, 0, row)).  Four legs per bucket, each checked row by
    row against the oracle: (1) dgx_dev_intersect_compressed_matrix with the pack and the matrix resident (CUDA
    events), (2) dgx_intersect_compressed_matrix with a named pack that hits the cache, the matrix crossing PCIe every
    call (wall clock), (3) dgx_intersect_compressed_ref per row from `threads` host threads, (4) the oracle row loop on
    one thread, as the reference's single goroutine runs it."""
    from concurrent.futures import ThreadPoolExecutor

    import gen_sort
    from dgraph_b200 import codec, pb
    from oracle import pyoracle as orc

    lib = L.lib
    master, rows_u, buckets = gen_sort.c7_inputs()
    nrows = len(rows_u)
    v_off = np.zeros(nrows + 1, np.uint64)
    np.cumsum([r.size for r in rows_u], out=v_off[1:])
    hv = np.ascontiguousarray(np.concatenate(rows_u))
    m = hv.size
    d_v = torch.from_numpy(hv.view(np.int64)).to(DEV)
    pv_off = v_off.ctypes.data_as(C.c_void_p)

    def wall(fn, reps):
        fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps * 1e3

    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(16 << 30))
    out_rows = []
    for bi, (bname, uids) in enumerate(buckets.items()):
        op = orc.encode(uids, 256)
        pk = pb.UidPack(op.block_size, op.base, op.num_uids, op.delta_off, op.deltas).normalized()
        view = codec.view_of(pk)  # pk stays alive for the whole bucket
        ref = _lib.PackRef(C.pointer(view), 700_000 + bi, 1)
        t0 = time.perf_counter()
        want = [orc.intersect_compressed_with(op, 0, r) for r in rows_u]
        t_orc = time.perf_counter() - t0
        want_off = np.concatenate([[0], np.cumsum([w.size for w in want])]).astype(np.uint64)
        want_all = np.concatenate(want) if want_off[-1] else np.zeros(0, np.uint64)
        nout = int(want_off[-1])
        cap = int(np.minimum(np.diff(v_off), uids.size).sum())
        abytes = gen_sort.matrix_algorithmic_bytes(pk.base, pk.delta_off, rows_u, nout)

        def same(out, off):
            return bool(np.array_equal(off, want_off) and np.array_equal(out[:nout], want_all))

        h = C.c_void_p()
        _lib.check(lib.dgx_dev_pack_upload(L.h, C.byref(view), C.byref(h)))
        try:
            d_out = torch.empty(cap + 8, dtype=torch.int64, device=DEV)
            d_off = torch.zeros(nrows + 1, dtype=torch.int64, device=DEV)

            def dev():
                _lib.check(lib.dgx_dev_intersect_compressed_matrix(L.h, h, C.c_void_p(d_v.data_ptr()), pv_off, nrows,
                                                                   C.c_void_p(d_out.data_ptr()), cap,
                                                                   C.c_void_p(d_off.data_ptr())))
            ms1, _ = timeit(dev, warm=3, reps=20)
            L.sync()
            ok1 = same(d_out[:nout].cpu().numpy().view(np.uint64), d_off.cpu().numpy().view(np.uint64))
        finally:
            lib.dgx_dev_pack_free(h)
        hout = np.empty(max(cap, 1), np.uint64)
        hoff = np.zeros(nrows + 1, np.uint64)

        def host():
            _lib.check(lib.dgx_intersect_compressed_matrix(C.byref(ref), hv.ctypes.data_as(C.c_void_p), pv_off, nrows,
                                                           hout.ctypes.data_as(C.c_void_p),
                                                           hoff.ctypes.data_as(C.c_void_p), cap))
        ms2 = wall(host, 10)
        ok2 = same(hout, hoff)
        single_out = [np.empty(max(r.size, 1), np.uint64) for r in rows_u]
        single_n = [C.c_size_t(0) for _ in range(nrows)]

        def one(i):
            r = rows_u[i]
            _lib.check(lib.dgx_intersect_compressed_ref(C.byref(ref), 0, r.ctypes.data_as(C.c_void_p), r.size,
                                                        single_out[i].ctypes.data_as(C.c_void_p), single_out[i].size,
                                                        C.byref(single_n[i])))

        def per_row():
            with ThreadPoolExecutor(max_workers=threads) as ex:
                list(ex.map(one, range(nrows)))
        ms3 = wall(per_row, 2)
        ok3 = all(np.array_equal(single_out[i][: single_n[i].value], want[i]) for i in range(nrows))
        cfg = (f"C7 sort buckets: bucket '{bname}' ({uids.size} UIDs, {op.base.size} blocks of BlockSize 256, a sample "
               f"of a 2e7 Zipf-gap master) against a uid matrix of {nrows} rows ({m} UIDs, sizes ~ power law alpha=2 "
               f"on [10,1e4], samples of the master), afterUID 0")
        extra = {"bucket": bname, "rows": nrows, "matrix_uids": m, "out": nout}
        for name, ms, ok, note in (
            ("IntersectCompressedWithMatrix (device, resident pack and matrix)", ms1, ok1,
             "dgx_dev_intersect_compressed_matrix, CUDA events"),
            ("IntersectCompressedWithMatrix (host, named pack, cache hit)", ms2, ok2,
             "dgx_intersect_compressed_matrix, the matrix crosses PCIe every call, wall clock incl. D2H"),
            (f"IntersectCompressedWith per row ({threads} host threads)", ms3, ok3,
             "dgx_intersect_compressed_ref per row, named pack, wall clock"),
            ("oracle row loop (1 thread)", t_orc * 1e3, True,
             "algo.IntersectCompressedWith restated in C, one row after another"),
        ):
            out_rows.append(row(name, cfg, ms, uids.size + m, abytes, ok,
                                dict(extra, rows_per_s=nrows / (ms * 1e-3), note=note)))
    lib.dgx_cache_clear()
    return out_rows


def c8_rows(L, reps: int = 10):
    """C8 "DestUIDs": sg.DestUIDs = algo.MergeSorted(result.UidMatrix) (query/query.go:2290) over three uid matrices
    (tests/gen_merge.py): C8a the C7 matrix, C8b the C6 rows, C8c 200 000 rows of 1-32 uids plus one hub uid in every
    row.  Legs on the same inputs, every output compared with the oracle's in full: (1) dgx_dev_merge_sorted_matrix with
    the matrix resident (CUDA events), (2) dgx_merge_sorted_matrix from pinned and (3) from pageable host memory (wall
    clock incl. D2H), (4) dgx_dev_merge_sorted with one device pointer per row (CUDA events), (5) dgx_merge_sorted with
    one host pointer per row (wall clock), (6) the oracle's MergeSorted with the reference's 10-thread split."""
    import gen_merge
    from oracle import pyoracle as orc

    lib = L.lib

    def wall(fn, n):
        fn()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        return (time.perf_counter() - t0) / n * 1e3

    out_rows = []
    for name, make in gen_merge.C8.items():
        hv, v_off = make()
        nrows, m = v_off.size - 1, hv.size
        rows_u = gen_merge.rows_of(hv, v_off)
        t0 = time.perf_counter()
        want = orc.merge_sorted(rows_u)
        t_orc = (time.perf_counter() - t0) * 1e3
        t_orc = min(t_orc, wall(lambda: orc.merge_sorted(rows_u), 2))
        nout = want.size
        abytes = gen_merge.algorithmic_bytes(m, nout)
        d_v = torch.from_numpy(hv.view(np.int64)).to(DEV)
        d_off = torch.from_numpy(v_off.view(np.int64)).to(DEV)
        d_out = torch.empty(m + 8, dtype=torch.int64, device=DEV)
        d_len = torch.zeros(1, dtype=torch.int64, device=DEV)

        def dev_got():
            L.sync()
            return d_out[: int(d_len.item())].cpu().numpy().view(np.uint64)

        l0, o0 = lib.dgx_lane_launches(L.h), lib.dgx_merge_matrix_overflows(None)

        def dev():
            _lib.check(lib.dgx_dev_merge_sorted_matrix(L.h, C.c_void_p(d_v.data_ptr()), C.c_void_p(d_off.data_ptr()), nrows,
                                                       m, C.c_void_p(d_out.data_ptr()), m, C.c_void_p(d_len.data_ptr())))
        dev()
        L.sync()
        # both counters around the first call only: per call, not summed over the timed calls
        launches = lib.dgx_lane_launches(L.h) - l0
        overflows = lib.dgx_merge_matrix_overflows(None) - o0
        ms1, _ = timeit(dev, warm=3, reps=reps)
        ok1 = bool(np.array_equal(dev_got(), want))
        # today's device path: one device pointer per row
        ptrs = (C.c_void_p * nrows)(*[d_v.data_ptr() + 8 * int(v_off[i]) for i in range(nrows)])
        lens = (C.c_size_t * nrows)(*np.diff(v_off).tolist())

        def dev_rows():
            _lib.check(lib.dgx_dev_merge_sorted(L.h, ptrs, lens, nrows, C.c_void_p(d_out.data_ptr()), m,
                                                C.c_void_p(d_len.data_ptr())))
        ms4, _ = timeit(dev_rows, warm=2, reps=max(3, reps // 2))
        ok4 = bool(np.array_equal(dev_got(), want))
        hout = np.empty(max(m, 1), np.uint64)
        n = C.c_size_t(0)
        pin_v = lib.dgx_host_alloc(max(m, 1) * 8)
        pin_off = lib.dgx_host_alloc((nrows + 1) * 8)
        try:
            pv = np.ctypeslib.as_array(C.cast(pin_v, C.POINTER(C.c_uint64)), (max(m, 1),))
            po = np.ctypeslib.as_array(C.cast(pin_off, C.POINTER(C.c_uint64)), (nrows + 1,))
            pv[:m], po[:] = hv, v_off
            res = {}
            for leg, (va, oa) in (("pinned", (pin_v, pin_off)), ("pageable", (hv.ctypes.data, v_off.ctypes.data))):
                def host(va=va, oa=oa):
                    _lib.check(lib.dgx_merge_sorted_matrix(C.c_void_p(va), C.c_void_p(oa), nrows,
                                                           hout.ctypes.data_as(C.c_void_p), m, C.byref(n)))
                res[leg] = wall(host, reps)
                res[leg + "_ok"] = bool(np.array_equal(hout[: n.value], want))
        finally:
            lib.dgx_host_free(pin_v)
            lib.dgx_host_free(pin_off)
        hptrs = (C.c_void_p * nrows)(*[hv.ctypes.data + 8 * int(v_off[i]) for i in range(nrows)])

        def host_rows():
            _lib.check(lib.dgx_merge_sorted(hptrs, lens, nrows, hout.ctypes.data_as(C.c_void_p), m, C.byref(n)))
        ms5 = wall(host_rows, max(2, reps // 2))
        ok5 = bool(np.array_equal(hout[: n.value], want))
        cfg = (f"C8 DestUIDs {name}: MergeSorted of a uid matrix of {nrows} rows, {m} UIDs -> {nout} distinct "
               f"({gen_merge.C8[name].__doc__.split(chr(10))[0]})")
        extra = {"matrix": name, "rows": nrows, "matrix_uids": m, "out": nout}
        for op, ms, ok, note in (
            ("MergeSortedMatrix (device, resident matrix)", ms1, ok1,
             f"dgx_dev_merge_sorted_matrix, CUDA events; {launches} launches per call, {overflows} overflow-path chunks"),
            ("MergeSortedMatrix (host, pinned)", res["pinned"], res["pinned_ok"],
             "dgx_merge_sorted_matrix from pinned memory, wall clock incl. H2D and D2H"),
            ("MergeSortedMatrix (host, pageable)", res["pageable"], res["pageable_ok"],
             "dgx_merge_sorted_matrix from pageable memory, wall clock incl. H2D and D2H"),
            ("MergeSorted, one device pointer per row", ms4, ok4, "dgx_dev_merge_sorted, CUDA events"),
            ("MergeSorted, one host pointer per row", ms5, ok5, "dgx_merge_sorted, wall clock incl. H2D and D2H"),
            ("oracle MergeSorted (10-thread split)", t_orc, True, "algo.MergeSorted restated in C, wall clock"),
        ):
            out_rows.append(row(op, cfg, ms, m, abytes, ok, dict(extra, note=note, launches_per_call=launches,
                                                                 overflow_chunks=overflows)))
        del d_v, d_off, d_out
    return out_rows


def c9_rows(L, threads: int = 16):
    """C9 "handleUidPostings with writes": the C6 task (10 000 UidPacks, one v of about 1e6 uids) where 30 % of the
    keys carry a mutable layer of about 1 % of their length (deletes, new uids from the master, value postings;
    tests/gen_mut.py), each key read with the List.Uids branch the ApproxLen rule picks.  Legs on the same inputs, each
    checked row by row against the oracle's List.Uids: (1) dgx_dev_list_uids_rows on resident packs (CUDA events),
    (2) dgx_list_uids_rows with named packs in steady state, (3) today's path: dgx_intersect_compressed_rows for the
    clean keys, then the oracle's List.Uids for every key with a layer on `threads` host threads, (4) the oracle row
    loop on one thread and on `threads` threads."""
    from concurrent.futures import ThreadPoolExecutor

    import gen_mut
    import gen_rows
    import list_uids_oracle as luo
    from oracle import pyoracle as orc

    lib = L.lib
    master, rows_u, v = gen_rows.c6_inputs()
    nrows, m = len(rows_u), v.size
    ops = [orc.encode(r, 256) for r in rows_u]
    rng = np.random.default_rng(909)
    muts, modes = [], []
    for r, op in zip(rows_u, ops):
        layer = rng.random() < 0.3
        mu, mf = gen_mut.layer(rng, r, master, max(1, r.size // 100)) if layer else (np.zeros(0, np.uint64),
                                                                                      np.zeros(0, np.uint8))
        muts.append((mu, mf))
        modes.append(gen_mut.mode_of(orc.approx_len(op), m, layer))
    exact = sum(r.size for r in rows_u)
    del rows_u
    mode = np.array(modes, np.uint8)
    mut_off = np.zeros(nrows + 1, np.uint64)
    np.cumsum([t[0].size for t in muts], out=mut_off[1:])
    mu_all = np.concatenate([t[0] for t in muts])
    mf_all = np.concatenate([t[1] for t in muts])
    nmut = int(mut_off[-1])
    dirty = [i for i in range(nrows) if modes[i] != gen_mut.COMPRESSED]
    clean = [i for i in range(nrows) if modes[i] == gen_mut.COMPRESSED]
    views = []
    for op in ops:
        arrs = (op.base, op.num_uids, op.delta_off, op.deltas)  # copies: they stay alive with the view
        views.append((_lib.PackView(256, op.nblocks, *[a.ctypes.data for a in arrs]),) + arrs)
    refs = (_lib.PackRef * nrows)()
    for i in range(nrows):
        refs[i].pack, refs[i].key, refs[i].version = C.pointer(views[i][0]), 950_000 + i, 1
    crefs = (_lib.PackRef * len(clean))(*[refs[i] for i in clean])
    hv = np.ascontiguousarray(v)
    cap = sum(min(m, int(op.num_uids.sum(dtype=np.uint64)) + t[0].size) for op, t in zip(ops, muts))
    hout = np.empty(max(cap, 1), np.uint64)
    hoff = np.zeros(nrows + 1, np.uint64)
    ccap = sum(min(m, int(ops[i].num_uids.sum(dtype=np.uint64))) for i in clean)
    cout = np.empty(max(ccap, 1), np.uint64)
    coff = np.zeros(len(clean) + 1, np.uint64)

    def p(a):
        return a.ctypes.data_as(C.c_void_p)

    def oracle_row(i, after):
        return luo.list_uids(ops[i], modes[i], muts[i][0], muts[i][1], after, v)

    def wall(fn, reps):
        fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps * 1e3

    handles = []
    for pv in views:
        h = C.c_void_p()
        _lib.check(lib.dgx_dev_pack_upload(L.h, C.byref(pv[0]), C.byref(h)))
        handles.append(h)
    tab = (C.c_void_p * nrows)(*[h.value for h in handles])
    d_v = torch.from_numpy(hv.view(np.int64)).to(DEV)
    d_mu = torch.from_numpy(mu_all.view(np.int64)).to(DEV)
    d_mf = torch.from_numpy(mf_all).to(DEV)
    d_out = torch.empty(cap + 8, dtype=torch.int64, device=DEV)
    d_off = torch.zeros(nrows + 1, dtype=torch.int64, device=DEV)
    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(16 << 30))
    out_rows = []
    try:
        for after in (0, int(v[v.size // 2])):
            t0 = time.perf_counter()
            want = [oracle_row(i, after) for i in range(nrows)]
            t_orc1 = time.perf_counter() - t0
            t0 = time.perf_counter()
            with ThreadPoolExecutor(max_workers=threads) as ex:   # ctypes releases the GIL
                list(ex.map(lambda i: oracle_row(i, after), range(nrows)))
            t_orcn = time.perf_counter() - t0
            want_off = np.concatenate([[0], np.cumsum([w.size for w in want])]).astype(np.uint64)
            want_all = np.concatenate(want) if want_off[-1] else np.zeros(0, np.uint64)
            nout = int(want_off[-1])

            def same(out, off):
                return bool(np.array_equal(off, want_off) and np.array_equal(out[:nout], want_all))

            def dev():
                _lib.check(lib.dgx_dev_list_uids_rows(L.h, tab, p(mode), nrows, C.c_void_p(d_mu.data_ptr()),
                                                      C.c_void_p(d_mf.data_ptr()), p(mut_off), after,
                                                      C.c_void_p(d_v.data_ptr()), m, C.c_void_p(d_out.data_ptr()), cap,
                                                      C.c_void_p(d_off.data_ptr())))
            ms1, _ = timeit(dev, warm=3, reps=10)
            L.sync()
            ok1 = same(d_out[:nout].cpu().numpy().view(np.uint64), d_off.cpu().numpy().view(np.uint64))

            def host():
                _lib.check(lib.dgx_list_uids_rows(refs, p(mode), nrows, p(mu_all), p(mf_all), p(mut_off), after, p(hv), m,
                                                  p(hout), p(hoff), cap))
            ms2 = wall(host, 5)
            ok2 = same(hout, hoff)
            got3 = [None] * nrows

            def today():
                _lib.check(lib.dgx_intersect_compressed_rows(crefs, len(clean), after, p(hv), m, p(cout), p(coff), ccap))
                for j, i in enumerate(clean):
                    got3[i] = cout[int(coff[j]): int(coff[j + 1])]
                with ThreadPoolExecutor(max_workers=threads) as ex:
                    for i, r in zip(dirty, ex.map(lambda i: oracle_row(i, after), dirty)):
                        got3[i] = r
            ms3 = wall(today, 3)
            ok3 = all(np.array_equal(got3[i], want[i]) for i in range(nrows))
            cfg = (f"C9 handleUidPostings with mutable layers: the C6 task ({nrows} UidPacks, BlockSize 256, {exact} UIDs; "
                   f"v of {m} UIDs); {len(dirty)} keys with a resolved layer of ~1 % of their length ({nmut} entries: "
                   f"deletes, new uids, value postings), modes by the ApproxLen rule "
                   f"({int((mode == 1).sum())} probe, {int((mode == 2).sum())} iterate); afterUID={after}")
            extra = {"rows": nrows, "out": nout, "after": after, "mutable_entries": nmut, "rows_with_layer": len(dirty),
                     "bytes_note": "algorithmic bytes here are 8 per pack uid, v uid, mutable entry and result uid: a "
                                   "size of the work, not an HBM rate (packs are read compressed and probed sparsely)"}
            for name, ms, ok, note in (
                ("ListUidsRows (device, resident packs)", ms1, ok1, "dgx_dev_list_uids_rows, CUDA events"),
                ("ListUidsRows (host, named packs, cache hits)", ms2, ok2, "dgx_list_uids_rows, wall clock incl. D2H"),
                (f"clean rows batched + oracle List.Uids per layered row ({threads} threads)", ms3, ok3,
                 "dgx_intersect_compressed_rows for keys without a layer, then the CPU for the rest, wall clock"),
                ("oracle row loop (1 thread)", t_orc1 * 1e3, True, "List.Uids restated in C, one row after another"),
                (f"oracle row loop ({threads} threads)", t_orcn * 1e3, True, "same, rows spread over host threads"),
            ):
                out_rows.append(row(name, cfg, ms, exact + m + nmut, 8 * (exact + m + nmut + nout), ok,
                                    dict(extra, rows_per_s=nrows / (ms * 1e-3), note=note)))
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_cache_clear()
    return out_rows


def c10_rows(L, threads: int = 16):
    """C10 "handleUidPostings without a filter": the C9 task (the C6 packs, mutable layers on 30 % of the keys) read as
    a plain edge traversal (List.Uids with Intersect == nil) and as count(pred), at after = 0 and after = the master's
    median, with first = MaxInt32 (opts.First 0), first = 10 and as counts.  Legs on the same inputs, each checked row
    by row against the oracle's unfiltered List.Uids / count: (1) the device form on resident packs (CUDA events),
    (2) the host form with named packs in steady state, (3) today's path: the oracle per key on 1 and on `threads`
    host threads."""
    from concurrent.futures import ThreadPoolExecutor

    import gen_mut
    import gen_mut_unfiltered
    import gen_rows
    import list_uids_unfiltered_oracle as luo
    from oracle import pyoracle as orc

    lib = L.lib
    master, rows_u, _ = gen_rows.c6_inputs()
    nrows = len(rows_u)
    ops = [orc.encode(r, 256) for r in rows_u]
    rng = np.random.default_rng(909)
    muts = []
    for r, op in zip(rows_u, ops):  # the C9 layers (the same draws)
        layer = rng.random() < 0.3
        muts.append(gen_mut.layer(rng, r, master, max(1, r.size // 100)) if layer else (np.zeros(0, np.uint64),
                                                                                        np.zeros(0, np.uint8)))
    exact = sum(r.size for r in rows_u)
    del rows_u
    mut_off = np.zeros(nrows + 1, np.uint64)
    np.cumsum([t[0].size for t in muts], out=mut_off[1:])
    mu_all = np.concatenate([t[0] for t in muts])
    mf_all = np.concatenate([t[1] for t in muts])
    nmut = int(mut_off[-1])
    views = []
    for op in ops:
        arrs = (op.base, op.num_uids, op.delta_off, op.deltas)  # copies: they stay alive with the view
        views.append((_lib.PackView(256, op.nblocks, *[a.ctypes.data for a in arrs]),) + arrs)
    refs = (_lib.PackRef * nrows)()
    for i in range(nrows):
        refs[i].pack, refs[i].key, refs[i].version = C.pointer(views[i][0]), 960_000 + i, 1
    pack_bytes = sum(int(op.deltas.size) + 12 * int(op.nblocks) for op in ops)
    lens = [int(op.num_uids.sum(dtype=np.uint64)) + t[0].size for op, t in zip(ops, muts)]

    def p(a):
        return a.ctypes.data_as(C.c_void_p)

    def wall(fn, reps):
        fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps * 1e3

    handles = []
    for pv in views:
        h = C.c_void_p()
        _lib.check(lib.dgx_dev_pack_upload(L.h, C.byref(pv[0]), C.byref(h)))
        handles.append(h)
    tab = (C.c_void_p * nrows)(*[h.value for h in handles])
    d_mu = torch.from_numpy(mu_all.view(np.int64)).to(DEV)
    d_mf = torch.from_numpy(mf_all).to(DEV)
    cap_full = sum(lens)
    d_out = torch.empty(cap_full + 8, dtype=torch.int64, device=DEV)
    d_off = torch.zeros(nrows + 1, dtype=torch.int64, device=DEV)
    d_cnt = torch.zeros(nrows, dtype=torch.int32, device=DEV)
    hout = np.empty(max(cap_full, 1), np.uint64)
    hoff = np.zeros(nrows + 1, np.uint64)
    hcnt = np.zeros(nrows, np.uint32)
    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(16 << 30))
    out_rows = []
    try:
        for after in (0, int(master[master.size // 2])):
            for first in (0, 10, None):  # None: the count
                if first is None:
                    def oracle_row(i):
                        return luo.list_count(ops[i], muts[i][0], muts[i][1], after)
                else:
                    def oracle_row(i):
                        return luo.list_uids_unfiltered(ops[i], muts[i][0], muts[i][1], after, first)
                t0 = time.perf_counter()
                want = [oracle_row(i) for i in range(nrows)]
                t_orc1 = time.perf_counter() - t0
                t0 = time.perf_counter()
                with ThreadPoolExecutor(max_workers=threads) as ex:   # ctypes releases the GIL
                    got_n = list(ex.map(oracle_row, range(nrows)))
                t_orcn = time.perf_counter() - t0
                if first is None:
                    want_cnt = np.array(want, np.uint32)
                    nout = 0
                    ok_n = bool(np.array_equal(np.array(got_n, np.uint32), want_cnt))

                    def dev():
                        _lib.check(lib.dgx_dev_list_count_rows(L.h, tab, nrows, C.c_void_p(d_mu.data_ptr()),
                                                               C.c_void_p(d_mf.data_ptr()), p(mut_off), after,
                                                               C.c_void_p(d_cnt.data_ptr())))

                    def host():
                        _lib.check(lib.dgx_list_count_rows(refs, nrows, p(mu_all), p(mf_all), p(mut_off), after,
                                                           p(hcnt)))
                    ms1, _ = timeit(dev, warm=3, reps=10)
                    L.sync()
                    ok1 = bool(np.array_equal(d_cnt.cpu().numpy().view(np.uint32), want_cnt))
                    ms2 = wall(host, 5)
                    ok2 = bool(np.array_equal(hcnt, want_cnt))
                    what = "count"
                else:
                    want_off = np.concatenate([[0], np.cumsum([w.size for w in want])]).astype(np.uint64)
                    want_all = np.concatenate(want) if want_off[-1] else np.zeros(0, np.uint64)
                    nout = int(want_off[-1])
                    ok_n = all(np.array_equal(a, b) for a, b in zip(got_n, want))
                    cap = sum(min(gen_mut_unfiltered.most_kept(first), n) for n in lens)

                    def same(out, off):
                        return bool(np.array_equal(off, want_off) and np.array_equal(out[:nout], want_all))

                    def dev():
                        _lib.check(lib.dgx_dev_list_uids_unfiltered_rows(
                            L.h, tab, nrows, C.c_void_p(d_mu.data_ptr()), C.c_void_p(d_mf.data_ptr()), p(mut_off),
                            after, first, C.c_void_p(d_out.data_ptr()), cap, C.c_void_p(d_off.data_ptr())))

                    def host():
                        _lib.check(lib.dgx_list_uids_unfiltered_rows(refs, nrows, p(mu_all), p(mf_all), p(mut_off),
                                                                     after, first, p(hout), p(hoff), cap))
                    ms1, _ = timeit(dev, warm=3, reps=10)
                    L.sync()
                    ok1 = same(d_out[:nout].cpu().numpy().view(np.uint64), d_off.cpu().numpy().view(np.uint64))
                    ms2 = wall(host, 5)
                    ok2 = same(hout, hoff)
                    what = "first = MaxInt32 (opts.First 0)" if first == 0 else f"first = {first}"
                cfg = (f"C10 handleUidPostings without a filter: the C9 task ({nrows} UidPacks, BlockSize 256, {exact} "
                       f"UIDs, {pack_bytes} pack bytes; {nmut} resolved entries on "
                       f"{int((np.diff(mut_off) > 0).sum())} keys); {what}; afterUID={after}")
                extra = {"rows": nrows, "out": nout, "after": after, "first": first, "mutable_entries": nmut,
                         "pack_bytes": pack_bytes,
                         "bytes_note": "algorithmic bytes: the pack bytes, 9 per mutable entry and 8 per result uid (4 "
                                       "per count); a size of the work, not an HBM rate"}
                algo_bytes = pack_bytes + 9 * nmut + (4 * nrows if first is None else 8 * nout)
                fn = "count_rows" if first is None else "unfiltered_rows"
                for name, ms, ok, note in (
                    (f"List {fn} (device, resident packs)", ms1, ok1, f"dgx_dev_list_{fn}, CUDA events"),
                    (f"List {fn} (host, named packs, cache hits)", ms2, ok2, f"dgx_list_{fn}, wall clock incl. D2H"),
                    ("today: oracle per key (1 thread)", t_orc1 * 1e3, True, "restated in C, one key after another"),
                    (f"today: oracle per key ({threads} threads)", t_orcn * 1e3, ok_n, "same, keys spread over threads"),
                ):
                    out_rows.append(row(name, cfg, ms, exact + nmut, algo_bytes, ok,
                                        dict(extra, rows_per_s=nrows / (ms * 1e-3), note=note)))
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_cache_clear()
    return out_rows


def c11_rows(L, threads: int = 16):
    """C11 "backup and restore": the C6 task's 10 000 packs (BlockSize 256) converted to BackupPostingList.uid_bytes
    (codec.DecodeToBuffer per key) and those bytes back to packs (codec.EncodeFromBuffer(uid_bytes, 256) per key).
    Legs on the same inputs, each checked row by row against the oracle's restatement (tests/backup_codec_oracle.c):
    (1) the device form on resident inputs (CUDA events), (2) the host form with named packs (backup) / pinned bytes
    (restore), (3) the host form with anonymous packs over PCIe (one run of images) / pageable bytes, (4) today's path:
    the oracle per key on 1 and on `threads` host threads."""
    from concurrent.futures import ThreadPoolExecutor

    import backup_codec_oracle as bco
    import gen_rows
    from backup_codec_cases import pack_images
    from oracle import pyoracle as orc

    lib = L.lib
    _, rows_u, _ = gen_rows.c6_inputs()
    nrows = len(rows_u)
    ops = [orc.encode(r, 256) for r in rows_u]
    exact = sum(r.size for r in rows_u)
    del rows_u
    pack_bytes = sum(int(op.deltas.size) + 12 * int(op.nblocks) for op in ops)

    def p(a):
        return a.ctypes.data_as(C.c_void_p)

    def wall(fn, reps):
        fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps * 1e3

    def per_key(fn):
        t0 = time.perf_counter()
        got = [fn(i) for i in range(nrows)]
        t1 = time.perf_counter() - t0
        t0 = time.perf_counter()
        with ThreadPoolExecutor(max_workers=threads) as ex:  # ctypes releases the GIL
            got_n = list(ex.map(fn, range(nrows)))
        return got, t1 * 1e3, got_n, (time.perf_counter() - t0) * 1e3

    # ---- backup: packs -> uid_bytes ----------------------------------------------------------------------------
    want, t_b1, got_n, t_bn = per_key(lambda i: bco.decode_to_buffer(ops[i]))
    ok_bn = got_n == want
    want_off = np.zeros(nrows + 1, np.uint64)
    np.cumsum([len(w) for w in want], out=want_off[1:])
    want_all = np.frombuffer(b"".join(want), np.uint8)
    nbytes = int(want_off[-1])

    def same_bytes(out, off):
        return bool(np.array_equal(off, want_off) and np.array_equal(out[:nbytes], want_all))

    views = []
    for op in ops:
        arrs = (op.base, op.num_uids, op.delta_off, op.deltas)  # copies: they stay alive with the view
        views.append((_lib.PackView(256, op.nblocks, *[a.ctypes.data for a in arrs]),) + arrs)
    named = (_lib.PackRef * nrows)()
    for i in range(nrows):
        named[i].pack, named[i].key, named[i].version = C.pointer(views[i][0]), 1_100_000 + i, 1
    img_in, img_in_off, img_in_nb, img_in_db = pack_images(ops)
    anon_views = [_lib.PackView() for _ in range(nrows)]
    anon = (_lib.PackRef * nrows)()
    for i in range(nrows):
        _lib.check(lib.dgx_pack_image_view(C.c_void_p(img_in.ctypes.data + int(img_in_off[i])), 256, int(img_in_nb[i]),
                                           int(img_in_db[i]), C.byref(anon_views[i])))
        anon[i].pack = C.pointer(anon_views[i])
    handles = []
    for pv in views:
        h = C.c_void_p()
        _lib.check(lib.dgx_dev_pack_upload(L.h, C.byref(pv[0]), C.byref(h)))
        handles.append(h)
    tab = (C.c_void_p * nrows)(*[h.value for h in handles])
    d_out = torch.empty(nbytes + 16, dtype=torch.uint8, device=DEV)
    d_off = torch.zeros(nrows + 1, dtype=torch.int64, device=DEV)
    hout = np.empty(nbytes + 16, np.uint8)
    hoff = np.zeros(nrows + 1, np.uint64)
    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(16 << 30))
    out_rows = []
    try:
        def b_dev():
            _lib.check(lib.dgx_dev_decode_to_buffer_rows(L.h, tab, nrows, C.c_void_p(d_out.data_ptr()), nbytes,
                                                         C.c_void_p(d_off.data_ptr())))
        ms_b_dev, _ = timeit(b_dev, warm=3, reps=10)
        L.sync()
        ok_b_dev = same_bytes(d_out.cpu().numpy(), d_off.cpu().numpy().view(np.uint64))
        legs = [("Backup DecodeToBuffer rows (device, resident packs)", ms_b_dev, ok_b_dev,
                 "dgx_dev_decode_to_buffer_rows, CUDA events")]
        for name, refs, note in (("host, named packs, cache hits", named, "dgx_decode_to_buffer_rows, wall clock"),
                                 ("host, anonymous packs over PCIe", anon,
                                  "dgx_decode_to_buffer_rows, one run of pack images, wall clock")):
            hout[:] = 0
            ms = wall(lambda: _lib.check(lib.dgx_decode_to_buffer_rows(refs, nrows, p(hout), p(hoff), nbytes)), 5)
            legs.append((f"Backup DecodeToBuffer rows ({name})", ms, same_bytes(hout, hoff), note))
        legs += [("Backup today: oracle per key (1 thread)", t_b1, True, "restated in C, one key after another"),
                 (f"Backup today: oracle per key ({threads} threads)", t_bn, ok_bn, "same, keys spread over threads")]
        cfg = (f"C11 backup: the C6 task ({nrows} UidPacks, BlockSize 256, {exact} UIDs, {pack_bytes} pack bytes) "
               f"to {nbytes} bytes of uvarint uid_bytes")
        for name, ms, ok, note in legs:
            out_rows.append(row(name, cfg, ms, exact, pack_bytes + nbytes,
                                ok, {"rows": nrows, "rows_per_s": nrows / (ms * 1e-3), "out_bytes": nbytes,
                                     "note": note, "bytes_note": "algorithmic bytes: pack bytes in + uid_bytes out"}))

        # ---- restore: uid_bytes -> packs ---------------------------------------------------------------------
        back, t_r1, back_n, t_rn = per_key(lambda i: bco.encode_from_buffer(want[i], 256))

        def same_pack(rp, op):
            rc, q = rp
            return rc == 0 and all(np.array_equal(getattr(q, f), getattr(op, f))
                                   for f in ("base", "num_uids", "delta_off", "deltas"))
        ok_r1 = all(same_pack(b, op) for b, op in zip(back, ops))
        ok_rn = all(same_pack(b, op) for b, op in zip(back_n, ops))
        img_want, io_want, nb_want, db_want = pack_images([q for _, q in back])
        itotal = int(io_want[-1])

        def same_img(img, io, nb, db):
            return bool(np.array_equal(io, io_want) and np.array_equal(nb, nb_want) and np.array_equal(db, db_want)
                        and np.array_equal(img[:itotal], img_want[:itotal]))

        buf_off = want_off.copy()
        d_buf = torch.from_numpy(want_all.copy()).to(DEV)
        d_img = torch.zeros(itotal + 16, dtype=torch.uint8, device=DEV)
        d_io = torch.zeros(nrows + 1, dtype=torch.int64, device=DEV)
        d_nb = torch.zeros(nrows, dtype=torch.int64, device=DEV)
        d_db = torch.zeros(nrows, dtype=torch.int64, device=DEV)

        def dp(t):
            return C.c_void_p(t.data_ptr())

        def r_dev():
            _lib.check(lib.dgx_dev_encode_from_buffer_rows(L.h, dp(d_buf), p(buf_off), nrows, 256, dp(d_img), itotal,
                                                           dp(d_io), dp(d_nb), dp(d_db)))
        ms_r_dev, _ = timeit(r_dev, warm=3, reps=10)
        L.sync()
        ok_r_dev = same_img(d_img.cpu().numpy(), d_io.cpu().numpy().view(np.uint64), d_nb.cpu().numpy().view(np.uint64),
                            d_db.cpu().numpy().view(np.uint64))
        legs = [("Restore EncodeFromBuffer rows (device, resident bytes)", ms_r_dev, ok_r_dev,
                 "dgx_dev_encode_from_buffer_rows, CUDA events")]
        pin = lib.dgx_host_alloc(max(nbytes, 1))
        try:
            pinned = np.ctypeslib.as_array(C.cast(pin, C.POINTER(C.c_uint8)), shape=(max(nbytes, 1),))
            pinned[:nbytes] = want_all
            raw = np.zeros(itotal + 32, np.uint8)
            himg = raw[(-raw.ctypes.data) % 16:][: itotal + 16]
            hio, hnb, hdb = np.zeros(nrows + 1, np.uint64), np.zeros(nrows, np.uint64), np.zeros(nrows, np.uint64)
            for name, src, note in (("host, pinned bytes", pinned, "dgx_encode_from_buffer_rows, wall clock"),
                                    ("host, pageable bytes over PCIe", want_all,
                                     "dgx_encode_from_buffer_rows, wall clock")):
                himg[:] = 0
                ms = wall(lambda: _lib.check(lib.dgx_encode_from_buffer_rows(p(src), p(buf_off), nrows, 256, p(himg),
                                                                             itotal, p(hio), p(hnb), p(hdb))), 5)
                legs.append((f"Restore EncodeFromBuffer rows ({name})", ms, same_img(himg, hio, hnb, hdb), note))
        finally:
            lib.dgx_host_free(pin)
        legs += [("Restore today: oracle per key (1 thread)", t_r1, ok_r1, "restated in C, one key after another"),
                 (f"Restore today: oracle per key ({threads} threads)", t_rn, ok_rn, "same, keys spread over threads")]
        cfg = f"C11 restore: the {nbytes} uid_bytes of the C6 task's {nrows} keys back to {itotal} bytes of pack images"
        for name, ms, ok, note in legs:
            out_rows.append(row(name, cfg, ms, exact, nbytes + itotal,
                                ok, {"rows": nrows, "rows_per_s": nrows / (ms * 1e-3), "image_bytes": itotal,
                                     "note": note, "bytes_note": "algorithmic bytes: uid_bytes in + images out"}))
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_cache_clear()
    return out_rows


C12_PATTERNS = ("abcd", "abc|def", "abc.*def", "(abc|xyz)def", "abc(de|fg)h", "qu[aeiou]ck")


def c12_trees(gt, idx):
    """(label, tree, trigrams) of C12: the six patterns' trees, then two trees over the index's largest trigram lists,
    the regime where a selective pattern still reads big lists: an AND of the three largest lists of different words and
    a rare trigram (one small driving leaf, three large non-driving ones), and an AND of the two largest (a large
    driving leaf)."""
    trees = [(f"/{pat}/", *gt.tree_of_pattern(gt.PATTERNS[pat])) for pat in C12_PATTERNS]
    words = np.diff(idx.word_off)  # values per word: a trigram's list is at most the sum over its words
    est = sorted(((int(words[ws].sum()), t) for t, ws in idx.tri_words.items()), reverse=True)
    big, used = [], set()
    for _, t in est:  # from different words, so that the lists are not near copies of each other
        if len(big) < 3 and not used & set(idx.tri_words[t]):
            big.append(t)
            used |= set(idx.tri_words[t])
    rare = min(est, key=lambda e: abs(e[0] - 20_000))[1]
    trees.append((f"large AND selective ({'&'.join(big)}&{rare})", [(gt.QAND, [0, 1, 2, 3], [])], big + [rare]))
    trees.append((f"large AND ({'&'.join(big[:2])})", [(gt.QAND, [0, 1], [])], big[:2]))
    return trees


def c12_rows(L, threads: int = 16, n_nodes: int = 10_000_000):
    """C12 "regexp() over a trigram index": a synthetic index of n_nodes string values (tests/gen_trigram.py), the query
    trees codesearch would build for six patterns and two trees over the index's largest lists (c12_trees), every
    trigram a posting list held as a UidPack (BlockSize 256, no mutable layer).  Legs per tree, each checked in full against the oracle's restatement of
    uidsForRegex (tests/trigram_oracle.c): (1) the device form on resident packs (CUDA events), (2) the host form with
    named packs, (3) with anonymous packs over PCIe, (4) the same tree composed from existing device calls -- the
    unfiltered rows, then dgx_dev_filter_batch per AND and dgx_dev_merge_sorted per OR, bottom up, reading each length
    back -- (5) the oracle on 1 thread (warmed up, then the mean of several calls), and 16 copies of the query on `threads`
    threads (time per query)."""
    from concurrent.futures import ThreadPoolExecutor

    import gen_trigram as gt
    import trigram_oracle as tgo
    import trigram_plan as tp
    from dgraph_b200 import algo, codec, pb
    from oracle import pyoracle as orc

    lib = L.lib
    idx = gt.TrigramIndex(seed=12, n_nodes=n_nodes, n_words=20_000)
    out_rows = []
    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(16 << 30))

    def dp(t):
        return C.c_void_p(t.data_ptr())

    def wall(fn, reps):
        fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps * 1e3

    for pi, (label, tree, tris) in enumerate(c12_trees(gt, idx)):
        uids = [idx.posting(t) for t in tris]
        ops = [orc.encode(u, 256) if u.size else None for u in uids]
        packs = [pb.UidPack(o.block_size, o.base, o.num_uids, o.delta_off, o.deltas) if o is not None else None
                 for o in ops]
        nl = len(tris)
        leaf_uids = int(sum(u.size for u in uids))
        plan = tp.plan(tree, [u.size for u in uids])
        cand = int(np.unique(np.concatenate([uids[j] for j in plan.drive] + [np.zeros(0, np.uint64)])).size)
        q = tgo.Query(tree, [(o, None) for o in ops])
        want = q.run(0)
        t_o1 = wall(lambda: q.run(0), 5)
        t0 = time.perf_counter()
        with ThreadPoolExecutor(max_workers=threads) as ex:  # ctypes releases the GIL
            got_n = list(ex.map(lambda _: q.run(0), range(16)))
        t_on = (time.perf_counter() - t0) * 1e3 / 16
        ok_on = all(np.array_equal(g, want) for g in got_n)
        cap = plan.root_bound
        qt, qa = algo.query_tree(tree)
        zero_off = np.zeros(nl + 1, np.uint64)
        dummy = np.zeros(1, np.uint64)
        named = [(1_200_000 + 100 * pi + j, 1) for j in range(nl)]
        refs_n, keep_n = algo._refs_of(packs, named)
        refs_a, keep_a = algo._refs_of(packs)
        hout = np.empty(max(cap, 1), np.uint64)
        n = C.c_size_t(0)

        def host(refs):
            _lib.check(lib.dgx_trigram_query(C.byref(qt), refs, nl, _p_(dummy), _p_(dummy), _p_(zero_off), _p_(dummy),
                                             _p_(zero_off), 0, 0, _p_(hout), cap, C.byref(n)))
        handles, tab = [], (C.c_void_p * nl)()
        for j, pk in enumerate(packs):
            if pk is None:
                continue
            view = codec.view_of(pk.normalized())
            h = C.c_void_p()
            _lib.check(lib.dgx_dev_pack_upload(L.h, C.byref(view), C.byref(h)))
            handles.append(h)
            tab[j] = h.value
        try:
            d_out = torch.empty(max(cap, 1) + 4, dtype=torch.int64, device=DEV)
            d_len = torch.zeros(1, dtype=torch.int64, device=DEV)
            d_mu = torch.zeros(1, dtype=torch.int64, device=DEV)
            d_mf = torch.zeros(16, dtype=torch.uint8, device=DEV)

            def dev():
                _lib.check(lib.dgx_dev_trigram_query(L.h, C.byref(qt), tab, nl, dp(d_mu), dp(d_mf), _p_(zero_off),
                                                     dp(d_mu), _p_(zero_off), 0, 0, dp(d_out), cap, dp(d_len)))
            ms_dev, _ = timeit(dev, warm=3, reps=10)
            L.sync()
            nd = int(d_len.cpu()[0])
            ok_dev = np.array_equal(d_out[:nd].cpu().numpy().view(np.uint64), want)
            legs = [("device form, resident packs", ms_dev, ok_dev, "dgx_dev_trigram_query, CUDA events")]
            for name, refs in (("host form, named packs", refs_n), ("host form, anonymous packs", refs_a)):
                ms = wall(lambda: host(refs), 5)
                legs.append((name, ms, bool(np.array_equal(hout[:n.value], want)), "dgx_trigram_query, wall clock"))

            # composed from existing device calls: rows, then each node bottom up with its length read back
            rows_cap = sum(u.size for u in uids)
            d_rows = torch.empty(rows_cap + 4, dtype=torch.int64, device=DEV)
            d_roff = torch.zeros(nl + 1, dtype=torch.int64, device=DEV)
            bufs = []

            def composed():
                bufs.clear()
                _lib.check(lib.dgx_dev_list_uids_unfiltered_rows(L.h, tab, nl, dp(d_mu), dp(d_mf), _p_(zero_off), 0, 0,
                                                                 dp(d_rows), rows_cap, dp(d_roff)))
                L.sync()
                off = d_roff.cpu().numpy()
                leaf = [(d_rows.data_ptr() + 8 * int(off[j]), int(off[j + 1] - off[j])) for j in range(nl)]
                val = [None] * len(tree)
                for i in reversed(range(len(tree))):
                    op, ls, subs = tree[i]
                    ch = [leaf[j] for j in ls] + [val[s] for s in subs]
                    if len(ch) == 1:
                        val[i] = ch[0]
                        continue
                    tot = sum(c[1] for c in ch) if op == gt.QOR else min(c[1] for c in ch)
                    o = torch.empty(tot + 4, dtype=torch.int64, device=DEV)
                    ln = torch.zeros(2, dtype=torch.int64, device=DEV)
                    bufs.extend([o, ln])
                    ptrs = (C.c_void_p * len(ch))(*[c[0] for c in ch])
                    lens = (C.c_size_t * len(ch))(*[c[1] for c in ch])
                    if op == gt.QOR:
                        _lib.check(lib.dgx_dev_merge_sorted(L.h, ptrs, lens, len(ch), dp(o), tot, dp(ln)))
                        L.sync()
                        val[i] = (o.data_ptr(), int(ln[0].cpu()))
                    else:
                        koff = (C.c_size_t * 2)(0, len(ch))
                        _lib.check(lib.dgx_dev_filter_batch(L.h, 0, ptrs, lens, koff, 1, dp(o), tot, dp(ln)))
                        L.sync()
                        val[i] = (o.data_ptr(), int(ln[1].cpu()))
                return val[0]
            res = composed()
            ms_c = wall(composed, 5)
            res = composed()
            got_c = np.empty(res[1], np.uint64)
            if res[1]:
                _lib.check(lib.dgx_memcpy_d2h(L.h, _p_(got_c), C.c_void_p(res[0]), 8 * res[1]))
            L.sync()
            legs.append(("composed from existing device calls", ms_c, bool(np.array_equal(got_c, want)),
                         "unfiltered rows, then dgx_dev_filter_batch / dgx_dev_merge_sorted per node, a sync per node"))
            legs += [("oracle uidsForRegex (1 thread)", t_o1, True, "restated in C"),
                     (f"oracle uidsForRegex, 16 queries on {threads} threads", t_on, ok_on, "time per query")]
            cfg = (f"C12 regexp {label}: {len(tree)} nodes, {nl} trigram packs of {leaf_uids} uids over {n_nodes} values, "
                   f"{cand} candidates, {want.size} uids out")
            for name, ms, ok, note in legs:
                out_rows.append(row(f"UidsForRegex {label} ({name})", cfg, ms, leaf_uids, 8 * (leaf_uids + want.size), ok,
                                    {"leaf_uids": leaf_uids, "candidates": cand, "driving_bound": plan.dcap,
                                     "result": int(want.size), "nodes": len(tree), "leaves": nl, "note": note,
                                     "bytes_note": "algorithmic bytes: 8 per leaf uid in and per uid out"}))
        finally:
            for h in handles:
                lib.dgx_dev_pack_free(h)
    lib.dgx_cache_clear()
    return out_rows



def c13_rows(L, n_sample: int = 20):
    """C13 "@groupby over a uid predicate": 1e6 source rows of about 20 values each after repeats are dropped (about 2e7
    edges), destinations drawn Zipf-popular over 1e6 uids (tests/gen_groupby.py c13_rows).  C13a: one parent holding
    every source (fillGroupedVars, or a @groupby at the root).  C13b: 10 000 parents of about 100 sources each.  Legs:
    (1) the device form on resident inputs with members and (2) counts only (CUDA events), (3) the host form (wall
    clock), (4) the line-by-line restatement (tests/groupby_oracle.c) on 1 thread as a stand-in for today's Go path --
    it is C, not Go.  C13a is checked in full against the restatement.  The restatement loops over every source row for
    every parent (formResult's IndexOf per child row), about 1e10 searches for C13b: there it runs on the first
    n_sample parents only, its time is per parent, and those parents' groups are checked against it; the device and
    host forms must agree in full."""
    import gen_groupby as gg
    import groupby_oracle as gbo

    lib = L.lib
    rng = np.random.default_rng(13)
    src, v, v_off, dest = gg.c13_rows(rng)
    nrows, m = src.size, int(v_off[-1])
    parents_b = [src[np.unique(rng.integers(0, nrows, int(rng.integers(50, 151))))] for _ in range(10_000)]
    work = {"C13a": [src], "C13b": parents_b}
    out_rows = []

    def dp(t):
        return C.c_void_p(t.data_ptr())

    def up(x):
        return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(DEV)

    d_src, d_v, d_voff, d_dest = up(src), up(v), up(v_off), up(dest)
    for name, parents in work.items():
        par, par_off = gbo.csr(parents)
        npar, pv = len(parents), int(par_off[-1])
        # the restatement (all parents for C13a, a sample for C13b)
        samp = parents if name == "C13a" else parents[:n_sample]
        lens = np.diff(v_off.astype(np.int64))
        scap = max(sum(int(lens[np.isin(src, pr)].sum()) for pr in samp), 1)  # the sample's edges
        skeys, sagg, smem = (np.empty(scap, np.uint64) for _ in range(3))
        sgrp, smoff = np.empty(len(samp) + 1, np.uint64), np.empty(scap + 1, np.uint64)
        spar, spar_off = gbo.csr(samp)

        def oracle():
            return gbo.lib().orc_groupby_uid(src.ctypes.data, nrows, v.ctypes.data, v_off.ctypes.data, spar.ctypes.data,
                                             spar_off.ctypes.data, len(samp), skeys.ctypes.data, sagg.ctypes.data,
                                             sgrp.ctypes.data, smoff.ctypes.data, smem.ctypes.data)
        t0 = time.perf_counter()
        ng_o = oracle()
        t_or = (time.perf_counter() - t0) * 1e3
        # the host form, sized from a first counts-only call
        grp_off = np.empty(npar + 1, np.uint64)
        ng, nm = C.c_size_t(), C.c_size_t()
        probe = np.empty(1, np.uint64)
        rc = lib.dgx_groupby_uid(_p_(src), nrows, _p_(v), _p_(v_off), _p_(dest), dest.size, _p_(par), _p_(par_off), npar,
                                 _p_(probe), _p_(grp_off), _p_(probe), 0, None, 0, C.byref(ng), C.byref(nm))
        assert rc in (0, -4), rc
        G, E = ng.value, nm.value
        keys, mem_off, mem = np.empty(G, np.uint64), np.empty(G + 1, np.uint64), np.empty(E, np.uint64)

        def host():
            _lib.check(lib.dgx_groupby_uid(_p_(src), nrows, _p_(v), _p_(v_off), _p_(dest), dest.size, _p_(par),
                                           _p_(par_off), npar, _p_(keys), _p_(grp_off), _p_(mem_off), G, _p_(mem), E,
                                           C.byref(ng), C.byref(nm)))
        host()
        t0 = time.perf_counter()
        for _ in range(3):
            host()
        t_host = (time.perf_counter() - t0) * 1e3 / 3
        # the device form, resident inputs
        d_par, d_poff = up(par), up(par_off)
        d_keys, d_grp = torch.empty(G + 1, dtype=torch.int64, device=DEV), torch.empty(npar + 1, dtype=torch.int64, device=DEV)
        d_moff, d_mem = torch.empty(G + 1, dtype=torch.int64, device=DEV), torch.empty(E + 1, dtype=torch.int64, device=DEV)
        d_sizes = torch.zeros(2, dtype=torch.int64, device=DEV)

        def dev(with_members):
            _lib.check(lib.dgx_dev_groupby_uid(L.h, dp(d_src), nrows, dp(d_v), dp(d_voff), m, dp(d_dest), dest.size,
                                               dp(d_par), dp(d_poff), npar, pv, E, dp(d_keys), dp(d_grp), dp(d_moff), G,
                                               dp(d_mem) if with_members else None, E, dp(d_sizes)))
        ms_cnt, _ = timeit(lambda: dev(False), warm=2, reps=10)
        L.sync()
        ok_cnt = (np.array_equal(d_keys[:G].cpu().numpy().view(np.uint64), keys)
                  and np.array_equal(d_moff[:G + 1].cpu().numpy().view(np.uint64), mem_off))
        ms_mem, _ = timeit(lambda: dev(True), warm=2, reps=10)
        L.sync()
        ok_dev = (np.array_equal(d_keys[:G].cpu().numpy().view(np.uint64), keys)
                  and np.array_equal(d_grp.cpu().numpy().view(np.uint64), grp_off)
                  and np.array_equal(d_moff[:G + 1].cpu().numpy().view(np.uint64), mem_off)
                  and np.array_equal(d_mem[:E].cpu().numpy().view(np.uint64), mem)
                  and tuple(d_sizes.cpu().numpy()) == (G, E))
        # the restatement's groups against the library's, parent by parent
        k = len(samp)
        g_end = int(grp_off[k])
        ok_or = (ng_o == g_end and np.array_equal(skeys[:ng_o], keys[:g_end])
                 and np.array_equal(sgrp[:k + 1], grp_off[:k + 1])
                 and np.array_equal(smoff[:ng_o + 1], mem_off[:g_end + 1])
                 and np.array_equal(smem[:int(smoff[ng_o])], mem[:int(mem_off[g_end])]))
        cfg = (f"{name}: {npar} parent(s) ({pv} parent values), {nrows} source rows, {m} row values over {dest.size} "
               f"destinations; {E} restricted edges in {G} groups")
        legs = [("device form, resident, members", ms_mem, ok_dev and ok_or, "dgx_dev_groupby_uid, CUDA events"),
                ("device form, resident, counts only", ms_cnt, ok_cnt and ok_or, "dgx_dev_groupby_uid, CUDA events"),
                ("host form, members", t_host, ok_or, "dgx_groupby_uid, wall clock, mean of 3 after one warm call"),
                (f"restatement, 1 thread (C, not Go){'' if name == 'C13a' else f', {k} parents'}", t_or, ok_or,
                 "tests/groupby_oracle.c, wall clock, one call" + ("" if name == "C13a" else
                                                                   f"; per parent {t_or / k:.1f} ms"))]
        for leg, ms, ok, how in legs:
            out_rows.append({"op": "GroupByUid", "workload": name, "leg": leg, "config": cfg, "ms": round(ms, 4),
                             "edges": E, "groups": G, "check": bool(ok), "timing": how})
            print(json.dumps(out_rows[-1]), flush=True)
    return out_rows


def _p_(a):
    return a.ctypes.data_as(C.c_void_p)


def c14_rows(L):
    """C14 "@recurse, loop: false": Zipf graphs of tests/gen_recurse.py (friend out-degree mean 8, follow mean 2, the
    popular targets the hubs), the per-level uid matrices precomputed on the host (gen_recurse.plan_levels) so the legs
    time the filter steps, not the row reads.  C14a: { friend }, depth 6 from 100 roots over 2e6 nodes.  C14b:
    { friend follow }, depth 5 from 100 roots over 2e5 nodes: many small sgs, the per-call cost.  C14c: { friend } over
    2e6 nodes until the default 1e6-edge limit stops it.  Legs, each a whole recursion with fresh sets: (1) the device
    form on resident inputs (CUDA events, one wait at the end), (2) the host form (wall clock), (3) the line-by-line
    restatement (tests/recurse_oracle.c) on 1 thread -- C with a hash set, not Go.  Every leg's rows and DestUIDs are
    checked against the plan."""
    import gen_recurse as gr
    import recurse_oracle as ro
    from dgraph_b200 import algo

    lib = L.lib
    big = gr.c14_graph(np.random.default_rng(14))
    small = gr.c14_graph(np.random.default_rng(15), 200_000)
    roots = np.random.default_rng(2).integers(1, 2_000_001, 100)
    cases = [("C14a", {"friend": big["friend"]}, ["friend"], 6, None, roots),
             ("C14b", small, ["friend", "follow"], 5, None, roots % 200_000 + 1),
             ("C14c", {"friend": big["friend"]}, ["friend"], 64, 10 ** 6, roots)]
    out_rows = []

    def dp(t):
        return C.c_void_p(t.data_ptr())

    def up(x):
        return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(DEV)

    for name, graph, preds, depth, limit, rts in cases:
        steps, total, err = gr.plan_levels(graph, rts, preds, depth, limit)
        vals = sum(s[2].size for s in steps)
        # (1) device form: inputs and outputs resident, one output buffer per step
        dev_in = [(up(s[1]), up(s[2]) if s[2].size else up(np.zeros(1, np.uint64)), up(s[3])) for s in steps]
        dev_out = [tuple(torch.empty(max(s[2].size, 1), dtype=torch.int64, device=DEV) for _ in range(2)) +
                   (torch.empty(s[1].size + 1, dtype=torch.int64, device=DEV),
                    torch.empty(2, dtype=torch.int64, device=DEV)) for s in steps]
        holder = {}

        def dev():
            sets = {p: algo.ReachSet() for p in preds}
            for s, (ds, dv, doff), (do, dd, doo, dz) in zip(steps, dev_in, dev_out):
                _lib.check(lib.dgx_dev_recurse_filter(L.h, sets[s[0]].handle, dp(ds), s[1].size, dp(dv), dp(doff),
                                                      s[2].size, None, 0, dp(do), dp(doo), s[2].size, dp(dd),
                                                      s[2].size, dp(dz)))
            for st in sets.values():
                st.size()  # waits for the queued steps
            holder["sets"] = sets
        ms_dev, _ = timeit(dev, warm=1, reps=3)
        L.sync()
        ok_dev = True
        for s, (do, dd, doo, dz) in zip(steps, dev_out):
            k, d = (int(x) for x in dz.cpu().numpy())
            ok_dev &= (k == s[7] and d == s[6].size and np.array_equal(doo.cpu().numpy().view(np.uint64), s[5])
                       and np.array_equal(do[:k].cpu().numpy().view(np.uint64), s[4])
                       and np.array_equal(dd[:d].cpu().numpy().view(np.uint64), s[6]))
        ok_dev &= sum(st.size() for st in holder["sets"].values()) == total
        for st in holder["sets"].values():
            st.close()
        # (2) host form
        bufs = [(np.empty(max(s[2].size, 1), np.uint64), np.empty(s[1].size + 1, np.uint64),
                 np.empty(max(s[2].size, 1), np.uint64)) for s in steps]
        lens = [C.c_size_t() for _ in steps]

        def host():
            sets = {p: algo.ReachSet() for p in preds}
            for s, (o, oo, dd), n in zip(steps, bufs, lens):
                v = s[2] if s[2].size else np.zeros(1, np.uint64)
                _lib.check(lib.dgx_recurse_filter(sets[s[0]].handle, _p_(s[1]), s[1].size, _p_(v), _p_(s[3]), None, 0,
                                                  _p_(o), _p_(oo), s[2].size, _p_(dd), s[2].size, C.byref(n)))
            for st in sets.values():
                st.close()
        host()
        t0 = time.perf_counter()
        host()
        t_host = (time.perf_counter() - t0) * 1e3
        ok_host = all(np.array_equal(oo, s[5]) and np.array_equal(o[:s[7]], s[4]) and n.value == s[6].size
                      and np.array_equal(dd[:n.value], s[6]) for s, (o, oo, dd), n in zip(steps, bufs, lens))
        # (3) the restatement, 1 thread
        attr_id = {p: i + 1 for i, p in enumerate(preds)}
        obufs = [(np.empty(max(s[2].size, 1), np.uint64), np.empty(s[1].size + 1, np.uint64),
                  np.empty(max(s[2].size, 1), np.uint64)) for s in steps]
        reach = ro.Reach()
        olens = [C.c_size_t() for _ in steps]
        t0 = time.perf_counter()
        kept_or = []
        for s, (o, oo, dd), n in zip(steps, obufs, olens):
            v = s[2] if s[2].size else np.zeros(1, np.uint64)
            kept_or.append(ro.lib().orc_recurse_sg(reach._h, attr_id[s[0]], s[1].ctypes.data, s[1].size, v.ctypes.data,
                                                   s[3].ctypes.data, 0, None, 0, 0, o.ctypes.data, oo.ctypes.data,
                                                   dd.ctypes.data, C.byref(n)))
        t_or = (time.perf_counter() - t0) * 1e3
        reach.close()
        ok_or = all(k == s[7] and np.array_equal(oo, s[5]) and np.array_equal(dd[:n.value], s[6])
                    for s, (o, oo, dd), n, k in zip(steps, obufs, olens, kept_or))
        cfg = (f"{name}: {'{ ' + ' '.join(preds) + ' }'}, {len(steps)} sg steps, {vals} row values, {total} kept edges"
               f"{', stopped by the edge limit' if err else ''}")
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev, "dgx_dev_recurse_filter, CUDA events, "
                                     "median of 3 after one warm recursion"),
                                    ("host form", t_host, ok_host, "dgx_recurse_filter, wall clock, one recursion after "
                                     "one warm recursion"),
                                    ("restatement, 1 thread (C, not Go)", t_or, ok_or, "orc_recurse_sg, wall clock")):
            out_rows.append({"op": "RecurseFilter", "workload": name, "leg": leg, "config": cfg, "ms": round(ms, 4),
                             "steps": len(steps), "values": vals, "kept": total, "check": bool(ok), "timing": timing})
            print(json.dumps(out_rows[-1]), flush=True)
        del dev_in, dev_out
    return out_rows


def c17_rows(L):
    """C17 "value variables": transformTo over a path and evalLevelAgg per row.  C17a: query-039's shape, math(1.0) and
    math(1) carried 3 levels from 1e4 roots over C14's 2e6-node Zipf friend graph (tests/gen_recurse.py c14_graph).
    C17b: min / max / sum / avg over C13's matrix (tests/gen_groupby.py c13_rows, 1e6 rows) with int and float maps
    over 90% of the destinations, and the same matrix as one propagation level, whose most popular destination is a
    hub.  C17c: a path of TestLevelBasedFacetVarSum2's size (2 levels, a handful of uids): latency-bound.  Legs: (1) the
    device form on resident inputs (CUDA events), (2) the host form (wall clock), (3) the line-by-line restatement
    (tests/valvar_oracle.c) on 1 thread -- C with hash maps, not Go.  Every leg is checked bit for bit against the
    restatement."""
    import gen_groupby as gg
    import gen_recurse as gr
    import valvar_oracle as vo

    lib = L.lib
    U64 = np.uint64

    def dp(t):
        return t.data_ptr()

    def up(x):
        x = np.concatenate([np.ascontiguousarray(x, U64), np.zeros(1, U64)])
        return torch.from_numpy(x.view(np.int64)).to(DEV)

    friend = gr.c14_graph(np.random.default_rng(14))["friend"]
    roots = np.unique(np.random.default_rng(17).integers(1, 2_000_001, 10_000).astype(U64))
    path_a, src = [], roots
    for _ in range(3):
        v, off = friend.csr(src)
        dest = np.unique(v)
        path_a.append((src, v, off, dest))
        src = dest
    csrc, cv, coff, cdest = gg.c13_rows(np.random.default_rng(13))
    indeg = int(np.bincount(np.searchsorted(cdest, cv)).max())
    path_c = [(np.array([1, 2, 3], U64), np.array([4, 5, 5, 6], U64), np.array([0, 2, 3, 4], U64),
               np.array([4, 5, 6], U64)),
              (np.array([4, 5, 6], U64), np.array([7, 7, 8], U64), np.array([0, 1, 2, 3], U64), np.array([7, 8], U64))]
    rng = np.random.default_rng(18)
    cases = []
    for typ, vals in (("float", np.ones(roots.size)), ("int", np.ones(roots.size, np.int64))):
        cases.append(("C17a", f"math(1{'.0' if typ == 'float' else ''}) over 3 friend levels from {roots.size} roots",
                      "propagate", roots, vals, path_a))
    for typ in ("int", "float"):
        mk = np.sort(rng.choice(cdest, int(cdest.size * 0.9), replace=False))
        mv = rng.integers(-1000, 1000, mk.size) if typ == "int" else rng.normal(0, 1e3, mk.size)
        for fn in ("min", "max", "sum", "avg"):
            cases.append(("C17b", f"{fn}(val(x)) over C13's matrix, {typ} map over 90% of dest", fn, mk, mv,
                          [(csrc, cv, coff, cdest)]))
        pk = np.sort(rng.choice(csrc, int(csrc.size * 0.9), replace=False))
        pv = rng.integers(-1000, 1000, pk.size) if typ == "int" else rng.normal(0, 1e3, pk.size)
        cases.append(("C17b", f"C13's matrix as one propagation level (hub of {indeg} in-edges), {typ} map over 90% "
                      "of src", "propagate", pk, pv, [(csrc, cv, coff, cdest)]))
    for typ, vals in (("float", np.array([0.1, 0.2, 0.3])), ("int", np.array([1, 2, 3], np.int64))):
        cases.append(("C17c", f"TestLevelBasedFacetVarSum2's size: 2 levels, {typ} map", "propagate",
                      np.array([1, 2, 3], U64), vals, path_c))
    out_rows = []
    for name, cfg, op, keys, vals, levels in cases:
        keys = np.ascontiguousarray(keys, U64)
        vals = np.ascontiguousarray(vals)
        typ = 2 if vals.dtype == np.float64 else 1
        w = vals.view(U64)
        values = sum(int(lv[2][-1]) for lv in levels)
        t0 = time.perf_counter()
        if op == "propagate":
            want = vo.propagate_csr(keys, vals, [lv[:3] for lv in levels])
        else:
            s_, v_, o_, _ = levels[0]
            want = vo.level_agg_csr(op, keys, vals, s_, v_, o_)
        t_or = (time.perf_counter() - t0) * 1e3
        cap = levels[-1][3].size if op == "propagate" else levels[0][0].size
        want_w = np.asarray(want[1]).view(U64)
        # (1) device form, inputs and outputs resident
        dk, dv = up(keys), up(w)
        dlv = [[up(x) for x in lv] for lv in levels]
        ok_t, ov_t = (torch.empty(cap + 1, dtype=torch.int64, device=DEV) for _ in range(2))
        dn = torch.empty(1, dtype=torch.int64, device=DEV)
        if op == "propagate":
            arr = (_lib.VarLevel * len(levels))()
            for i, (lv, t) in enumerate(zip(levels, dlv)):
                arr[i] = _lib.VarLevel(dp(t[0]), dp(t[2]), dp(t[1]), dp(t[3]), lv[2].size - 1, int(lv[2][-1]),
                                       lv[3].size)

            def dev():
                _lib.check(lib.dgx_dev_var_propagate(L.h, typ, dp(dk), dp(dv), keys.size, arr, len(levels), dp(ok_t),
                                                     dp(ov_t), cap, dp(dn)))
        else:
            t = dlv[0]

            def dev():
                _lib.check(lib.dgx_dev_var_level_agg(L.h, typ, vo.AGG[op], dp(dk), dp(dv), keys.size, dp(t[0]),
                                                     levels[0][0].size, dp(t[2]), dp(t[1]), int(levels[0][2][-1]),
                                                     dp(ok_t), dp(ov_t), cap, dp(dn)))
        ms_dev, _ = timeit(dev, warm=2, reps=10)
        L.sync()
        n = int(dn.cpu().numpy()[0])
        ok_dev = (n == want[0].size and np.array_equal(ok_t[:n].cpu().numpy().view(U64), want[0]) and
                  np.array_equal(ov_t[:n].cpu().numpy().view(U64), want_w))
        # (2) host form
        hk, hv, hn = np.empty(max(cap, 1), U64), np.empty(max(cap, 1), U64), C.c_size_t(0)
        if op == "propagate":
            harr = (_lib.VarLevel * len(levels))()
            hkeep = [[np.concatenate([np.ascontiguousarray(x, U64), np.zeros(1, U64)]) for x in lv] for lv in levels]
            for i, (lv, h) in enumerate(zip(levels, hkeep)):
                harr[i] = _lib.VarLevel(h[0].ctypes.data, h[2].ctypes.data, h[1].ctypes.data, h[3].ctypes.data,
                                        lv[2].size - 1, 0, lv[3].size)

            def host():
                _lib.check(lib.dgx_var_propagate(typ, keys.ctypes.data, w.ctypes.data, keys.size, harr, len(levels),
                                                 hk.ctypes.data, hv.ctypes.data, cap, C.byref(hn)))
        else:
            s_, v_, o_, _ = (np.ascontiguousarray(x, U64) for x in levels[0])

            def host():
                _lib.check(lib.dgx_var_level_agg(typ, vo.AGG[op], keys.ctypes.data, w.ctypes.data, keys.size,
                                                 s_.ctypes.data, s_.size, o_.ctypes.data, v_.ctypes.data,
                                                 hk.ctypes.data, hv.ctypes.data, cap, C.byref(hn)))
        host()
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            host()
            ts.append((time.perf_counter() - t0) * 1e3)
        t_host = float(np.median(ts))
        m = hn.value
        ok_host = m == want[0].size and np.array_equal(hk[:m], want[0]) and np.array_equal(hv[:m], want_w)
        full = f"{name}: {cfg}; {len(levels)} level(s), {values} row values, map {keys.size}, result {want[0].size}"
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev, "CUDA events, median of 10 after 2 warm"),
                                    ("host form", t_host, ok_host, "wall clock, median of 3 after 1 warm"),
                                    ("restatement, 1 thread (C, not Go)", t_or, True, "orc_propagate / orc_level_agg, "
                                     "wall clock, one run; the reference the other legs are checked against")):
            out_rows.append({"op": "PropagateVar" if op == "propagate" else f"LevelAgg({op})", "workload": name,
                             "leg": leg, "config": full, "ms": round(ms, 4), "values": values,
                             "max_in_degree": indeg if name == "C17b" else None, "check": bool(ok), "timing": timing})
            print(json.dumps(out_rows[-1]), flush=True)
        del dk, dv, dlv, ok_t, ov_t
    return out_rows


def c18_rows(L):
    """C18 "math() over value variables".  C18a: math(p * 2 + a / s) over a float map p of 1.78e7 keys (C17a's row
    values as a map size), an int age map a over half as many keys and s a {0: v} aggregate.  C18b: a 25-node tree of
    arithmetic, comparisons and cond over three maps sharing 1e7 keys (shared keys: no comparison meets a missing
    entry, so nothing is refused).  C18c: TestMathCeil2's size, a handful of keys (launch-bound).  Legs: (1) the device
    form on resident inputs (CUDA events), (2) the host form (wall clock), (3) the line-by-line restatement
    (tests/math_oracle.c) on 1 thread -- C, not Go.  Every leg is checked against the restatement in keys, words and
    tags."""
    import math_oracle as mo
    from dgraph_b200 import algo

    lib = L.lib
    rng = np.random.default_rng(18)
    U64 = np.uint64

    def dp(t):
        return t.data_ptr()

    def up(x):
        x = np.concatenate([np.ascontiguousarray(x, U64), np.zeros(1, U64)])
        return torch.from_numpy(x.view(np.int64)).to(DEV)

    def keys(n, span):
        return np.sort(rng.choice(np.arange(1, span, dtype=U64), n, replace=False))

    na = 17_800_000
    pk, ak = keys(na, 3 * na), keys(na // 2, 3 * na)
    c18a = ({"p": (pk, rng.random(na) * 100), "a": (ak, rng.integers(1, 90, ak.size)),
             "s": (np.zeros(1, U64), np.array([3.0]))},
            ("+", ("*", ("var", "p"), ("const", 2)), ("/", ("var", "a"), ("var", "s"))))
    nb = 10_000_000
    kb = keys(nb, 2 * nb)
    x, y, z = ("var", "x"), ("var", "y"), ("var", "z")
    tb = ("cond", ("<", ("+", x, ("*", y, ("const", 0.5))), ("-", z, ("const", 3))),
          ("max", ("floor", ("/", x, ("const", 7))), ("sqrt", ("+", y, ("const", 1)))),
          ("cond", (">=", z, x), ("min", ("%", x, ("const", 13)), y), ("u-", z)))
    c18b = ({"x": (kb, rng.integers(0, 1000, nb)), "y": (kb, rng.random(nb) * 500), "z": (kb, rng.integers(0, 1000, nb))},
            tb)
    kc = np.array([1, 23, 24, 25, 31], U64)
    c18c = ({"a": (kc, np.array([38, 15, 15, 17, 19], np.int64))}, ("ceil", ("/", ("var", "a"), ("const", 2.5))))
    out_rows = []
    for name, (maps, tree) in (("C18a", c18a), ("C18b", c18b), ("C18c", c18c)):
        t0 = time.perf_counter()
        want = mo.evaluate(tree, maps)
        t_or = (time.perf_counter() - t0) * 1e3
        assert want[0] == "map" and not want[4]
        names = {}
        prog = algo.math_program(tree, names)
        leaves = [None] * len(names)
        for nm, j in names.items():
            leaves[j] = algo.math_leaf_arrays(maps[nm])
        cap = 1 + sum(k.size for k, *_ in leaves)
        nodes = (_lib.MathNode * len(prog))(*prog)
        # (1) device form, inputs and outputs resident
        dleaf = [(up(k), up(w)) for k, w, *_ in leaves]
        arr = (_lib.MathLeaf * len(leaves))()
        for j, ((k, w, t, typ, nil), (dk, dw)) in enumerate(zip(leaves, dleaf)):
            arr[j] = _lib.MathLeaf(dp(dk), dp(dw), None, None, k.size, typ, nil)
        ok_t, ow_t = (torch.empty(cap, dtype=torch.int64, device=DEV) for _ in range(2))
        ot_t = torch.empty(cap, dtype=torch.uint8, device=DEV)
        di = torch.empty(1, dtype=torch.int64, device=DEV)

        def dev():
            _lib.check(lib.dgx_dev_math_eval(L.h, nodes, len(prog), arr, len(leaves), None, 0, dp(ok_t), dp(ow_t),
                                             dp(ot_t), cap, dp(di)))
        ms_dev, _ = timeit(dev, warm=2, reps=10)
        L.sync()
        n = int(di.cpu().numpy()[0]) & 0xFFFFFFFF
        ok_dev = (n == want[1].size and np.array_equal(ok_t[:n].cpu().numpy().view(U64), want[1]) and
                  np.array_equal(ow_t[:n].cpu().numpy().view(U64), want[2]) and
                  np.array_equal(ot_t[:n].cpu().numpy(), want[3]))
        # (2) host form
        algo.EvalMath(tree, maps)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            got = algo.EvalMath(tree, maps)
            ts.append((time.perf_counter() - t0) * 1e3)
        ok_host = got[0] == want[0] and all(np.array_equal(a, b) for a, b in zip(got[1:], want[1:4]))
        full = (f"{name}: {len(prog)} nodes over {len(leaves)} maps of {', '.join(str(k.size) for k, *_ in leaves)} "
                f"keys; result {want[1].size} entries")
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev, "CUDA events, median of 10 after 2 warm"),
                                    ("host form", float(np.median(ts)), ok_host, "wall clock, median of 3 after 1 warm"),
                                    ("restatement, 1 thread (C, not Go)", t_or, True, "orc_math, wall clock, one run; "
                                     "the reference the other legs are checked against")):
            out_rows.append({"op": "EvalMath", "workload": name, "leg": leg, "config": full, "ms": round(ms, 4),
                             "keys": int(cap - 1), "check": bool(ok), "timing": timing})
            print(json.dumps(out_rows[-1]), flush=True)
        del dleaf, ok_t, ow_t, ot_t
    return out_rows


def c19_rows(L):
    """C19 "@filter and first / offset".  C19a: 10 000 parent rows of about 1e7 values over 1.2e7 uids, D0 of about
    3e6, the 7-node tree AND(COUNT gt 1, OR(LIST 1e5, LIST 1e6), NOT(LIST 5e5)), first: 10.  C19b: C19a in counts-only
    mode (count(friend @filter(...))).  C19c: TestToFastJSONFilterOrFirst's size (launch-bound).  Legs: (1) the device
    form on resident inputs (CUDA events), (2) the host form with its copies (wall clock), (3) the line-by-line
    restatement (tests/sg_filter_oracle.c) on 1 thread -- C, not Go.  Every leg is checked against the restatement."""
    import gen_sg_filter as gs
    import sg_filter_oracle as so
    from dgraph_b200 import algo

    lib = L.lib
    U64 = np.uint64

    def dp(t):
        return t.data_ptr()

    def up(x, dt=U64):
        x = np.concatenate([np.ascontiguousarray(x, dt), np.zeros(1, dt)])
        return torch.from_numpy(x.view(np.int64 if dt == U64 else np.int32)).to(DEV)

    big = gs.big_case(np.random.default_rng(19), nrows=10_000, nvals=10_000_000, n0=3_000_000)
    small = (("or", [0, 1, 2]), [("list", [31]), ("list", [24]), ("list", [25])], [23, 24, 25, 31, 101],
             [np.array([23, 24, 25, 31, 101], U64)], 2, 0)
    out_rows = []
    for name, case, co in (("C19a", big, False), ("C19b", big, True), ("C19c", small, False)):
        tree, leaves, d0, rows, count, offset = case
        t0 = time.perf_counter()
        want = so.sg_filter(*case)
        t_or = (time.perf_counter() - t0) * 1e3
        d0 = np.asarray(d0, U64)
        off = np.zeros(len(rows) + 1, U64)
        np.cumsum([len(r) for r in rows], out=off[1:])
        v = np.concatenate([np.asarray(r, U64) for r in rows])
        f = algo.sg_filter_flat(tree)
        t = algo.sg_filter_tree(f)
        dleaf, descs = [], []
        for lf in leaves:
            if lf[0] == "list":
                d = up(lf[1])
                descs.append(_lib.SgFilterLeaf(0, 0, 0, dp(d), len(lf[1]), None, None, None))
            else:
                d = up(lf[3], np.uint32)
                descs.append(_lib.SgFilterLeaf(1, algo.SGF_CMP[lf[1]], int(lf[2]), None, 0, None, dp(d), None))
            dleaf.append(d)
        tab = (_lib.SgFilterLeaf * len(descs))(*descs)
        d_d0, d_v, d_off = up(d0), up(v), up(off)
        n0, nrows, m = d0.size, len(rows), v.size
        d_dest, d_len = torch.empty(n0 + 1, dtype=torch.int64, device=DEV), torch.empty(1, dtype=torch.int64,
                                                                                         device=DEV)
        d_out = None if co else torch.empty(m + 1, dtype=torch.int64, device=DEV)
        d_oo, d_c = torch.empty(nrows + 1, dtype=torch.int64, device=DEV), torch.empty(nrows + 1, dtype=torch.int32,
                                                                                        device=DEV)

        def dev():
            _lib.check(lib.dgx_dev_sg_filter(L.h, C.byref(t), tab, len(descs), dp(d_d0), n0, None, dp(d_v), dp(d_off),
                                             nrows, m, count, offset, dp(d_dest), n0, dp(d_len),
                                             None if co else dp(d_out), dp(d_oo), m, dp(d_c)))
        ms_dev, _ = timeit(dev, warm=2, reps=10)
        L.sync()
        D = int(d_len.cpu().numpy()[0])
        oo = d_oo.cpu().numpy().view(U64)
        ok_dev = (np.array_equal(d_dest[:D].cpu().numpy().view(U64), want[2]) and
                  np.array_equal(d_c[:nrows].cpu().numpy().view(np.uint32), want[1]) and
                  int(oo[nrows]) == int(want[1].sum()))
        if not co:
            ok_dev = ok_dev and np.array_equal(d_out[:int(oo[nrows])].cpu().numpy().view(U64),
                                               np.concatenate(want[0] + [np.zeros(0, U64)]))
        algo.SubgraphFilter(*case[:4], count=count, offset=offset, counts_only=co)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            got = algo.SubgraphFilter(*case[:4], count=count, offset=offset, counts_only=co)
            ts.append((time.perf_counter() - t0) * 1e3)
        ok_host = (np.array_equal(got[1], want[1]) and np.array_equal(got[2].Uids, want[2]) and
                   (co or all(np.array_equal(a, b) for a, b in zip(got[0], want[0]))))
        full = (f"{name}: {nrows} rows of {m} values, |D0| {n0}, {f['nnodes']} tree nodes over {len(leaves)} leaves "
                f"({', '.join(str(len(lf[1])) if lf[0] == 'list' else 'COUNT' for lf in leaves)}), first {count}"
                f"{', counts only' if co else ''}; new dest {want[2].size}, kept values {int(want[1].sum())}")
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev, "CUDA events, median of 10 after 2 warm"),
                                    ("host form", float(np.median(ts)), ok_host, "wall clock, median of 3 after 1 warm"),
                                    ("restatement, 1 thread (C, not Go)", t_or, True, "orc_sg_filter, wall clock, one "
                                     "run; the reference the other legs are checked against")):
            out_rows.append({"op": "SubgraphFilter", "workload": name, "leg": leg, "config": full, "ms": round(ms, 4),
                             "values": int(m), "check": bool(ok), "timing": timing})
            print(json.dumps(out_rows[-1]), flush=True)
        del dleaf, d_d0, d_v, d_off, d_dest, d_out, d_oo, d_c
    return out_rows


def c20_rows(L):
    """C20 "orderasc / orderdesc by a value variable".  C20a: C19a's matrix shape (10 000 rows, about 1e7 values over
    1.2e7 uids), dest every row value but 3 %, an int map over about 90 % of dest with values in 0..99 (nearly every row
    tier 2), orderdesc, first: 10.  C20b: the same matrix with a distinct-valued float map (every row tier 1).  C20c:
    the root shape, one row of 3e6 uids: (i) distinct floats, orderdesc, first: 100; (ii) ints in 0..99, so one CTA's
    pdqsort carries the call.  C20d: TestQueryVarValAggMul's size (launch-bound).  Legs: (1) the device form on
    resident inputs (CUDA events), (2) the host form with its copies (wall clock), (3) the line-by-line restatement
    (tests/var_order_oracle.c) on 1 thread -- C, not Go.  Every leg is checked against the restatement."""
    import var_order_oracle as vo
    from dgraph_b200 import algo

    lib = L.lib
    U64 = np.uint64
    rng = np.random.default_rng(20)

    def dp(t):
        return t.data_ptr()

    def up(x, dt=U64):
        x = np.concatenate([np.ascontiguousarray(x, dt), np.zeros(1, dt)])
        return torch.from_numpy(x.view(np.int64) if dt == U64 else x).to(DEV)

    N = 12_000_000
    lens = rng.integers(500, 1500, 10_000)
    big_rows = [np.unique(rng.integers(1, N + 1, int(k)).astype(U64)) for k in lens]
    allv = np.unique(np.concatenate(big_rows))
    big_dest = allv[rng.random(allv.size) < 0.97]
    mk = big_dest[rng.random(big_dest.size) < 0.9]
    tied = (mk, rng.integers(0, 100, mk.size).astype(np.int64))
    distinct = (mk, rng.permutation(mk.size).astype(np.float64) * 0.5 - 1e6)
    root = np.sort(rng.choice(np.arange(1, 4_000_001, dtype=U64), 3_000_000, replace=False))
    r_distinct = (root, rng.permutation(root.size).astype(np.float64) + 0.25)
    r_tied = (root, rng.integers(0, 100, root.size).astype(np.int64))
    fr = np.array([23, 24, 25, 31, 101], U64)
    small = ((fr, np.array([15, 0, 0, 19, 0], np.int64)), True, fr, [fr], 0, 0)
    work = (("C20a", (tied, True, big_dest, big_rows, 10, 0)), ("C20b", (distinct, True, big_dest, big_rows, 10, 0)),
            ("C20c(i)", (r_distinct, True, root, [root], 100, 0)), ("C20c(ii)", (r_tied, False, root, [root], 0, 0)),
            ("C20d", small))
    out_rows = []
    for name, case in work:
        m, desc, dest, rows, count, offset = case
        t0 = time.perf_counter()
        want = vo.var_order(*case)
        t_or = (time.perf_counter() - t0) * 1e3
        off = np.zeros(len(rows) + 1, U64)
        np.cumsum([len(r) for r in rows], out=off[1:])
        v = np.concatenate([np.asarray(r, U64) for r in rows])
        keys, vals = m
        d_k, d_w = up(keys), up(np.ascontiguousarray(vals).view(U64))
        typ = 1 if vals.dtype == np.int64 else 2
        leaf = _lib.MathLeaf(dp(d_k), dp(d_w), None, None, keys.size, typ, 0)
        d_dest, d_v, d_off = up(dest), up(v), up(off)
        nd, nrows, M = dest.size, len(rows), v.size
        d_out = torch.empty(M + 1, dtype=torch.int64, device=DEV)
        d_oo = torch.empty(nrows + 1, dtype=torch.int64, device=DEV)
        d_do = torch.empty(nd + 1, dtype=torch.int64, device=DEV)
        d_len = torch.empty(1, dtype=torch.int64, device=DEV)

        def dev():
            _lib.check(lib.dgx_dev_var_order(L.h, C.byref(leaf), int(desc), dp(d_dest), nd, None, dp(d_v), dp(d_off),
                                             nrows, M, count, offset, dp(d_out), dp(d_oo), M, dp(d_do), nd,
                                             dp(d_len)))
        ms_dev, _ = timeit(dev, warm=2, reps=10)
        L.sync()
        D = int(d_len.cpu().numpy()[0])
        oo = d_oo.cpu().numpy().view(U64)
        K = int(oo[nrows])
        wv = np.concatenate(want[0] + [np.zeros(0, U64)])
        woff = np.zeros(nrows + 1, U64)
        np.cumsum([len(r) for r in want[0]], out=woff[1:])
        ok_dev = (np.array_equal(d_do[:D].cpu().numpy().view(U64), want[1]) and np.array_equal(oo, woff) and
                  np.array_equal(d_out[:K].cpu().numpy().view(U64), wv))
        algo.OrderByVar(*case)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            got = algo.OrderByVar(*case)
            ts.append((time.perf_counter() - t0) * 1e3)
        ok_host = np.array_equal(got[1].Uids, want[1]) and all(np.array_equal(a, b) for a, b in zip(got[0], want[0]))
        full = (f"{name}: {nrows} rows of {M} values, |dest| {nd}, a {'float' if typ == 2 else 'int'} map of "
                f"{keys.size} entries ({np.unique(vals).size} distinct values), {'orderdesc' if desc else 'orderasc'}"
                f"{f', first {count}' if count else ''}; output values {K}, new dest {D}")
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev, "CUDA events, median of 10 after 2 warm"),
                                    ("host form", float(np.median(ts)), ok_host, "wall clock, median of 3 after 1 warm"),
                                    ("restatement, 1 thread (C, not Go)", t_or, True, "orc_var_order, wall clock, one "
                                     "run; the reference the other legs are checked against")):
            out_rows.append({"op": "OrderByVar", "workload": name, "leg": leg, "config": full, "ms": round(ms, 4),
                             "values": int(M), "check": bool(ok), "timing": timing})
            print(json.dumps(out_rows[-1]), flush=True)
        del d_k, d_w, d_dest, d_v, d_off, d_out, d_oo, d_do, d_len
    return out_rows


def c21_rows(L):
    """C21 "match()": handleMatchFunction's candidates tested against a string value column.  C21a: a name-like column
    of 1e7 uids (5-20 bytes, some multi-byte), a UidList of 3e6 of them, "alice" with max 2 (short tier).  C21b: the
    trigram branch, 6 synthetic trigram rows (list leaves) over C21a's column whose union is about 1e6 candidates, an
    8-byte query, max 3.  C21c: 1e5 text values of 1-4 KB, a 40-rune query, max 8: the short tier, where the length
    shortcut decides every pair.  C21e: 1e5 values each up to 30 edits from a 110-rune (120-byte) query, max 20:
    the long tier (warp per pair), every pair decided by the distance.  C21d: TestMatchFuncWithAfterWithValidUid's
    size (launch-bound).  Legs: (1) the device form on resident inputs (CUDA events; the column, candidates or rows
    already on the device), (2) the host form with its copies (wall clock), (3) the line-by-line restatement
    (tests/match_oracle.c) on 1 thread -- C, not Go.  Every leg is checked against the restatement."""
    import gen_match as gm
    import match_cases as mc
    import match_oracle as mo
    from dgraph_b200 import algo

    U64 = np.uint64
    rng = np.random.default_rng(21)

    def up(x, dt=U64):
        x = np.concatenate([np.ascontiguousarray(x, dt), np.zeros(1, dt)])
        return torch.from_numpy(x.view(np.int64) if dt == U64 else x).to(DEV)

    names = gm.name_column(rng, 10_000_000)
    cands = np.sort(rng.choice(names.uid, 3_000_000, replace=False))
    rows = [np.sort(rng.choice(names.uid, 170_000, replace=False)) for _ in range(6)]
    text = gm.text_column(rng, 100_000, 1024, 4096)
    q40 = "the graph caf\u00e9 query node \u20ac index abc edge of a graph"[:40]
    q120 = ("graph query node caf\u00e9 \u20ac edge " * 6).encode()[:120]
    near = gm.text_column(rng, 100_000, 0, 0, base=q120, edits=30)
    g, cols = mc.golden()
    gu, gv = cols["name"]
    small = mc.column(gu, gv)
    ali = np.array(sorted(u for u, (v,) in zip(gu, gv) if b"Ali" in v and u > 0x2710), U64)
    work = [("C21a", names, "alice", 2, cands, []), ("C21b", names, "aliceros", 3, None, rows),
            ("C21c", text, q40, 8, text.uid, []), ("C21e", near, q120, 20, near.uid, []),
            ("C21d", small, "Ali", 5, None, [ali])]
    out_rows = []
    for name, col, query, mx, uids, leaves in work:
        t0 = time.perf_counter()
        want = mo.match(col, query, mx, uids=uids, leaves=leaves)
        t_or = (time.perf_counter() - t0) * 1e3
        dt = [up(col.uid), up(col.val_off), up(col.byte_off), up(col.bytes, np.uint8)]
        dcol = _lib.StrColumn(dt[0].data_ptr(), dt[1].data_ptr(), dt[2].data_ptr(), dt[3].data_ptr(), col.uid.size,
                              int(col.byte_off.size - 1), int(col.byte_off[-1]))
        if uids is not None:
            d_u = up(uids)
            cap = int(uids.size)
            kw = dict(d_uids=d_u.data_ptr(), nuids=cap)
        else:
            lo = np.zeros(len(leaves) + 1, U64)
            np.cumsum([r.size for r in leaves], out=lo[1:])
            d_l = up(np.concatenate(leaves))
            cap = int(lo[-1])
            kw = dict(d_lists=d_l.data_ptr(), list_off=lo)
        d_out = torch.empty(cap + 1, dtype=torch.int64, device=DEV)
        d_len = torch.empty(1, dtype=torch.int64, device=DEV)

        def dev():
            algo.dev_match(L.h, dcol, query, mx, d_out.data_ptr(), cap, d_len.data_ptr(), **kw)
        ms_dev, _ = timeit(dev, warm=2, reps=10)
        L.sync()
        k = int(d_len.cpu().numpy()[0])
        ok_dev = np.array_equal(d_out[:k].cpu().numpy().view(U64), want)
        host_kw = dict(uids=uids) if uids is not None else dict(leaves=leaves)
        algo.MatchFuzzy(col, query, mx, **host_kw)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            got = algo.MatchFuzzy(col, query, mx, **host_kw)
            ts.append((time.perf_counter() - t0) * 1e3)
        ok_host = np.array_equal(got.Uids, want)
        nv = int(col.byte_off.size - 1)
        full = (f"{name}: column of {col.uid.size} uids, {nv} values, {int(col.byte_off[-1])} bytes; "
                f"{'UidList of %d' % cap if uids is not None else '%d trigram rows, %d uids' % (len(leaves), cap)}; "
                f"query of {len(gm.runes(query.encode() if isinstance(query, str) else query))} runes, max {mx}; "
                f"kept {want.size}")
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev, "CUDA events, median of 10 after 2 warm"),
                                    ("host form", float(np.median(ts)), ok_host, "wall clock, median of 3 after 1 warm"),
                                    ("restatement, 1 thread (C, not Go)", t_or, True, "orc_match, wall clock, one run; "
                                     "the reference the other legs are checked against")):
            out_rows.append({"op": "MatchFuzzy", "workload": name, "leg": leg, "config": full, "ms": round(ms, 4),
                             "candidates": cap, "check": bool(ok), "timing": timing})
            print(json.dumps(out_rows[-1]), flush=True)
        del dt, d_out, d_len
    return out_rows


def c23_rows(L):
    """C23 "the compare functions": eq / le / lt / ge / gt / between over a typed value column.  C23a: an int64 column
    of 1e8 uids, a UidList of 2e7, ge keeping about half.  C23b: a float list predicate, 1e7 uids of 1-8 values with
    NaNs mixed in, between.  C23c: C21a's 1e7-uid name column with 3e6 candidates: eq with 1 argument, eq with 1 000
    arguments, and ge.  C23d: ge at root on a float index of 1e7 values in about 1e4 buckets, as the device chain (the
    rows resident -> row 0 filtered by dgx_dev_compare_rows -> dgx_dev_merge_sorted_matrix), beside the same chain
    without the filter.  C23e: TestFilterNonIndexedPredicate's size (launch-bound).  C23f: a UidList of 9 against
    C23a's resident column: the whole-column check every value-column call pays (DESIGN section 3.17).  C23d's legs
    start from the index rows resident on the device; the rows read before them is not timed.  Legs: (1) the
    device form on resident inputs (CUDA events), (2) the host form with its copies (wall clock), (3) the line-by-line
    restatement (tests/compare_oracle.c) on 1 thread -- C, not Go.  Every leg is checked against the restatement.
    Algorithmic bytes: candidates read and written (16 per candidate), each tested value's word or bytes, and the
    column's uid and val_off arrays, which every call reads whole for its checks.  For C23a, C23b and C23c's one-argument
    eq, each kernel's time (torch.profiler, a run of its own) is set against the bytes that kernel must move."""
    import compare_oracle as co
    import gen_match as gm
    from dgraph_b200 import algo

    U64 = np.uint64
    rng = np.random.default_rng(23)

    def kernel_times(fn, reps=5):
        """Mean device time per call of each named kernel, from torch.profiler with CUDA activities."""
        from torch.profiler import ProfilerActivity, profile

        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        t = {}
        for e in prof.key_averages():
            for k in ("fz_lookup_kernel", "scan_u64_kernel", "cmp_pairs_kernel", "cmp_finish_kernel",
                      "compact_kernel", "cmp_rows_kernel", "cmp_place_kernel"):
                if k in e.key:
                    us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    t[k] = t.get(k, 0.0) + us / 1e3 / reps
        return t
    peak, _ = peak_gbs()

    def up(x, dt=U64):
        x = np.concatenate([np.ascontiguousarray(x, dt), np.zeros(1, dt)])
        return torch.from_numpy(x.view(np.int64) if dt == U64 else x.view(np.int32) if dt == np.uint32 else x).to(DEV)

    def dev_col(col):
        keep = []

        def d(a, dt=U64):
            if a is None:
                return None
            t = up(a, dt)
            keep.append(t)
            return t.data_ptr()
        if col.type == algo.VAL_STRING:
            s = col.str
            sc = _lib.StrColumn(d(s.uid), d(s.val_off), d(s.byte_off), d(s.bytes, np.uint8), s.uid.size,
                                int(s.byte_off.size - 1), int(s.byte_off[-1]))
            keep.append(sc)
            return _lib.ValColumn(col.type, None, None, None, None, None, C.pointer(sc), 0, 0), keep
        return _lib.ValColumn(col.type, d(col.uid), d(col.val_off), d(col.word), d(col.nsec, np.uint32), None, None,
                              col.uid.size, int(col.val_off[-1])), keep

    n = 100_000_000
    a_uid = np.arange(1, 2 * n, 2, dtype=U64)
    a_col = algo.ValColumn.from_arrays(algo.VAL_INT64, a_uid, np.arange(n + 1, dtype=U64),
                                       rng.integers(-10 ** 9, 10 ** 9, n).astype(np.int64))
    a_cands = np.sort(rng.choice(a_uid, 20_000_000, replace=False))
    nb = 10_000_000
    b_cnt = rng.integers(1, 9, nb)
    b_words = rng.normal(0, 100, int(b_cnt.sum()))
    b_words[rng.random(b_words.size) < 0.05] = np.nan
    b_off = np.zeros(nb + 1, U64)
    np.cumsum(b_cnt, out=b_off[1:])
    b_uid = np.arange(1, nb + 1, dtype=U64)
    b_col = algo.ValColumn.from_arrays(algo.VAL_FLOAT64, b_uid, b_off, b_words)
    names = gm.name_column(rng, 10_000_000)
    c_col = algo.ValColumn.from_arrays(algo.VAL_STRING, str_col=names)
    c_cands = np.sort(rng.choice(names.uid, 3_000_000, replace=False))
    stored = [bytes(names.bytes[int(names.byte_off[j]):int(names.byte_off[j + 1])])
              for j in rng.integers(0, names.byte_off.size - 1, 1000)]
    e_col = algo.ValColumn(algo.VAL_INT64, np.arange(1, 22), [[int(x)] for x in rng.integers(0, 100, 21)])
    work = [("C23a", a_col, "ge", [0], a_cands), ("C23b", b_col, "between", [-50.0, 50.0], b_uid),
            ("C23c eq 1", c_col, "eq", [b"alice"], c_cands), ("C23c eq 1000", c_col, "eq", stored, c_cands),
            ("C23c ge", c_col, "ge", [b"m"], c_cands), ("C23e", e_col, "ge", [50], np.arange(1, 22, dtype=U64)),
            ("C23f", a_col, "ge", [0], np.sort(rng.choice(a_uid, 9, replace=False)))]
    out_rows = []
    dcols = {}
    for name, col, op, args, cands in work:
        t0 = time.perf_counter()
        want = co.compare_uids(col, op, args, cands)
        t_or = (time.perf_counter() - t0) * 1e3
        if id(col) not in dcols:
            dcols = {id(col): dev_col(col)}
        dcol, _ = dcols[id(col)]
        a = algo.ValArgs(col.type, args)
        nc = int(cands.size)
        d_u = up(cands)
        d_out = torch.empty(nc + 1, dtype=torch.int64, device=DEV)
        d_len = torch.empty(1, dtype=torch.int64, device=DEV)
        d_cnt = torch.empty(nc + 1, dtype=torch.int32, device=DEV)

        def dev():
            algo.dev_compare_uids(L.h, dcol, op, a, d_u.data_ptr(), nc, d_out.data_ptr(), nc, d_len.data_ptr(),
                                  d_counts=d_cnt.data_ptr())
        ms_dev, _ = timeit(dev, warm=2, reps=10)
        L.sync()
        k = int(d_len.cpu().numpy()[0])
        ok_dev = np.array_equal(d_out[:k].cpu().numpy().view(U64), want[0]) and \
            np.array_equal(d_cnt[:nc].cpu().numpy().view(np.uint32), want[1])
        algo.CompareUids(col, op, a, cands)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            got, cnt = algo.CompareUids(col, op, a, cands, counts=True)
            ts.append((time.perf_counter() - t0) * 1e3)
        ok_host = np.array_equal(got.Uids, want[0]) and np.array_equal(cnt, want[1])
        ncol = col.uid.size
        lo = np.searchsorted(col.uid, cands)
        hit = (lo < ncol) & (col.uid[np.minimum(lo, ncol - 1)] == cands)
        pairs = int((col.val_off[lo[hit] + 1] - col.val_off[lo[hit]]).sum())
        vbytes = pairs * 8 if col.type != algo.VAL_STRING else int(
            (col.str.byte_off[col.val_off[lo[hit] + 1].astype(np.int64)] -
             col.str.byte_off[col.val_off[lo[hit]].astype(np.int64)]).sum()) + pairs * 16
        abytes = 16 * nc + vbytes + 16 * ncol
        full = (f"{name}: {op} with {len(args)} argument(s); column of {ncol} uids, {int(col.val_off[-1])} values; "
                f"UidList of {nc}; {pairs} (candidate, value) pairs; kept {want[0].size}")
        kernels = None
        if name in ("C23a", "C23b", "C23c eq 1"):  # each kernel's time and share of peak, in a profiled run of its own
            kt = kernel_times(dev)
            kb = {"fz_lookup_kernel": 16 * ncol + 24 * nc, "scan_u64_kernel": 16 * nc,
                  "cmp_pairs_kernel": vbytes + 20 * nc, "cmp_finish_kernel": 9 * nc,
                  "compact_kernel": 9 * nc + 8 * int(want[0].size)}
            kernels = {k: {"ms": round(kt[k], 4), "algorithmic_bytes": b,
                           "frac_of_hbm_peak": round(b / (kt[k] * 1e-3) / 1e9 / peak, 4)}
                       for k, b in kb.items() if kt.get(k)}
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev, "CUDA events, median of 10 after 2 warm"),
                                    ("host form", float(np.median(ts)), ok_host, "wall clock, median of 3 after 1 warm"),
                                    ("restatement, 1 thread (C, not Go)", t_or, True, "orc_compare_uids, wall clock, "
                                     "one run; the reference the other legs are checked against")):
            r = {"op": "CompareUids", "workload": name, "leg": leg, "config": full, "ms": round(ms, 4),
                 "candidates": nc, "check": bool(ok), "timing": timing}
            if leg.startswith("device"):
                gbs = abytes / (ms * 1e-3) / 1e9
                r.update({"algorithmic_bytes": abytes, "algorithmic_GBps": round(gbs, 1),
                          "frac_of_hbm_peak": round(gbs / peak, 4)})
                if kernels:
                    r["kernels"] = kernels
            out_rows.append(r)
            print(json.dumps(r), flush=True)
        del d_u, d_out, d_len, d_cnt
    dcols.clear()
    # C23d: ge at root on a float index: rows are the buckets int64(f) of 1e7 values, row 0 the bucket of the argument
    nd = 10_000_000
    vals = rng.uniform(0, 10_000, nd)
    d_uid = np.arange(1, nd + 1, dtype=U64)
    d_col = algo.ValColumn.from_arrays(algo.VAL_FLOAT64, d_uid, np.arange(nd + 1, dtype=U64), vals)
    arg = 2500.5
    bk = vals.astype(np.int64)
    order = np.lexsort((d_uid, bk))
    keys, starts = np.unique(bk[order], return_index=True)
    sel = keys >= int(arg)
    rows_v = d_uid[order][starts[sel][0]:]
    off = np.concatenate([starts[sel] - starts[sel][0], [rows_v.size]]).astype(U64)
    nrows = int(sel.sum())
    ra = algo.CompareRowArgs("ge", nrows, 1, True)
    want_rows = co.compare_rows(d_col, "ge", [arg], [rows_v[int(off[r]):int(off[r + 1])] for r in range(nrows)], ra)
    want = np.unique(np.concatenate(want_rows))
    dcol, keep = dev_col(d_col)
    a = algo.ValArgs(algo.VAL_FLOAT64, [arg])
    M = rows_v.size
    dv, doff = up(rows_v), up(off)
    fo, foo = torch.empty(M + 1, dtype=torch.int64, device=DEV), torch.empty(nrows + 1, dtype=torch.int64, device=DEV)
    dest, dlen = torch.empty(M + 1, dtype=torch.int64, device=DEV), torch.empty(1, dtype=torch.int64, device=DEV)
    lib = _lib.load()

    def chain():
        algo.dev_compare_rows(L.h, dcol, "ge", a, dv.data_ptr(), doff.data_ptr(), nrows, M, ra, fo.data_ptr(),
                              foo.data_ptr(), M)
        _lib.check(lib.dgx_dev_merge_sorted_matrix(L.h, fo.data_ptr(), foo.data_ptr(), nrows, M, dest.data_ptr(), M,
                                                   dlen.data_ptr()))

    def merge_only():
        _lib.check(lib.dgx_dev_merge_sorted_matrix(L.h, dv.data_ptr(), doff.data_ptr(), nrows, M, dest.data_ptr(), M,
                                                   dlen.data_ptr()))
    ms_m, _ = timeit(merge_only, warm=2, reps=10)
    L.sync()
    ms_c, _ = timeit(chain, warm=2, reps=10)
    L.sync()
    k = int(dlen.cpu().numpy()[0])
    ok = np.array_equal(dest[:k].cpu().numpy().view(U64), want)
    full = (f"C23d: ge({arg}) at root on a float index of {nd} values in {keys.size} buckets; the {nrows} index rows "
            f"({M} uids) already resident, as the rows read leaves them (the read itself is not timed); row 0 of "
            f"{int(off[1])} filtered; DestUIDs {want.size}")
    for leg, ms, okk in (("device chain: rows -> compare_rows -> merge_sorted_matrix", ms_c, ok),
                         ("device chain without the filter: rows -> merge_sorted_matrix", ms_m, True)):
        r = {"op": "CompareRows", "workload": "C23d", "leg": leg, "config": full, "ms": round(ms, 4), "check": bool(okk),
             "timing": "CUDA events, median of 10 after 2 warm"}
        out_rows.append(r)
        print(json.dumps(r), flush=True)
    return out_rows


def c16_rows(L):
    """C16 "shortest() without weights": searches with Go's exec structure (tests/gen_shortest.py), each level's arrays
    precomputed on the host (gen_shortest.plan) so the legs time the search, not the row reads.  C16a: C14's 2e6-node
    Zipf friend graph, from a random root to a node at the deepest level reached within 6 hops.  C16b: { friend follow }
    over C14b's 2e5-node graph, depth 5 (up to 2^k sgs at level k), to a node at the deepest level reached.  C16c: the
    fixture's TestShortestPath4 search (launch-bound).  C16d: C16a's graph and root with an unreachable To.  Legs, each
    a whole search: (1) the device form on resident inputs (CUDA events, the path read at the end), (2) the host form
    (wall clock), (3) the line-by-line restatement (tests/shortest_oracle.c) on 1 thread -- C, not Go.  Every leg is
    checked against the plan's formula: the device and host forms level by level and by path, the restatement by
    reachability, path length and each level's numEdges."""
    import gen_recurse as gr
    import gen_shortest as gs
    import shortest_oracle as so
    from dgraph_b200 import algo

    lib = L.lib
    big = gr.c14_graph(np.random.default_rng(14))
    small = gr.c14_graph(np.random.default_rng(15), 200_000)

    def graph_of(g, preds):
        return gs.Graph(g[preds[0]].ptr.size - 1, [(g[p].ptr.astype(np.uint64), g[p].idx) for p in preds],
                        [(i, None) for i in range(len(preds))])

    ga, gb = graph_of(big, ["friend"]), graph_of(small, ["friend", "follow"])
    with open(os.path.join(ROOT, "tests", "golden", "shortest_path_follow.json")) as f:
        gc, fc, tc, _ = gs.fixture_case(json.load(f), "TestShortestPath4")
    rng = np.random.default_rng(16)
    root_a, root_b = int(rng.integers(1, 2_000_001)), int(rng.integers(1, 200_001))

    def deepest(g, frm, hops):
        lv, f = gs.plan(g, frm, g.nnodes + 5, hops)
        far = np.flatnonzero(f.level_of == f.level_of.max())
        return int(far[len(far) // 2])

    cases = [("C16a", ga, root_a, deepest(ga, root_a, 6), 6), ("C16b", gb, root_b, deepest(gb, root_b, 5), 5),
             ("C16c", gc, fc, tc, None), ("C16d", ga, root_a, ga.nnodes + 5, 6)]
    out_rows = []

    def dp(t):
        return t.data_ptr()

    def up(x):
        x = np.concatenate([x, np.zeros(1, x.dtype)])
        return torch.from_numpy(x.view(np.int32 if x.dtype == np.uint32 else np.int64)).to(DEV)

    for name, g, frm, to, hops in cases:
        levels, f = gs.plan(g, frm, to, hops)
        want_u, want_a = f.path()
        vals = sum(int(a[4].size) for a, _, _, _ in levels)
        sgs = sum(int(a[0].size) for a, _, _, _ in levels)
        # (1) device form: inputs and outputs resident
        dev_in = [[up(x) for x in a] for a, _, _, _ in levels]
        dev_lv = [_lib.PathLevel(int(a[0].size), *[dp(x) for x in t]) for (a, _, _, _), t in zip(levels, dev_in)]
        dev_out = [(torch.empty(max(int(a[6].size), 1), dtype=torch.int64, device=DEV),
                    torch.empty(int(a[0].size) + 1, dtype=torch.int64, device=DEV),
                    torch.empty(3, dtype=torch.int64, device=DEV)) for a, _, _, _ in levels]
        holder = {}

        def dev():
            with algo.PathSearch(frm, to) as ps:
                for (a, _, _, _), lv, (dn, do, dst) in zip(levels, dev_lv, dev_out):
                    _lib.check(lib.dgx_dev_path_expand(L.h, ps.handle, C.byref(lv), a[2].size, a[4].size, a[6].size,
                                                       dp(dn), dp(do), a[6].size, dp(dst)))
                holder["path"] = ps.path()  # waits for the queued levels
        ms_dev, _ = timeit(dev, warm=1, reps=3)
        L.sync()
        ok_dev = np.array_equal(holder["path"][0], want_u) and np.array_equal(holder["path"][1], want_a)
        for (a, nxt, noff, st), (dn, do, dst) in zip(levels, dev_out):
            k = int(noff[-1])
            ok_dev &= (tuple(int(x) for x in dst.cpu().numpy()) == st and
                       np.array_equal(do.cpu().numpy().view(np.uint64), noff) and
                       np.array_equal(dn[:k].cpu().numpy().view(np.uint64), nxt))
        # (2) host form
        bufs = [(np.empty(max(int(a[6].size), 1), np.uint64), np.empty(int(a[0].size) + 1, np.uint64),
                 _lib.PathStats()) for a, _, _, _ in levels]
        hkeep = [[x if x.size else np.zeros(1, x.dtype) for x in a] for a, _, _, _ in levels]
        host_lv = [_lib.PathLevel(int(a[0].size), *[x.ctypes.data for x in k]) for (a, _, _, _), k in
                   zip(levels, hkeep)]

        def host():
            with algo.PathSearch(frm, to) as ps:
                for (a, _, _, _), lv, (n, no, st) in zip(levels, host_lv, bufs):
                    _lib.check(lib.dgx_path_expand(ps.handle, C.byref(lv), n.ctypes.data, no.ctypes.data, a[6].size,
                                                   C.byref(st)))
                return ps.path()
        host()
        t0 = time.perf_counter()
        hp = host()
        t_host = (time.perf_counter() - t0) * 1e3
        ok_host = np.array_equal(hp[0], want_u) and np.array_equal(hp[1], want_a) and all(
            (st.edges, st.discovered, st.to_level) == w[3] and np.array_equal(no, w[2]) and
            np.array_equal(n[:int(w[2][-1])], w[1]) for w, (n, no, st) in zip(levels, bufs))
        # (3) the restatement, 1 thread
        t0 = time.perf_counter()
        r = so.run(g, frm, to, hops, 0x9E3779B97F4A7C15)
        t_or = (time.perf_counter() - t0) * 1e3
        L_ = f.to_level
        k = len(levels)
        ok_or = ((to in r.dist) == bool(L_) and r.level_edges[:k] == [w[3][0] for w in levels] and
                 (r.levels in (L_, L_ + 1) if L_ else r.levels == k) and len(r.path) == (L_ + 1 if L_ else 0))
        cfg = (f"{name}: {len(g.children)} child(ren), {g.nnodes - 1} nodes, {k} levels, {sgs} sgs, {vals} row "
               f"values, {'To at level ' + str(L_) if L_ else 'To unreachable'}")
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev, "dgx_dev_path_expand per level and "
                                     "dgx_path_result, CUDA events, median of 3 after one warm search"),
                                    ("host form", t_host, ok_host, "dgx_path_expand per level and dgx_path_result, "
                                     "wall clock, one search after one warm search"),
                                    ("restatement, 1 thread (C, not Go)", t_or, ok_or, "orc_shortest including its "
                                     "ProcessGraph restatement, wall clock")):
            out_rows.append({"op": "ShortestPath", "workload": name, "leg": leg, "config": cfg, "ms": round(ms, 4),
                             "levels": k, "sgs": sgs, "values": vals, "to_level": L_, "check": bool(ok),
                             "timing": timing})
            print(json.dumps(out_rows[-1]), flush=True)
        del dev_in, dev_out
    return out_rows


def c15_chain(rng, levels=8, width=64, deg=4):
    """C15b: a narrow chain of `levels` cascaded nodes, each with first: 2, offset: 1, `width` uids a level and about
    `deg` values a row: launch-bound."""
    from dgraph_b200.algo import CC_CASCADE, CC_CHECKED, CascadeNode

    dest = np.arange(1, width + 1, dtype=np.uint64)
    nodes = [CascadeNode(-1, CC_CASCADE, 2, 1, 0, dest, [dest])]
    for k in range(1, levels):
        rows = [np.unique(rng.integers(1, 2 * width, int(rng.integers(0, 2 * deg)))).astype(np.uint64)
                for _ in range(nodes[-1].dest.size)]
        d = np.unique(np.concatenate(rows)).astype(np.uint64)
        nodes.append(CascadeNode(k - 1, CC_CASCADE | CC_CHECKED, 2, 1, 0, d, rows))
    return nodes


def c15_directive():
    """C15c: TestCascadeDirective's tree (query/query0_test.go) on the friend fixture's uids: me(func: uid(0x01))
    @cascade { name gender friend { name friend { name dob age } } } -- a handful of values."""
    from dgraph_b200.algo import CC_CASCADE, CC_CHECKED, CascadeNode

    C2 = CC_CASCADE | CC_CHECKED
    f1 = np.array([23, 24, 25, 31, 101], np.uint64)
    return [CascadeNode(-1, CC_CASCADE, 0, 0, 0, [1], [[1]]),
            CascadeNode(0, C2, 0, 0, 0, [], [], [1]), CascadeNode(0, C2, 0, 0, 0, [], [], [1]),
            CascadeNode(0, C2, 0, 0, 0, f1, [f1]),
            CascadeNode(3, C2, 0, 0, 0, [], [], [1, 1, 1, 1, 0]),
            CascadeNode(3, C2, 0, 0, 0, [1, 24], [[1], [], [], [24], []]),
            CascadeNode(5, C2, 0, 0, 0, [], [], [1, 1]), CascadeNode(5, C2, 0, 0, 0, [], [], [1, 1]),
            CascadeNode(5, C2, 0, 0, 0, [], [], [1, 1])]


def c15_rows(L):
    """C15 "@cascade": C15a, TestCascadeWithPaginationDeep scaled up (tests/gen_cascade.c15a_arrays: 1e6 Person roots,
    friend rows Zipf over 2e6 uids, has_val densities 0.8 and 0.5, first: 2, offset: 1 at the leaf); C15b, a chain 8
    levels deep with pagination at every level (launch-bound); C15c, TestCascadeDirective's tree.  Legs: (1) the device
    form on resident inputs (CUDA events), (2) the host form (wall clock), (3) the line-by-line restatement
    (tests/cascade_oracle.c) on 1 thread -- C, not Go.  Every leg is checked against the restatement."""
    import cascade_oracle as co
    import cascade_plan as cp
    import gen_cascade as gc
    from dgraph_b200.algo import cascade_arrays, cascade_tree

    lib = L.lib

    def up(x, dt=np.uint64):
        x = np.ascontiguousarray(np.asarray(x, dt))
        if x.size == 0:
            x = np.zeros(1, dt)
        return torch.from_numpy(x.view(np.int64) if dt == np.uint64 else x).to(DEV)

    cases = [("C15a", gc.c15a_arrays(np.random.default_rng(15)), 3),
             ("C15b", cascade_arrays(c15_chain(np.random.default_rng(16))), 50),
             ("C15c", cascade_arrays(c15_directive()), 200)]
    out_rows = []
    for name, a, reps in cases:
        n = a["nnodes"]
        m, nd, nr = int(a["v_off"][-1]), int(a["dest_off"][-1]), int(a["row_off"][-1])
        t0 = time.perf_counter()
        want = co.cascade_flat(a)
        t_or = (time.perf_counter() - t0) * 1e3
        ok_or = True  # the restatement is the reference of the other legs
        tree = cascade_tree(a)
        # (1) device form: every node's arrays resident, the outputs resident
        keep, descs = [], []
        for k in range(n):
            r0, r1 = int(a["row_off"][k]), int(a["row_off"][k + 1])
            b0, b1 = int(a["v_off"][r0]), int(a["v_off"][r1])
            dv, doff = up(a["v"][b0:b1]), up(a["v_off"][r0:r1 + 1] - np.uint64(b0))
            dd = up(a["dest"][int(a["dest_off"][k]):int(a["dest_off"][k + 1])])
            dh = up(a["has_val"][int(a["hv_off"][k]):int(a["hv_off"][k + 1])], np.uint8)
            keep += [dv, doff, dd, dh]
            descs.append(_lib.CascadeNode(dv.data_ptr(), doff.data_ptr(), r1 - r0, b1 - b0, dd.data_ptr(),
                                          int(a["dest_off"][k + 1] - a["dest_off"][k]), dh.data_ptr(),
                                          int(a["hv_off"][k + 1] - a["hv_off"][k])))
        tab = (_lib.CascadeNode * n)(*descs)
        d_out, d_oo, d_dout, d_do, d_sz = (torch.empty(x, dtype=torch.int64, device=DEV)
                                           for x in (max(m, 1), nr + 1, max(nd, 1), n + 1, 2))

        def dev():
            _lib.check(lib.dgx_dev_cascade(L.h, C.byref(tree), tab, C.c_void_p(d_out.data_ptr()),
                                           C.c_void_p(d_oo.data_ptr()), m, C.c_void_p(d_dout.data_ptr()),
                                           C.c_void_p(d_do.data_ptr()), nd, C.c_void_p(d_sz.data_ptr())))
        l0 = lib.dgx_lane_launches(L.h)
        dev()
        L.sync()
        launches = lib.dgx_lane_launches(L.h) - l0
        ms_dev, _ = timeit(dev, warm=2, reps=reps)
        L.sync()
        K, D = (int(x) for x in d_sz.cpu().numpy())
        ok_dev = (np.array_equal(d_oo.cpu().numpy().view(np.uint64), want[1]) and
                  np.array_equal(d_do.cpu().numpy().view(np.uint64), want[3]) and
                  np.array_equal(d_out[:K].cpu().numpy().view(np.uint64), want[0][:K]) and
                  np.array_equal(d_dout[:D].cpu().numpy().view(np.uint64), want[2][:D]))
        # (2) host form
        out, oo = np.empty(max(m, 1), np.uint64), np.empty(nr + 1, np.uint64)
        dout, do = np.empty(max(nd, 1), np.uint64), np.empty(n + 1, np.uint64)
        p = {k: a[k].ctypes.data for k in ("v", "v_off", "row_off", "dest", "dest_off", "has_val", "hv_off")}

        def host():
            _lib.check(lib.dgx_cascade(C.byref(tree), p["v"], p["v_off"], p["row_off"], p["dest"], p["dest_off"],
                                       p["has_val"], p["hv_off"], out.ctypes.data, oo.ctypes.data, m,
                                       dout.ctypes.data, do.ctypes.data, nd))
        host()
        hreps = max(1, min(reps, 20))
        t0 = time.perf_counter()
        for _ in range(hreps):
            host()
        t_host = (time.perf_counter() - t0) * 1e3 / hreps
        ok_host = (np.array_equal(oo, want[1]) and np.array_equal(do, want[3]) and
                   np.array_equal(out[:K], want[0][:K]) and np.array_equal(dout[:D], want[2][:D]))
        depth, work = [0] * n, set()
        for k in range(n):
            pk = int(a["parent"][k])
            depth[k] = 0 if pk == 0xFFFFFFFF else depth[pk] + 1
            r0, r1 = int(a["row_off"][k]), int(a["row_off"][k + 1])
            if a["dest_off"][k + 1] > a["dest_off"][k] or a["v_off"][r1] > a["v_off"][r0]:
                work.add(depth[k])
        levels = max(depth) + 1
        ok_launch = launches == cp.launches(len(work))
        cfg = f"{name}: {n} nodes, {levels} levels, {nr} rows, {m} row values, {nd} dest values -> {K} values, {D} dest"
        for leg, ms, ok, timing in (("device form, resident", ms_dev, ok_dev and ok_launch,
                                     f"dgx_dev_cascade, CUDA events, median of {reps} after 2 warm calls"),
                                    ("host form", t_host, ok_host, f"dgx_cascade, wall clock, mean of {hreps} after "
                                     "one warm call"),
                                    ("restatement, 1 thread (C, not Go)", t_or, ok_or, "orc_cascade, wall clock")):
            out_rows.append({"op": "Cascade", "workload": name, "leg": leg, "config": cfg, "ms": round(ms, 4),
                             "values": m, "launches": launches, "check": bool(ok), "timing": timing})
            print(json.dumps(out_rows[-1]), flush=True)
        del keep
    return out_rows



def c24_rows(L):
    """C24 "orderasc / orderdesc by a predicate without its index" (dgx_pred_order).  C24a: 10 000 rows of about 1e7
    values over an int64 column of 1e7 uids with 10 % absent, distinct values (tier 1).  C24b: the same matrix over a
    string column of 10^4 distinct names (tied rows, tier 2 on threads).  C24c: one row of 3e6 uids over datetimes at
    second resolution with 10^5 distinct instants (the CTA tier).  C24d: one row of 3e6 distinct strings sharing their
    first 8 bytes (tier 2 on a CTA, byte comparisons).  C24e: a reference test's size (launch-bound).  Every call pages
    with count 1000, the query layer's default.  Legs: (1) the device form on resident inputs (CUDA events), (2) the
    host form with its copies (wall clock), (3) the line-by-line restatement (tests/pred_order_oracle.c) on 1 thread --
    C, not Go.  Every leg is checked against the restatement."""
    import pred_order_oracle as po
    from dgraph_b200 import algo

    U64 = np.uint64
    rng = np.random.default_rng(24)

    def up(x, dt=U64):
        x = np.concatenate([np.ascontiguousarray(x, dt), np.zeros(1, dt)])
        return torch.from_numpy(x.view(np.int64) if dt == U64 else x.view(np.int32) if dt == np.uint32 else x).to(DEV)

    def dev_col(col):
        keep = []

        def d(a, dt=U64):
            if a is None:
                return None
            t = up(a, dt)
            keep.append(t)
            return t.data_ptr()
        if col.type == algo.VAL_STRING:
            s = col.str
            sc = _lib.StrColumn(d(s.uid), d(s.val_off), d(s.byte_off), d(s.bytes, np.uint8), s.uid.size,
                                int(s.byte_off.size - 1), int(s.byte_off[-1]))
            keep.append(sc)
            return _lib.ValColumn(col.type, None, None, None, None, None, C.pointer(sc), 0, 0), keep
        return _lib.ValColumn(col.type, d(col.uid), d(col.val_off), d(col.word), d(col.nsec, np.uint32), None, None,
                              col.uid.size, int(col.val_off[-1])), keep

    def str_col(uids, width, codes, prefix=b""):
        """A string column of fixed-width values prefix + the decimal code, built as arrays."""
        w = len(prefix) + width
        txt = np.char.zfill(codes.astype(str), width).astype("S%d" % width)
        buf = np.frombuffer(b"".join([prefix + x for x in txt.tolist()]), np.uint8)
        boff = np.arange(uids.size + 1, dtype=U64) * U64(w)
        sc = algo.StrColumn.from_csr(uids, np.arange(uids.size + 1, dtype=U64), boff, buf)
        return algo.ValColumn.from_arrays(algo.VAL_STRING, str_col=sc)

    nu = 10_000_000
    uids = np.arange(1, nu + 1, dtype=U64)
    present = np.sort(uids[rng.random(nu) < 0.9])
    a_col = algo.ValColumn.from_arrays(algo.VAL_INT64, present, np.arange(present.size + 1, dtype=U64),
                                       rng.permutation(present.size).astype(np.int64) * 7 - 10 ** 6)
    rows = []
    for _ in range(10_000):
        k = int(rng.integers(800, 1200))
        s0 = int(rng.integers(0, nu - 4 * k))
        rows.append(uids[s0:s0 + 4 * k:4][:k].copy())
    b_col = str_col(present, 5, rng.integers(0, 10_000, present.size), b"name")
    n3 = 3_000_000
    u3 = np.arange(1, n3 + 1, dtype=U64)
    c_col = algo.ValColumn.from_arrays(algo.VAL_DATETIME, u3, np.arange(n3 + 1, dtype=U64),
                                       (rng.integers(0, 100_000, n3) * 3600 - 10 ** 9).astype(np.int64),
                                       np.zeros(n3, np.uint32))
    d_col = str_col(u3, 9, rng.permutation(n3), b"prefix00")
    e_col = algo.ValColumn(algo.VAL_STRING, [23, 24, 25, 31, 101],
                           [["Zambo Alice"], ["John Alice"], ["Bob Joe"], ["Allan Matt"], ["John Oliver"]])
    e_row = np.array([23, 24, 25, 31, 101], U64)
    work = [("C24a", a_col, False, uids, rows), ("C24b", b_col, False, uids, rows), ("C24c", c_col, True, u3, [u3]),
            ("C24d", d_col, False, u3, [u3]), ("C24e", e_col, False, e_row, [e_row])]
    count, offset = 1000, 0
    out_rows = []
    for name, col, desc, dest, rws in work:
        t0 = time.perf_counter()
        want_rows, want_dest = po.pred_order(col, desc, dest, rws, count, offset)
        t_or = (time.perf_counter() - t0) * 1e3
        dcol, keep = dev_col(col)
        v = np.concatenate(rws)
        v_off = np.zeros(len(rws) + 1, U64)
        np.cumsum([r.size for r in rws], out=v_off[1:])
        nr, m, nd = len(rws), int(v.size), int(dest.size)
        d_d, d_v, d_vo = up(dest), up(v), up(v_off)
        d_out = torch.empty(m + 1, dtype=torch.int64, device=DEV)
        d_off = torch.empty(nr + 1, dtype=torch.int64, device=DEV)
        d_dest = torch.empty(nd + 1, dtype=torch.int64, device=DEV)
        d_len = torch.empty(1, dtype=torch.int64, device=DEV)

        def dev():
            algo.dev_order_by_pred(L.h, dcol, desc, d_d.data_ptr(), nd, d_v.data_ptr(), d_vo.data_ptr(), nr, m,
                                   d_out.data_ptr(), d_off.data_ptr(), m, d_dest.data_ptr(), nd, d_len.data_ptr(),
                                   count, offset)
        ms_dev, _ = timeit(dev, warm=1, reps=5)
        L.sync()
        off = d_off.cpu().numpy().view(U64)
        out = d_out.cpu().numpy().view(U64)
        k = int(d_len.cpu().numpy()[0])
        ok_dev = all(np.array_equal(out[int(off[i]):int(off[i + 1])], want_rows[i]) for i in range(nr)) and \
            np.array_equal(d_dest[:k].cpu().numpy().view(U64), want_dest)
        del keep
        t0 = time.perf_counter()
        h_rows, h_dest = algo.OrderByPred(col, desc, dest, rws, count, offset)
        ms_host = (time.perf_counter() - t0) * 1e3
        ok_host = all(np.array_equal(a, b) for a, b in zip(h_rows, want_rows)) and \
            np.array_equal(h_dest.Uids, want_dest)
        r = {"op": name, "type": int(col.type), "rows": nr, "values": m, "dest": nd, "desc": desc, "count": count,
             "ms_resident": ms_dev, "ms_host_form": ms_host, "ms_restatement_1_thread": t_or,
             "check_resident": bool(ok_dev), "check_host_form": bool(ok_host)}
        if not QUIET:
            print(json.dumps(r), flush=True)
        out_rows.append(r)
    return out_rows


if __name__ == "__main__":
    main()
