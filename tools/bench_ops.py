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
    else:
        rows = run(Lane(), 10 if args.small else 1, quick=False)
    if args.c6_only or args.c7_only or args.c8_only or args.c9_only or args.c10_only:  # the card and its power limit, read in the same run as the numbers
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
        launches = lib.dgx_lane_launches(L.h) - l0
        ms1, _ = timeit(dev, warm=3, reps=reps)
        ok1 = bool(np.array_equal(dev_got(), want))
        overflows = lib.dgx_merge_matrix_overflows(None) - o0
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


if __name__ == "__main__":
    main()
