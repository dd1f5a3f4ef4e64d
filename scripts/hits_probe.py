#!/usr/bin/env python3
"""Times edlibB200FindHits (all end locations within k) on the H100, next to the HW distance call on the same reads.

    python scripts/hits_probe.py [--reads 1000000] [--short 100000] [--repeats 3] [--out results.json]
    python scripts/hits_probe.py --task loc|path [--reads 1000000] [--repeats 3] [--out results.json]

Workloads: config-2 reads (150 bp, 3 % errors, seeded generator of bench.py) over the E. coli genome at k = 3 and 10
(seed route) and, on fewer reads, k = 20 (above the largest seed threshold of a 150 bp read, 17: whole-target sweep);
seeded 23-mers at k = 4 (beyond every seed level's reach: whole-target sweep); and, for comparison, the same read sets
through edlibAlignBatch (HW distance).  Per workload: time per call (host clock around the whole call, median and
spread over the repeats after one warm-up call), per-kernel device times of the last call (edlibB200LastKernelReport),
hits per read, filterDecided / filterFallback.  The card's name and power limit are read in the same run.  Needs a
GPU; prints one JSON document (and writes it to --out when given).

--task loc / path times edlibB200FindHitAlignments instead (start locations / alignment paths of every hit) for the
150 bp reads at k = 3 and 10, next to edlibB200FindHits of the same call (task DISTANCE) and edlibAlignBatch HW LOC /
PATH of the same reads at the same k; the stored scripts' total length is reported for PATH."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from edlib_b200 import workloads  # noqa: E402
from edlib_b200._ffi import AlignResult, HitAlignments, Hits, make_config, product_path  # noqa: E402


class Stats(C.Structure):  # include/edlib_b200.h EdlibB200Stats
    _fields_ = [("kernelMs", C.c_double), ("k1Ms", C.c_double), ("launches", C.c_int), ("filterWindows", C.c_int),
                ("h2dBytes", C.c_longlong), ("d2hBytes", C.c_longlong), ("k1Cells", C.c_longlong), ("wCells", C.c_longlong),
                ("filterDecided", C.c_longlong), ("filterFallback", C.c_longlong)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = "unknown (%s)" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--reads-k20", type=int, default=10_000)  # k = 20 is above every seed level of 150 bp reads
    ap.add_argument("--short", type=int, default=100_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--task", choices=("loc", "path"), default=None,
                    help="time the start locations / paths of every hit instead of the hit lists")
    ap.add_argument("--out", default=None, help="also write the JSON document to this file")
    a = ap.parse_args()
    lib = C.CDLL(product_path())
    if lib.edlibB200Available() != 1:
        sys.exit("no usable CUDA device: this probe measures the GPU only")
    lib.edlibB200FindHits.restype = C.c_int
    lib.edlibB200FindHits.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.c_char_p, C.c_int,
                                      type(make_config()[0]), C.c_int, C.c_longlong, C.POINTER(Hits)]
    lib.edlibB200FreeHits.argtypes = [C.POINTER(Hits)]
    lib.edlibB200FindHitAlignments.restype = C.c_int
    lib.edlibB200FindHitAlignments.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.c_char_p, C.c_int,
                                               type(make_config()[0]), C.c_int, C.c_longlong, C.POINTER(HitAlignments)]
    lib.edlibB200FreeHitAlignments.argtypes = [C.POINTER(HitAlignments)]
    lib.edlibAlignBatch.restype = C.c_int
    lib.edlibAlignBatch.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                                    C.c_int, type(make_config()[0]), C.POINTER(AlignResult)]
    lib.edlibB200FreeResults.argtypes = [C.POINTER(AlignResult), C.c_int]
    lib.edlibB200LastKernelReport.argtypes = [C.c_char_p, C.c_int]
    genome = workloads.ecoli_genome()
    tbytes = genome.tobytes()
    tbuf = C.create_string_buffer(tbytes, len(tbytes))

    def read_set(arr):
        n, m = arr.shape
        bufs = [C.create_string_buffer(arr[i].tobytes(), m) for i in range(n)]
        ptrs = (C.c_char_p * n)(*[C.cast(b, C.c_char_p) for b in bufs])
        lens = (C.c_int * n)(*([m] * n))
        return bufs, ptrs, lens, n

    def last():
        s = Stats()
        lib.edlibB200LastStats(C.byref(s))
        buf = C.create_string_buffer(8192)
        lib.edlibB200LastKernelReport(buf, 8192)
        kernels = {}
        for part in buf.value.decode().split(";"):
            if part:
                name, ms, count = part.split(":")
                kernels[name] = [round(float(ms), 4), int(count)]
        return s, kernels

    def timed(fn):
        fn()  # warm-up
        times = []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            fn()
            times.append((time.perf_counter() - t0) * 1e3)
        times.sort()
        return {"ms_median": round(times[len(times) // 2], 3), "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3)}

    def hits_run(rs, k):
        _, ptrs, lens, n = rs
        cfg, _ = make_config(k, 2, 0)
        info = {}

        def call():
            h = Hits()
            st = lib.edlibB200FindHits(ptrs, lens, n, tbuf, len(tbytes), cfg, 0, 1 << 40, C.byref(h))
            assert st == 0
            info["hits"] = h.offsets[n]
            lib.edlibB200FreeHits(C.byref(h))
        r = timed(call)
        s, kern = last()
        r.update(hits_per_read=round(info["hits"] / n, 3), filterDecided=s.filterDecided, filterFallback=s.filterFallback,
                 filterWindows=s.filterWindows, kernel_ms=round(s.kernelMs, 3), kernels=kern)
        return r

    def alignments_run(rs, k, task):
        _, ptrs, lens, n = rs
        cfg, _ = make_config(k, 2, task)
        info = {}

        def call():
            h = HitAlignments()
            st = lib.edlibB200FindHitAlignments(ptrs, lens, n, tbuf, len(tbytes), cfg, 0, 1 << 40, C.byref(h))
            assert st == 0
            stored = h.hits.offsets[n]
            info["hits"] = stored
            info["script_bytes"] = h.alignmentOffsets[stored] if h.alignmentOffsets else 0
            lib.edlibB200FreeHitAlignments(C.byref(h))
        r = timed(call)
        s, kern = last()
        r.update(hits_per_read=round(info["hits"] / n, 3), filterDecided=s.filterDecided, filterFallback=s.filterFallback,
                 kernel_ms=round(s.kernelMs, 3), kernels=kern)
        if task == 2:
            r["script_bytes"] = info["script_bytes"]
        return r

    def distance_run(rs, k=-1, task=0):
        _, ptrs, lens, n = rs
        cfg, _ = make_config(k, 2, task)
        tptr = (C.c_char_p * n)(*([C.cast(tbuf, C.c_char_p)] * n))
        tlen = (C.c_int * n)(*([len(tbytes)] * n))
        res = (AlignResult * n)()

        def call():
            assert lib.edlibAlignBatch(ptrs, lens, tptr, tlen, n, cfg, res) == 0
            lib.edlibB200FreeResults(res, n)
        r = timed(call)
        s, kern = last()
        r.update(filterDecided=s.filterDecided, filterFallback=s.filterFallback, kernel_ms=round(s.kernelMs, 3), kernels=kern)
        return r

    if a.task:
        task = 1 if a.task == "loc" else 2
        out = {"card": card(), "repeats": a.repeats, "warmup": 1, "reads": a.reads, "task": a.task}
        long_reads = read_set(workloads.reads_of(genome, a.reads, read_len=150, seed=42))
        for k in (3, 10):
            out["hits_%s_150bp_k%d" % (a.task, k)] = alignments_run(long_reads, k, task)
            out["hits_distance_150bp_k%d" % k] = hits_run(long_reads, k)
            out["batch_%s_150bp_k%d" % (a.task, k)] = distance_run(long_reads, k, task)
        out["card_after"] = card()
        text = json.dumps(out, indent=1)
        print(text)
        if a.out:
            with open(a.out, "w") as f:
                f.write(text + "\n")
        return
    out = {"card": card(), "repeats": a.repeats, "warmup": 1, "reads": a.reads, "reads_k20": a.reads_k20, "short_reads": a.short}
    long_reads = read_set(workloads.reads_of(genome, a.reads, read_len=150, seed=42))
    for k in (3, 10):
        out["hits_150bp_k%d" % k] = hits_run(long_reads, k)
    out["distance_150bp"] = distance_run(long_reads)
    del long_reads
    few = read_set(workloads.reads_of(genome, a.reads_k20, read_len=150, seed=42))
    out["hits_150bp_k20_%d_reads" % a.reads_k20] = hits_run(few, 20)
    out["distance_150bp_%d_reads" % a.reads_k20] = distance_run(few)
    del few
    short_reads = read_set(workloads.reads_of(genome, a.short, read_len=23, seed=7))
    out["hits_23mer_k4"] = hits_run(short_reads, 4)
    out["distance_23mer"] = distance_run(short_reads)
    out["card_after"] = card()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
