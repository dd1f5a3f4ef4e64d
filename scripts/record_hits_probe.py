#!/usr/bin/env python3
"""Times edlibB200FindRecordHits (all hits over a multi-record reference in one call) on the H100.

    python scripts/record_hits_probe.py [--reads 1000000] [--short 100000] [--records 1,8,512] [--repeats 3] [--out f]

The E. coli genome is cut at seeded points into R records.  Workloads: config-2 reads (150 bp, 3 % errors, seeded
generator of bench.py) at k = 3, and seeded 23-mers at k = 4.  For each R and workload, three things are timed:
  * one edlibB200FindRecordHits call over the R records (median and spread over the repeats after one warm-up);
  * R edlibB200FindHits calls, one per record (one pass after the warm-up above; its kernel time is the sum);
  * one edlibB200FindHits call over the unsplit genome (median and spread over the repeats).
Per-kernel device times of the last call of each (edlibB200LastKernelReport) are reported, and the records call's hit
lists are checked to be identical to the R single-record calls merged by (read, record, column).  The card's name,
power limit and SM clock are read in the same run.  Needs a GPU; prints one JSON document (and writes it to --out)."""
import argparse
import ctypes as C
import json
import os
import random
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))

from edlib_b200 import workloads  # noqa: E402
from edlib_b200._ffi import Hits, RecordHits, make_config, product_path  # noqa: E402
from hits_probe import Stats, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--short", type=int, default=100_000)
    ap.add_argument("--records", default="1,8,512")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON document to this file")
    a = ap.parse_args()
    lib = C.CDLL(product_path())
    if lib.edlibB200Available() != 1:
        sys.exit("no usable CUDA device: this probe measures the GPU only")
    cfg_t = type(make_config()[0])
    lib.edlibB200FindHits.restype = C.c_int
    lib.edlibB200FindHits.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.c_char_p, C.c_int, cfg_t,
                                      C.c_int, C.c_longlong, C.POINTER(Hits)]
    lib.edlibB200FreeHits.argtypes = [C.POINTER(Hits)]
    lib.edlibB200FindRecordHits.restype = C.c_int
    lib.edlibB200FindRecordHits.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_char_p),
                                            C.POINTER(C.c_int), C.c_int, cfg_t, C.c_int, C.c_longlong,
                                            C.POINTER(RecordHits)]
    lib.edlibB200FreeRecordHits.argtypes = [C.POINTER(RecordHits)]
    lib.edlibB200LastKernelReport.argtypes = [C.c_char_p, C.c_int]
    genome = workloads.ecoli_genome()
    gbytes = genome.tobytes()

    def read_set(arr):
        n, m = arr.shape
        bufs = [C.create_string_buffer(arr[i].tobytes(), m) for i in range(n)]
        ptrs = (C.c_char_p * n)(*[C.cast(b, C.c_char_p) for b in bufs])
        return bufs, ptrs, (C.c_int * n)(*([m] * n)), n

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
        return {"kernel_ms": round(s.kernelMs, 3), "filterDecided": s.filterDecided, "filterFallback": s.filterFallback,
                "kernels": kernels}

    def timed(fn, repeats):
        times = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            fn()
            times.append((time.perf_counter() - t0) * 1e3)
        times.sort()
        return {"ms_median": round(times[len(times) // 2], 3), "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3)}

    def flat(h, n):  # (read, column, score) of every hit, as numpy arrays
        s = h.offsets[n]
        counts = np.diff(np.ctypeslib.as_array(h.offsets, shape=(n + 1,)))
        read = np.repeat(np.arange(n, dtype=np.int64), counts)
        if s == 0:
            return read, np.zeros(0, np.int64), np.zeros(0, np.int64)
        return (read, np.ctypeslib.as_array(h.columns, shape=(s,)).astype(np.int64),
                np.ctypeslib.as_array(h.scores, shape=(s,)).astype(np.int64))

    def workload(rs, k, recs):
        _, ptrs, lens, n = rs
        cfg, _ = make_config(k, 2, 0)
        R = len(recs)
        rbufs = [C.create_string_buffer(r, len(r)) for r in recs]
        rptrs = (C.c_char_p * R)(*[C.cast(b, C.c_char_p) for b in rbufs])
        rlens = (C.c_int * R)(*[len(r) for r in recs])
        got = {}

        def one_call():
            h = RecordHits()
            assert lib.edlibB200FindRecordHits(ptrs, lens, n, rptrs, rlens, R, cfg, 0, 1 << 40, C.byref(h)) == 0
            read, col, score = flat(h.aln.hits, n)
            s = len(col)
            rec = np.ctypeslib.as_array(h.records, shape=(s,)).astype(np.int64) if s else np.zeros(0, np.int64)
            got["one"] = (read, rec, col, score)
            lib.edlibB200FreeRecordHits(C.byref(h))
        one_call()  # warm-up
        out = {"records_call": timed(one_call, a.repeats)}
        out["records_call"].update(last())
        parts = []
        kernel_ms = 0.0

        def separate():
            nonlocal kernel_ms
            parts.clear()
            kernel_ms = 0.0
            for r in range(R):
                h = Hits()
                assert lib.edlibB200FindHits(ptrs, lens, n, rbufs[r], len(recs[r]), cfg, 0, 1 << 40, C.byref(h)) == 0
                kernel_ms += last()["kernel_ms"]
                read, col, score = flat(h, n)
                parts.append((read, np.full(len(col), r, np.int64), col, score))
                lib.edlibB200FreeHits(C.byref(h))
        out["separate_calls"] = timed(separate, 1)
        out["separate_calls"].update(kernel_ms_sum=round(kernel_ms, 3), last_call=last())
        read, rec, col, score = (np.concatenate([p[i] for p in parts]) for i in range(4))
        order = np.lexsort((col, rec, read))
        one = got["one"]
        out["identical"] = bool(len(order) == len(one[0]) and all(np.array_equal(x[order], y)
                                                               for x, y in zip((read, rec, col, score), one)))
        out["hits_per_read"] = round(len(one[0]) / n, 3)
        return out

    def unsplit(rs, k):
        _, ptrs, lens, n = rs
        cfg, _ = make_config(k, 2, 0)
        gbuf = C.create_string_buffer(gbytes, len(gbytes))

        def call():
            h = Hits()
            assert lib.edlibB200FindHits(ptrs, lens, n, gbuf, len(gbytes), cfg, 0, 1 << 40, C.byref(h)) == 0
            lib.edlibB200FreeHits(C.byref(h))
        call()
        r = timed(call, a.repeats)
        r.update(last())
        return r

    rng = random.Random(7)
    out = {"card": card(), "repeats": a.repeats, "warmup": 1, "reads": a.reads, "short_reads": a.short}
    for name, rs, k in (("150bp_k3", read_set(workloads.reads_of(genome, a.reads, read_len=150, seed=42)), 3),
                        ("23mer_k4", read_set(workloads.reads_of(genome, a.short, read_len=23, seed=7)), 4)):
        out["unsplit_" + name] = unsplit(rs, k)
        for R in (int(x) for x in a.records.split(",")):
            cuts = sorted(rng.sample(range(1, len(gbytes)), R - 1))
            edges = [0] + cuts + [len(gbytes)]
            recs = [gbytes[x:y] for x, y in zip(edges, edges[1:])]
            out["R%d_%s" % (R, name)] = workload(rs, k, recs)
        del rs
    out["card_after"] = card()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
