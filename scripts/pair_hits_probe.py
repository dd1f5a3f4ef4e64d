#!/usr/bin/env python3
"""Times edlibB200FindPairHits (every hit of each query in its own target, one call) on the H100.

    python scripts/pair_hits_probe.py [--long 100000] [--short 1000000] [--repeats 3] [--sample 200] [--out f]

Workloads:
  (a) `--long` seeded reads of 1-20 kbp from the E. coli genome (3 % errors), a quarter of them chimeric with a 30 bp
      adapter planted 0-3 times (5 % edits); each read is the target of one pair whose query is the adapter; k = 3, 6;
  (b) `--short` config-2 reads (150 bp, 3 % errors, the seeded generator of bench.py), each the target of two pairs
      whose queries are two 20 bp primers taken from the genome; k = 3.
For each: one call (median and range over the repeats after one warm-up) with its per-kernel device times
(edlibB200LastKernelReport) and hits per pair; `edlibAlignBatch` HW DISTANCE at the same k over the same pairs as a
yardstick; and a seeded sample of pairs checked against single-target edlibB200FindHitAlignments calls.  The card's
name, power limit and SM clock are read in the same run.  Needs a GPU; prints one JSON document (and writes it to --out)."""
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
from edlib_b200._ffi import AlignResult, HitAlignments, make_config, product_path  # noqa: E402
from hits_probe import Stats, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--long", type=int, default=100_000)
    ap.add_argument("--short", type=int, default=1_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sample", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the JSON document to this file")
    a = ap.parse_args()
    lib = C.CDLL(product_path())
    if lib.edlibB200Available() != 1:
        sys.exit("no usable CUDA device: this probe measures the GPU only")
    cfg_t = type(make_config()[0])
    PP, PI = C.POINTER(C.c_char_p), C.POINTER(C.c_int)
    lib.edlibB200FindPairHits.restype = C.c_int
    lib.edlibB200FindPairHits.argtypes = [PP, PI, PP, PI, C.c_int, cfg_t, C.c_int, C.c_longlong, C.POINTER(HitAlignments)]
    lib.edlibB200FindHitAlignments.restype = C.c_int
    lib.edlibB200FindHitAlignments.argtypes = [PP, PI, C.c_int, C.c_char_p, C.c_int, cfg_t, C.c_int, C.c_longlong,
                                               C.POINTER(HitAlignments)]
    lib.edlibB200FreeHitAlignments.argtypes = [C.POINTER(HitAlignments)]
    lib.edlibAlignBatch.restype = C.c_int
    lib.edlibAlignBatch.argtypes = [PP, PI, PP, PI, C.c_int, cfg_t, C.POINTER(AlignResult)]
    lib.edlibB200FreeResults.argtypes = [C.POINTER(AlignResult), C.c_int]
    lib.edlibB200LastKernelReport.argtypes = [C.c_char_p, C.c_int]
    genome = workloads.ecoli_genome()
    G = len(genome)

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
        return {"kernel_ms": round(s.kernelMs, 3), "launches": s.launches, "filterDecided": s.filterDecided,
                "filterFallback": s.filterFallback, "kernels": kernels}

    def timed(fn, repeats):
        fn()  # warm-up
        times = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            fn()
            times.append((time.perf_counter() - t0) * 1e3)
        times.sort()
        return {"ms_median": round(times[len(times) // 2], 3), "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3)}

    def ptrs(addrs):  # numpy uint64 addresses -> const char* const*
        arr = np.ascontiguousarray(addrs, dtype=np.uint64)
        return arr, arr.ctypes.data_as(PP)

    def lens(x):
        arr = np.ascontiguousarray(x, dtype=np.int32)
        return arr, arr.ctypes.data_as(PI)

    def workload(qaddr, qlen, taddr, tlen, k, qbytes, tbytes):
        """qbytes / tbytes: pair -> bytes of its query / target (for the sampled single-target checks)."""
        n = len(qaddr)
        keep = [ptrs(qaddr), lens(qlen), ptrs(taddr), lens(tlen)]
        qp, ql, tp, tl = (x[1] for x in keep)
        cfg, _ = make_config(k, 2, 0)
        got = {}

        def call():
            h = HitAlignments()
            assert lib.edlibB200FindPairHits(qp, ql, tp, tl, n, cfg, 0, 1 << 40, C.byref(h)) == 0
            got["hits"] = int(h.hits.offsets[n])
            lib.edlibB200FreeHitAlignments(C.byref(h))
        out = {"pairs": n, "k": k, "pair_call": timed(call, a.repeats)}
        out["pair_call"].update(last())
        out["hits_per_pair"] = round(got["hits"] / n, 4)
        res = (AlignResult * n)()

        def yardstick():
            assert lib.edlibAlignBatch(qp, ql, tp, tl, n, cfg, res) == 0
            lib.edlibB200FreeResults(res, n)
        out["align_batch_hw_distance"] = timed(yardstick, a.repeats)
        out["align_batch_hw_distance"].update(last())
        # sampled pairs: the pair call's entry against a single-target edlibB200FindHitAlignments call (task PATH)
        cfgp, _ = make_config(k, 2, 2)
        h = HitAlignments()
        assert lib.edlibB200FindPairHits(qp, ql, tp, tl, n, cfgp, 1, 1 << 40, C.byref(h)) == 0

        def entry(x, i, j=0):
            lo, hi = x.hits.offsets[i], x.hits.offsets[i + 1]
            off = x.alignmentOffsets
            return (x.hits.counts[i], list(x.hits.columns[lo:hi]), list(x.hits.scores[lo:hi]), list(x.hits.strands[lo:hi]),
                    list(x.starts[lo:hi]), [C.string_at(C.cast(x.alignments, C.c_void_p).value + off[h], off[h + 1] - off[h])
                                            for h in range(lo, hi)])
        rng = random.Random(11)
        bad = 0
        sample = rng.sample(range(n), min(a.sample, n))
        for i in sample:
            q, t = qbytes(i), tbytes(i)
            s1 = HitAlignments()
            qa = (C.c_char_p * 1)(q)
            la = (C.c_int * 1)(len(q))
            assert lib.edlibB200FindHitAlignments(qa, la, 1, t, len(t), cfgp, 1, 1 << 40, C.byref(s1)) == 0
            bad += entry(s1, 0) != entry(h, i)
            lib.edlibB200FreeHitAlignments(C.byref(s1))
        lib.edlibB200FreeHitAlignments(C.byref(h))
        out["sample_checked"] = len(sample)
        out["sample_mismatches"] = bad
        return out

    rng = np.random.Generator(np.random.PCG64(5))
    out = {"card": card(), "repeats": a.repeats, "warmup": 1}
    # ---- (a) long reads, each the target of one adapter pair ----
    adapter = workloads.random_dna(30, 77).tobytes()
    lib_s = workloads._synth()
    lengths = rng.integers(1_000, 20_001, size=a.long)
    starts = rng.integers(0, G - 20_001, size=a.long)
    reads = []
    buf = np.empty(2 * 20_001 + 64, dtype=np.uint8)
    pyr = random.Random(9)
    for i in range(a.long):
        w = np.ascontiguousarray(genome[starts[i]:starts[i] + lengths[i]])
        m = lib_s.synth_mutate(w.ctypes.data, len(w), buf.ctypes.data, 0.03, 1_000_003 + i)
        r = bytearray(buf[:m].tobytes())
        if i % 4 == 0:  # chimeric: the adapter 0-3 times with 5 % edits
            for _ in range(pyr.randrange(0, 4)):
                ad = np.frombuffer(adapter, dtype=np.uint8).copy()
                mb = np.empty(80, dtype=np.uint8)
                mm = lib_s.synth_mutate(ad.ctypes.data, len(ad), mb.ctypes.data, 0.05, 7_000_003 + i * 4 + len(r) % 4)
                at = pyr.randrange(0, len(r) - mm)
                r[at:at + mm] = mb[:mm].tobytes()
        reads.append(bytes(r))
    rbufs = [C.create_string_buffer(r, len(r)) for r in reads]
    taddr = np.array([C.addressof(b) for b in rbufs], dtype=np.uint64)
    abuf = C.create_string_buffer(adapter, len(adapter))
    qaddr = np.full(a.long, C.addressof(abuf), dtype=np.uint64)
    out["a_read_bp_total"] = int(sum(len(r) for r in reads))
    for k in (3, 6):
        out["a_long_reads_adapter_k%d" % k] = workload(qaddr, np.full(a.long, 30), taddr, [len(r) for r in reads], k,
                                                       lambda i: adapter, lambda i: reads[i])
    del rbufs, reads
    # ---- (b) config-2 reads, each the target of two primer pairs ----
    short = workloads.reads_of(genome, a.short, read_len=150, seed=42)
    primers = [genome[p:p + 20].tobytes() for p in (1_000_000, 3_000_000)]
    pbufs = [C.create_string_buffer(p, 20) for p in primers]
    n = 2 * a.short
    qaddr = np.array([C.addressof(pbufs[0]), C.addressof(pbufs[1])], dtype=np.uint64)[np.arange(n) % 2]
    taddr = short.ctypes.data + 150 * (np.arange(n, dtype=np.uint64) // 2)
    out["b_config2_two_primers_k3"] = workload(qaddr, np.full(n, 20), taddr, np.full(n, 150), 3,
                                               lambda i: primers[i % 2], lambda i: short[i // 2].tobytes())
    out["card_after"] = card()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
