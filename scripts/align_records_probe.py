#!/usr/bin/env python3
"""Times edlibB200AlignRecords (each read's best record of a multi-record reference, in one call) on the H100.

    python scripts/align_records_probe.py [--reads 1000000] [--records 1,8,512] [--tasks distance,loc,path]
                                          [--separate-reads 100000] [--repeats 3] [--out f]

The E. coli genome is cut at seeded points into R records; the reads are config-2 reads (150 bp, 3 % errors, seeded
generator of bench.py), aligned HW at k = -1 with task DISTANCE, LOC and PATH.  For each task three things are timed:
  * one edlibAlignBatch call over the unsplit genome (median and spread over the repeats after one warm-up);
  * for each R, one edlibB200AlignRecords call over the R records (median and spread over the repeats after one
    warm-up);
  * for each R, R edlibAlignBatch calls, one per record, of the first --separate-reads reads (one pass; its kernel time
    is the sum).  Over a record that holds only a part of the genome, most reads have no close match, and a call of
    1 M such reads at k = -1 can run out of device memory; a failed call is reported with its error.
Per-kernel device times of the last call of each (edlibB200LastKernelReport) are reported.  On those reads the records
call is checked against the R single-record calls merged by the rule of include/edlib_b200.h (least distance, lowest
record): the distance, record, number of locations, alignment length and alphabet length of every read, and every
location and alignment byte of a sample of them.  The card's name, power limit and SM clock are read in the same run.  Needs a GPU;
prints one JSON document (and writes it to --out)."""
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
from edlib_b200._ffi import AlignResult, make_config, product_path  # noqa: E402
from hits_probe import Stats, card  # noqa: E402

TASKS = {"distance": 0, "loc": 1, "path": 2}
# include/edlib.h EdlibAlignResult as a numpy record (48 bytes)
RESULT = np.dtype([("status", "<i4"), ("ed", "<i4"), ("end", "<u8"), ("start", "<u8"), ("num", "<i4"), ("pad", "<i4"),
                   ("aln", "<u8"), ("alnLen", "<i4"), ("alpha", "<i4")])
SAMPLE = 2000  # reads whose locations and alignments are compared byte for byte


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--records", default="1,8,512")
    ap.add_argument("--tasks", default="distance,loc,path")
    ap.add_argument("--separate-reads", type=int, default=100_000, help="0: no single-record calls")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON document to this file")
    a = ap.parse_args()
    lib = C.CDLL(product_path())
    if lib.edlibB200Available() != 1:
        sys.exit("no usable CUDA device: this probe measures the GPU only")
    cfg_t = type(make_config()[0])
    lib.edlibAlignBatch.restype = C.c_int
    lib.edlibAlignBatch.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_char_p),
                                    C.POINTER(C.c_int), C.c_int, cfg_t, C.POINTER(AlignResult)]
    lib.edlibB200AlignRecords.restype = C.c_int
    lib.edlibB200AlignRecords.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_char_p),
                                          C.POINTER(C.c_int), C.c_int, cfg_t, C.c_int, C.POINTER(AlignResult),
                                          C.POINTER(C.c_int), C.POINTER(C.c_ubyte)]
    lib.edlibB200FreeResults.argtypes = [C.POINTER(AlignResult), C.c_int]
    lib.edlibB200LastKernelReport.argtypes = [C.c_char_p, C.c_int]
    lib.edlibB200LastError.restype = C.c_char_p
    genome = workloads.ecoli_genome()
    gbytes = genome.tobytes()
    arr = workloads.reads_of(genome, a.reads, read_len=150, seed=42)
    n, m = arr.shape
    rbufs = [C.create_string_buffer(arr[i].tobytes(), m) for i in range(n)]
    qptrs = (C.c_char_p * n)(*[C.cast(b, C.c_char_p) for b in rbufs])
    qlens = (C.c_int * n)(*([m] * n))
    del arr

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

    def view(res, count=n):
        return np.frombuffer(res, dtype=RESULT, count=count)

    def arrays(r):  # every array of one result, as bytes
        out = []
        for ptr, count, size in ((r["end"], r["num"], 4), (r["start"], r["num"], 4), (r["aln"], r["alnLen"], 1)):
            out.append(C.string_at(int(ptr), int(count) * size) if ptr else None)
        return out

    def targets(buf, tlen, count):  # the per-pair target arrays of one target, built outside the timed calls
        return (C.c_char_p * count)(*([C.cast(buf, C.c_char_p)] * count)), (C.c_int * count)(*([tlen] * count)), count

    def batch(t, cfg, res):  # "" or the error of the call (the first t[2] reads)
        ok = lib.edlibAlignBatch(qptrs, qlens, t[0], t[1], t[2], cfg, res) == 0
        return "" if ok else lib.edlibB200LastError().decode()

    rng = random.Random(7)
    S = min(n, a.separate_reads)
    sample = sorted(rng.sample(range(S), min(SAMPLE, S))) if S else []
    out = {"card": card(), "repeats": a.repeats, "warmup": 1, "reads": n, "read_len": m, "k": -1, "separate_reads": S}
    gbuf = C.create_string_buffer(gbytes, len(gbytes))
    gt = targets(gbuf, len(gbytes), n)
    splits = {}
    for R in (int(x) for x in a.records.split(",")):
        cuts = sorted(rng.sample(range(1, len(gbytes)), R - 1))
        edges = [0] + cuts + [len(gbytes)]
        splits[R] = [gbytes[x:y] for x, y in zip(edges, edges[1:])]
    for task in a.tasks.split(","):
        cfg, _ = make_config(-1, 2, TASKS[task])
        res = (AlignResult * n)()

        def unsplit():
            err = batch(gt, cfg, res)
            assert not err, err
            lib.edlibB200FreeResults(res, n)
        unsplit()
        out["unsplit_" + task] = timed(unsplit, a.repeats)
        out["unsplit_" + task].update(last())
        for R, recs in splits.items():
            bufs = [C.create_string_buffer(r, len(r)) for r in recs]
            rptrs = (C.c_char_p * R)(*[C.cast(b, C.c_char_p) for b in bufs])
            rlens = (C.c_int * R)(*[len(r) for r in recs])
            chosen = (C.c_int * n)()

            def records_call():
                lib.edlibB200FreeResults(res, n)
                if lib.edlibB200AlignRecords(qptrs, qlens, n, rptrs, rlens, R, cfg, 0, res, chosen, None) != 0:
                    raise RuntimeError(lib.edlibB200LastError().decode())
            try:
                records_call()
                entry = {"records_call": timed(records_call, a.repeats)}
            except RuntimeError as e:
                out["R%d_%s" % (R, task)] = {"records_call": {"failed": str(e)}}
                print(json.dumps({"R": R, "task": task, "records_failed": str(e)}), file=sys.stderr, flush=True)
                continue
            entry["records_call"].update(last())
            got = view(res, S).copy()
            got_rec = np.ctypeslib.as_array(chosen)[:S].copy()
            got_arrays = [arrays(got[i]) for i in sample]
            lib.edlibB200FreeResults(res, n)
            entry["reads_per_record_max"] = int(np.bincount(got_rec, minlength=R).max()) if S else None
            out["R%d_%s" % (R, task)] = entry
            if S == 0:
                print(json.dumps({"R": R, "task": task, "records_ms": entry["records_call"]["ms_median"]}), file=sys.stderr,
                      flush=True)
                continue
            # R single-record calls, merged by the rule: least distance (-1: none), then lowest record
            best = np.full(S, -1, np.int64)
            best_rec = np.zeros(S, np.int64)
            merged = np.zeros(S, RESULT)
            merged_arrays = [None] * len(sample)
            kernel_ms = 0.0
            one = (AlignResult * S)()
            per = [targets(bufs[r], len(recs[r]), S) for r in range(R)]
            t0 = time.perf_counter()
            failed = None
            for r in range(R):
                err = batch(per[r], cfg, one)
                if err:  # reported, and the comparison is left out
                    failed = {"record": r, "record_len": len(recs[r]), "error": err}
                    break
                kernel_ms += last()["kernel_ms"]
                v = view(one, S)
                better = (v["ed"] >= 0) & ((best < 0) | (v["ed"] < best))
                if r == 0:
                    better[:] = True
                best = np.where(better, np.where(v["ed"] >= 0, v["ed"], -1), best)
                best_rec[better] = r
                merged[better] = v[better]
                for j, i in enumerate(sample):
                    if better[i]:
                        merged_arrays[j] = arrays(v[i])
                lib.edlibB200FreeResults(one, S)
            entry["separate_calls"] = {"ms": round((time.perf_counter() - t0) * 1e3, 3), "kernel_ms_sum": round(kernel_ms, 3),
                                       "last_call": last()}
            if failed:
                entry["separate_calls"] = {"failed": failed}
            fields = ("status", "ed", "num", "alnLen", "alpha")
            entry["identical"] = None if failed else bool(np.array_equal(got_rec, best_rec) and all(np.array_equal(got[f], merged[f]) for f in fields)
                                      and got_arrays == merged_arrays)
            print(json.dumps({"R": R, "task": task, "records_ms": entry["records_call"]["ms_median"],
                              "separate_ms": entry["separate_calls"].get("ms"), "identical": entry["identical"],
                              "separate_failed": failed}),
                  file=sys.stderr, flush=True)
    out["card_after"] = card()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
