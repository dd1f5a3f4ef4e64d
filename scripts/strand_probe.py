#!/usr/bin/env python
"""Cost of aligning both strands: the headline read set of bench.py (1M x 150 bp reads from the E. coli genome, HW,
distance) with a seeded half of the reads reverse-complemented, resident in HBM.

Two staged batches, computed alternately for several repeats (L2 flushed before every step):
  forward  edlibB200BatchPrepare on the truly oriented reads (what a caller who knew every strand would run);
  strands  edlibB200BatchPrepareStrands on the mixed reads (every read and its reverse complement, one call).
Prints one JSON line: step times of both, per-kernel CUDA-event times of a step, filterDecided / filterFallback, the
card's name and power limit, and a check that every read's strand-call distance equals the forward-only distance or is
smaller on the read's other strand.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "scripts"))

from edlib_b200 import workloads  # noqa: E402
from seed_stage_probe import card  # noqa: E402

NUM_READS, READ_LEN = 1_000_000, 150

COMP = np.arange(256, dtype=np.uint8)
for a, b in (b"AT", b"CG", b"RY", b"KM", b"BV", b"DH"):
    for x, y in ((a, b), (a | 0x20, b | 0x20)):
        COMP[x], COMP[y] = y, x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()

    import torch

    import bench
    assert torch.cuda.is_available(), "needs a CUDA device"
    E = bench.Engine(0)
    L = E.L
    L.edlibB200BatchPrepareStrands.restype = C.c_void_p
    L.edlibB200BatchPrepareStrands.argtypes = L.edlibB200BatchPrepare.argtypes
    L.edlibB200BatchStrands.argtypes = [C.c_void_p, C.c_void_p]
    L.edlibB200FreeResults.argtypes = [C.c_void_p, C.c_int]

    target = workloads.ecoli_genome()
    true = workloads.reads_of(target, NUM_READS, READ_LEN, seed=42, pinned=True)
    flip = np.random.Generator(np.random.PCG64(7)).random(NUM_READS) < 0.5
    mixed = workloads.pinned_empty(true.shape)
    mixed[:] = true
    mixed[flip] = COMP[true[flip, ::-1]]
    cfg, _ = bench.make_config(-1, bench.MODE_HW, bench.TASK_DISTANCE)

    def prepare(reads, fn):
        qptr, qlen, tptr, tlen = bench.pointer_arrays(reads, target)
        b = fn(bench.as_pp(qptr), bench.as_pi(qlen), bench.as_pp(tptr), bench.as_pi(tlen), NUM_READS, cfg)
        assert b, L.edlibB200LastError()
        return b, (qptr, qlen, tptr, tlen)

    batches = {"forward": prepare(true, L.edlibB200BatchPrepare), "strands": prepare(mixed, L.edlibB200BatchPrepareStrands)}
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    st = bench.Stats()
    step_ms = {k: [] for k in batches}
    per_kernel = {k: {} for k in batches}
    filt = {}
    before = card()
    for _ in range(args.repeats):
        for name, (batch, _keep) in batches.items():
            for i in range(args.warmup + args.steps):
                flush_buf.zero_()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                assert L.edlibB200BatchCompute(batch, C.byref(st)) == 0, L.edlibB200LastError()
                torch.cuda.synchronize()
                if i < args.warmup:
                    continue
                step_ms[name].append(1e3 * (time.perf_counter() - t0))
                for kname, (ms, cnt) in E.kernel_report().items():
                    a = per_kernel[name].setdefault(kname, [0.0, 0.0])
                    n = args.steps * args.repeats
                    a[0] += ms / n
                    a[1] += cnt / n
            filt[name] = {"decided": int(st.filterDecided), "fallback": int(st.filterFallback), "windows": int(st.filterWindows)}

    dist = {}
    for name, (batch, _keep) in batches.items():
        res = np.zeros(NUM_READS, dtype=bench.RESULT_DTYPE)
        assert L.edlibB200BatchResults(batch, res.ctypes.data) == 0, L.edlibB200LastError()
        dist[name] = res["editDistance"].copy()
        L.edlibB200FreeResults(res.ctypes.data, NUM_READS)
    strands = np.zeros(NUM_READS, dtype=np.uint8)
    assert L.edlibB200BatchStrands(batches["strands"][0], strands.ctypes.data) == 0
    for batch, _keep in batches.values():
        L.edlibB200BatchFree(batch)
    # a strand call gives the forward-only distance, or a smaller one found on the read's other strand (the reverse
    # complement of its true orientation: '-' for a read left as drawn, '+' for a flipped one)
    same = dist["strands"] == dist["forward"]
    better = (strands.astype(bool) != flip) & (dist["strands"] >= 0) & ((dist["forward"] < 0) | (dist["strands"] < dist["forward"]))
    print(json.dumps({
        "probe": "strands", "reads": NUM_READS, "read_len": READ_LEN, "reverse_complemented": int(flip.sum()),
        "steps": args.steps, "repeats": args.repeats,
        "step_ms": {k: {"mean": round(float(np.mean(v)), 3), "min": round(min(v), 3), "max": round(max(v), 3)} for k, v in step_ms.items()},
        "ratio_mean": round(float(np.mean(step_ms["strands"]) / np.mean(step_ms["forward"])), 3),
        "kernels_ms": {k: {n: round(v[0], 4) for n, v in sorted(d.items(), key=lambda kv: -kv[1][0])} for k, d in per_kernel.items()},
        "launches_per_step": {k: {n: v[1] for n, v in d.items()} for k, d in per_kernel.items()},
        "filter": filt,
        "check": {"ok": bool((same | better).all()), "equal": int(same.sum()), "smaller_on_other_strand": int((better & ~same).sum()),
                  "strand_matches_flip": int((strands.astype(bool) == flip).sum())},
        "device": before, "device_after": card()}))


if __name__ == "__main__":
    main()
