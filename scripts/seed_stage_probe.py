#!/usr/bin/env python
"""Where the seed stage's time goes on the headline workload of bench.py (1M x 150 bp reads, HW distance, E. coli).

  --gpu      runs the headline inputs through edlibB200BatchPrepare / edlibB200BatchCompute (L2 flushed between steps)
             and prints one JSON line: per-kernel CUDA-event times of a step (edlibB200LastKernelReport, averaged over the
             timed steps), the step time, the filter counters, and the card's name, power limit and SM clock.  Run it
             once as is and once with EDLIB_B200_FILTER_SEED_LEVELS=1, which leaves only the level-0 launch of
             `seed_plan` under that name (the other reads then take the plain sweep, so that run's step time means
             nothing): the difference is what the later levels cost.
  --cpu      a numpy pass over the same reads and genome that counts, for the level-0 seeds of every read (the engine's
             rules: eb_pass_lane.cpp build_seed_index / fill_seed_plan, eb_core.h seed_plan_read), how often each path
             of the planning kernel runs: index range sizes, long ranges (> 4 entries, walked by the whole group),
             candidates per read, reads over 32 candidates (the bitonic sort) and saturated reads.  Needs no GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from edlib_b200 import workloads  # noqa: E402

NUM_READS, READ_LEN = 1_000_000, 150


def headline_inputs(pinned):
    target = workloads.ecoli_genome()
    reads = workloads.reads_of(target, NUM_READS, READ_LEN, seed=42, pinned=pinned)
    return target, reads


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), (v.strip() for v in out[0].split(",")))) if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def gpu_run(steps, warmup):
    import ctypes as C

    import torch

    import bench
    assert torch.cuda.is_available(), "--gpu needs a CUDA device"
    E = bench.Engine(0)
    L = E.L
    target, reads = headline_inputs(pinned=True)
    qptr, qlen, tptr, tlen = bench.pointer_arrays(reads, target)
    cfg, _ = bench.make_config(-1, bench.MODE_HW, bench.TASK_DISTANCE)
    batch = L.edlibB200BatchPrepare(bench.as_pp(qptr), bench.as_pi(qlen), bench.as_pp(tptr), bench.as_pi(tlen),
                                    NUM_READS, cfg)
    assert batch, L.edlibB200LastError()
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    st = bench.Stats()
    per_kernel, step_ms = {}, []
    before = card()
    for i in range(warmup + steps):
        flush_buf.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        assert L.edlibB200BatchCompute(batch, C.byref(st)) == 0, L.edlibB200LastError()
        torch.cuda.synchronize()
        if i < warmup:
            continue
        step_ms.append(1e3 * (time.perf_counter() - t0))
        for name, (ms, cnt) in E.kernel_report().items():
            a = per_kernel.setdefault(name, [0.0, 0])
            a[0] += ms / steps
            a[1] += cnt / steps
    L.edlibB200BatchFree(batch)
    print(json.dumps({
        "probe": "gpu", "seed_levels_env": os.environ.get("EDLIB_B200_FILTER_SEED_LEVELS"), "steps": steps,
        "step_ms": {"mean": round(float(np.mean(step_ms)), 3), "min": round(min(step_ms), 3), "max": round(max(step_ms), 3)},
        "kernel_ms": round(float(st.kernelMs), 3),
        "kernels_ms": {k: round(v[0], 4) for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1][0])},
        "launches_per_step": {k: v[1] for k, v in per_kernel.items()},
        "filter": {"decided": int(st.filterDecided), "fallback": int(st.filterFallback), "windows": int(st.filterWindows)},
        "device": before, "device_after": card()}))


def cpu_run():
    target, reads = headline_inputs(pinned=False)
    n = len(target)
    code = np.zeros(256, dtype=np.uint32)
    for i, ch in enumerate(b"ACGT"):
        code[ch] = i
    g = code[target]
    sigma = 4
    # the engine's level-0 geometry for this target (build_seed_index / fill_seed_plan / seed_threshold, defaults)
    L0, v = 4, float(sigma) ** 4
    while v < 4.0 * n and L0 < 32:
        v *= sigma
        L0 += 1
    Lidx, keys = 1, sigma
    while Lidx < 16 and keys * sigma <= min(max(2 * n, 4096), 1 << 28):
        keys *= sigma
        Lidx += 1
    Ls, Lk = L0, min(L0, Lidx)
    t = min(READ_LEN // Ls - 1, 20)
    stride = READ_LEN // (t + 1)
    max_bucket = min(128 << 1, 8192)

    def kmer_keys(a, L):  # key of the L codes at every position of `a` (missing codes past the end count as 0)
        k = np.zeros(a.shape[-1], dtype=np.uint64)
        padded = np.concatenate([a, np.zeros(L, dtype=a.dtype)])
        for x in range(L):
            k = k * np.uint64(sigma) + padded[x:x + a.shape[-1]].astype(np.uint64)
        return k

    bucket = np.bincount(kmer_keys(g, Lk).astype(np.int64), minlength=keys)
    full = np.sort(kmer_keys(g[:n - Ls + 1], Ls))  # exact occurrences of whole seeds (verified candidates)

    q = code[reads]
    sizes = np.zeros((NUM_READS, t + 1), dtype=np.int64)
    hits = np.zeros((NUM_READS, t + 1), dtype=np.int64)
    for j in range(t + 1):
        s = q[:, j * stride:j * stride + Ls].astype(np.uint64)
        kl = np.zeros(NUM_READS, dtype=np.uint64)
        kf = np.zeros(NUM_READS, dtype=np.uint64)
        for x in range(Ls):
            if x < Lk:
                kl = kl * np.uint64(sigma) + s[:, x]
            kf = kf * np.uint64(sigma) + s[:, x]
        sizes[:, j] = bucket[kl.astype(np.int64)]
        hits[:, j] = np.searchsorted(full, kf, side="right") - np.searchsorted(full, kf, side="left")
    repeat = (sizes > max_bucket).any(axis=1)
    cand = np.where(sizes > max_bucket, 0, hits).sum(axis=1)
    longr = (sizes > 4) & (sizes <= max_bucket)
    saturated = repeat | (cand > 256)
    q_c = np.percentile(cand, [50, 90, 99, 99.9]).tolist()
    print(json.dumps({
        "probe": "cpu", "level": 0, "Ls": Ls, "Lidx": Lidx, "t": t, "seeds_per_read": t + 1, "stride": stride,
        "max_bucket": max_bucket,
        "index_range_entries": {"mean": round(float(sizes.mean()), 3), "p99": float(np.percentile(sizes, 99)),
                                "max": int(sizes.max())},
        "seeds_long_range": {"count": int(longr.sum()), "frac": round(float(longr.mean()), 5),
                             "reads_with_one": int(longr.any(axis=1).sum())},
        "seeds_over_max_bucket": int((sizes > max_bucket).sum()),
        "candidates_per_read": {"mean": round(float(cand.mean()), 3), "p50_p90_p99_p999": q_c, "max": int(cand.max())},
        "reads_over_16_candidates": int((cand > 16).sum()),
        "reads_over_32_candidates": int((cand > 32).sum()),
        "reads_saturated": int(saturated.sum()), "reads_repeat": int(repeat.sum())}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpu", action="store_true")
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if args.cpu:
        cpu_run()
    if args.gpu:
        gpu_run(args.steps, args.warmup)
    if not (args.cpu or args.gpu):
        ap.error("give --gpu and/or --cpu")


if __name__ == "__main__":
    main()
