"""The seed stage of the candidate filter at kernel level: the index build (seed_count / scan / seed_fill) and the
planning kernel (seed_plan_read) are called through a backend's own launches (tests/kernel_probe) and their outputs
compared exactly with a brute-force reference (seed_ref.py).  Results-only tests cannot see most planner bugs: a read
that loses candidates or windows goes on to a later stage and still gets the right answer.

The CPU part runs the emulation serially (one member per read) and with lane groups of the width the device uses (one
thread per lane, EDLIB_EMUL_SEED_GROUP=device; in subprocesses with a timeout, since lanes that disagree on the number
of syncs hang).  The gpu part runs the same generators on the CUDA backend, on every planning instance it can pick."""
import ctypes as C
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import seed_ref as R
from edlib_b200._ffi import REPO

PROBE_DIR = os.path.join(REPO, "tests", "kernel_probe")
TESTS_DIR = os.path.join(REPO, "tests")
TILE = 4096  # keys per tile of the CUDA scan (eb_kernels.cu: SCAN_TILE); its top level gives 1024 threads the tile sums
SCAN_COUNTS = [0, 1, 4095, 4096, 4097, TILE * 1024 - 1, TILE * 1024, TILE * 1024 + 1, TILE * 4096 + 17]


class Probe:
    def __init__(self, which):
        if which == "emul":
            subprocess.run(["make", "-s", "-C", os.path.join(REPO, "tests", "emul")], check=True)
        subprocess.run(["make", "-s", "-C", PROBE_DIR, which], check=True)
        self.L = C.CDLL(os.path.join(PROBE_DIR, "libprobe_%s.so" % which))
        self.L.probe_error.restype = C.c_char_p
        self.L.probe_plan.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]

    def _ok(self, status):
        assert status == 0, self.L.probe_error().decode()

    def scan(self, data):
        buf = np.zeros(len(data) + 1, dtype=np.int32)
        buf[:len(data)] = data
        self._ok(self.L.probe_scan(C.c_void_p(buf.ctypes.data), C.c_int(len(data))))
        return buf

    def index(self, tcodes, Lidx, sigma, numPos=None):
        tcodes = np.ascontiguousarray(tcodes, dtype=np.uint8)
        numPos = len(tcodes) if numPos is None else numPos
        bs = np.zeros(sigma ** Lidx + 1, dtype=np.int32)
        pos = np.zeros(max(numPos, 1), dtype=np.int32)
        self._ok(self.L.probe_index(C.c_void_p(tcodes.ctypes.data), C.c_int(len(tcodes)), C.c_int(Lidx), C.c_int(sigma),
                                    C.c_int(numPos), C.c_void_p(bs.ctypes.data), C.c_void_p(pos.ctypes.data)))
        return bs, pos[:numPos]

    def build_index(self, tcodes, ncodes):
        """The engine's build_seed_index: (ok, Lidx, sigma, bucketStart, positions)."""
        tcodes = np.ascontiguousarray(tcodes, dtype=np.uint8)
        info = np.zeros(8, dtype=np.int32)
        self._ok(self.L.probe_build_index(C.c_void_p(tcodes.ctypes.data), C.c_int(len(tcodes)), C.c_int(ncodes),
                                          C.c_void_p(info.ctypes.data)))
        if not info[0]:
            return False, 0, 0, None, None
        bs = np.zeros(int(info[3]) + 1, dtype=np.int32)
        pos = np.zeros(len(tcodes), dtype=np.int32)
        self._ok(self.L.probe_fetch_index(C.c_void_p(bs.ctypes.data), C.c_void_p(pos.ctypes.data)))
        return True, int(info[1]), int(info[2]), bs, pos

    def plan(self, case, bs, pos, level, maxLen, winCap):
        t = np.ascontiguousarray(case["t"], dtype=np.uint8)
        qs = case["qs"]
        qlen = np.array([len(q) for q in qs], dtype=np.int32)
        qoff = np.zeros(len(qs), dtype=np.uint64)
        qoff[1:] = np.cumsum(qlen[:-1])
        qcodes = np.ascontiguousarray(np.concatenate(qs) if qs else np.zeros(0), dtype=np.uint8)
        rl = None if case.get("readList") is None else np.ascontiguousarray(case["readList"], dtype=np.int32)
        thr = None if case.get("thr") is None else np.ascontiguousarray(case["thr"], dtype=np.int32)
        numReads = case["numReads"]
        ip = np.array([case["kBound"], case["seedK"], maxLen, case["Ls"], case["Lidx"], case["sigma"], case["maxBucket"],
                       level, case["spread"], winCap, case.get("firstPair", 0)], dtype=np.int32)
        plan = np.zeros((max(numReads, 1), 4), dtype=np.int32)
        win = np.zeros((5, max(winCap, 1)), dtype=np.int32)
        cnt = np.zeros(1, dtype=np.int32)
        inst = np.zeros(3, dtype=np.int32)
        ptr = (lambda a: None if a is None else C.c_void_p(a.ctypes.data))
        self._ok(self.L.probe_plan(ptr(t), len(t), ptr(qcodes), qcodes.nbytes, ptr(qoff), ptr(qlen), len(qs), ptr(rl),
                                   ptr(thr), numReads, ptr(ip), ptr(bs), len(bs) - 1, ptr(pos), len(pos), ptr(plan),
                                   ptr(win), ptr(cnt), ptr(inst)))
        return plan[:numReads], win[:, :winCap], int(cnt[0]), tuple(int(x) for x in inst)


# ---------------------------------------------------------------------------------------------------------------
# plan cases: dicts of the SeedPlanParams inputs (t: target codes, qs: read codes, ...) and the reference check
# ---------------------------------------------------------------------------------------------------------------

def rand_codes(rng, n, sigma):
    return np.array([rng.randrange(sigma) for _ in range(n)], dtype=np.uint8)


def make_case(t, qs, sigma, Ls, Lidx, **kw):
    case = dict(t=np.asarray(t, dtype=np.uint8), qs=[np.asarray(q, dtype=np.uint8) for q in qs], sigma=sigma, Ls=Ls,
                Lidx=Lidx, kBound=-1, seedK=20, maxBucket=256, spread=1024, thr=None, readList=None, firstPair=0)
    case.update(kw)
    if case.get("numReads") is None:
        case["numReads"] = len(case["readList"]) if case["readList"] is not None else len(qs) - case["firstPair"]
    return case


def expected_plan(case, cap):
    target = case.setdefault("_target", R.Target(case["t"]))
    out = []
    for slot in range(case["numReads"]):
        pair = case["readList"][slot] if case["readList"] is not None else case["firstPair"] + slot
        q = case["qs"][pair]
        t = case["thr"][slot] if case["thr"] is not None else R.seed_threshold(len(q), case["kBound"], case["Ls"],
                                                                              case["seedK"])
        state, thr, wins = R.plan_read(target, q, t, case["Ls"], case["Lidx"], case["sigma"], case["maxBucket"],
                                       case["spread"], cap)
        out.append((pair, state, thr, wins))
    return out


def instances_of(case):
    """(level, maxLen) of every planning instance the choice (eb_dispatch.h: with_seed_plan_instance) can pick for the
    case: level 0 with the true longest read (16-lane groups when all seeds fit), level 0 with unknown lengths (warps),
    the last level (warps, CAP 4096)."""
    maxLen = max((len(q) for q in case["qs"]), default=0)
    return [(0, maxLen), (0, 0), (2, maxLen)]


def check_plan(probe, case, level, maxLen, winCap=None):
    """Runs one launch and compares it with the reference; returns (instance, reads with windows, windows)."""
    cap = 4096 if level >= 2 else 256
    exp = expected_plan(case, cap)
    total = sum(len(w) for _p, s, _t, w in exp if s == R.SEED_WINDOWS)
    winCap = total if winCap is None else winCap
    plan, win, count, inst = probe.plan(case, case.setdefault("_bs", R.index(case["t"], case["Lidx"], case["sigma"])[0]
                                                              .astype(np.int32)),
                                        case.setdefault("_pos", np.argsort(R.padded_keys(case["t"], case["Lidx"],
                                                                                         case["sigma"]),
                                                                           kind="stable").astype(np.int32)),
                                        level, maxLen, winCap)
    assert inst[0] == cap
    what = "instance %s, level %d, maxLen %d" % (inst, level, maxLen)
    assert count == total, what
    used = np.zeros(max(winCap, 1), dtype=bool)
    overflow = total > winCap
    for slot, (pair, state, thr, wins) in enumerate(exp):
        first, cnt, gstate, gthr = (int(x) for x in plan[slot])
        where = "%s, slot %d (pair %d, m %d, t %d)" % (what, slot, pair, len(case["qs"][pair]), thr)
        assert gthr == thr, where
        if overflow and gstate == R.SEED_SATURATED and state == R.SEED_WINDOWS:
            assert cnt == 0, where  # its windows did not fit (which reads these are depends on atomic order)
            continue
        assert (gstate, cnt) == (state, len(wins)), where
        if cnt:
            assert 0 <= first and first + cnt <= winCap, where
            assert not used[first:first + cnt].any(), where
            used[first:first + cnt] = True
            got = [tuple(int(x) for x in win[1:, w]) for w in range(first, first + cnt)]
            assert list(win[0, first:first + cnt]) == [pair] * cnt, where
            assert got == wins, where
    return inst, sum(1 for e in exp if e[1] == R.SEED_WINDOWS), total


def planted(rng, sigma, n_bg, copies, gap=(40, 200)):
    """Target of random codes with the given motifs laid in: copies is a list of (motif, count); returns
    (target, {motif index: [positions]}).  Copies are shuffled and separated by random gaps."""
    order = [i for i, (_m, k) in enumerate(copies) for _ in range(k)]
    rng.shuffle(order)
    parts, at, where = [rand_codes(rng, n_bg, sigma)], n_bg, {}
    for i in order:
        g = rand_codes(rng, rng.randint(*gap), sigma)
        parts += [g, copies[i][0]]
        at += len(g)
        where.setdefault(i, []).append(at)
        at += len(copies[i][0])
    parts.append(rand_codes(rng, 50, sigma))
    return np.concatenate(parts), where


def fresh_motif(rng, sigma, L, used):
    while True:
        m = rand_codes(rng, L, sigma)
        if bytes(m) not in used:
            used.add(bytes(m))
            return m


def seeds_read(seeds, Ls, stride, foreign):
    """A read whose seed j (at j * stride) is seeds[j] (None: foreign codes, never looked up), filled with foreign codes."""
    q = np.full(stride * len(seeds), foreign, dtype=np.uint8)
    for j, s in enumerate(seeds):
        if s is not None:
            q[j * stride:j * stride + Ls] = s
    return q


def counted_case(rng, counts_per_read, sigma=4, Ls=12, Lidx=10, stride=None, gap=(40, 200), **kw):
    """Reads built from seeds with a known number of planted copies each (0: a word absent from the target,
    None: a seed with a foreign code).  Chance occurrences elsewhere are counted by the reference like any other."""
    stride = stride or Ls
    used, copies, reads = set(), [], []
    for counts in counts_per_read:
        seeds = []
        for k in counts:
            if k is None:
                seeds.append(None)
                continue
            m = fresh_motif(rng, sigma, Ls, used)
            if k:
                copies.append((m, k))
            seeds.append(m)
        reads.append(seeds)
    t, _ = planted(rng, sigma, 2000, copies, gap)
    qs = [seeds_read(s, Ls, stride, sigma) for s in reads]
    thr = [len(s) - 1 for s in reads]
    return make_case(t, qs, sigma, Ls, Lidx, thr=thr, seedK=max(thr), maxBucket=kw.pop("maxBucket", 8192), **kw)


def edge_cases(seed):
    """(name, case) of the corners of seed_plan_read."""
    rng = random.Random(seed)
    out = []
    # t + 1 seeds of reads copied from a target with few chance occurrences (several rounds of lookups for t+1 > W)
    t = rand_codes(rng, 30000, 4)
    qs, thr = [], []
    for seeds in (1, 2, 15, 16, 17, 31, 32, 33, 65):
        for _ in range(3):
            m = seeds * 12 + rng.randrange(12)
            a = rng.randrange(0, len(t) - m)
            q = t[a:a + m].copy()
            for _x in range(rng.choice([0, 1, 3])):  # a few seeds lose their occurrence
                q[rng.randrange(m)] = rng.randrange(4)
            qs.append(q)
            thr.append(seeds - 1)
    out.append(("seeds per read", make_case(t, qs, 4, 12, 10, thr=thr, seedK=64)))
    # long queries, several hundred seeds, as the long-HW seeds use the last level
    qs = [t[a:a + 4000].copy() for a in (0, 9000, len(t) - 4000)]
    out.append(("hundreds of seeds", make_case(t, qs, 4, 12, 10, thr=[330, 300, 199], seedK=1024)))
    # empty ranges between non-empty ones, ranges longer than 4 W entries, totals of 4 W and 4 W + 1 (W = 16, 32)
    reads = [[3, 0, 5, 0, 0, 2, 0, 1], [0, 0, 0, 7], [0, 2, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 4],
             [130], [0, 140, 0, 3], [64], [65], [40, 24], [40, 25], [128], [129], [100, 0, 28], [100, 0, 29],
             [0] * 16 + [5], [None, 3, None, 0, 4]]
    out.append(("range walks", counted_case(rng, reads, Ls=12, Lidx=10)))
    out.append(("range walks, Ls < Lidx", counted_case(rng, reads, Ls=9, Lidx=10)))
    out.append(("range walks, Ls = Lidx", counted_case(rng, reads, Ls=10, Lidx=10)))
    # candidates around CAP (256 at levels 0 / 1, 4096 at the last) and around powers of two; spaced copies: as many windows
    reads = [[k] for k in (31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257)] + [[200, 56], [200, 57]]
    out.append(("candidates around 256", counted_case(rng, reads, gap=(20, 80))))
    reads = [[k] for k in (4095, 4096, 4097)] + [[2000, 2096], [2000, 2097]]
    out.append(("candidates around 4096", counted_case(rng, reads, gap=(5, 30))))
    # windows per read around W and 2 W + 1: copies far apart (one window each), t small
    reads = [[k, None] for k in (15, 16, 17, 31, 32, 33, 63, 65)]
    out.append(("windows per read", counted_case(rng, reads, gap=(150, 300))))
    # a seed's range right at maxBucket and one past it
    c = counted_case(rng, [[50, 2], [51, 2], [49, 1]], maxBucket=8192)
    out.append(("maxBucket", dict(c, maxBucket=R.Target(c["t"]).range_length(bytes(c["qs"][0][:10])))))
    # occurrences at p = 0, p = n - Ls and in the padded tail; windows clipped at both ends; overlapping windows
    sigma, Ls, Lidx = 20, 4, 4
    body = rand_codes(rng, 3000, sigma)
    head, tail = body[:Ls].copy(), body[-Ls:].copy()
    pad = np.concatenate([body[-2:], np.zeros(Ls - 2, dtype=np.uint8)])  # a key of the last positions, padded with 0
    qs = [np.concatenate([rand_codes(rng, 4 * Ls, sigma), head]),          # last seed at p = 0: clipped at 0
          np.concatenate([tail, rand_codes(rng, 4 * Ls, sigma)]),          # first seed at p = n - Ls: past n - 1
          np.concatenate([pad, rand_codes(rng, 4 * Ls, sigma)]),            # only the padded tail holds the key
          np.concatenate([head, rand_codes(rng, 3 * Ls, sigma), tail]),
          body[:8 * Ls].copy(), body[-8 * Ls:].copy(), body[1000:1000 + 9 * Ls].copy()]
    thr = [4, 4, 4, 4, 7, 7, 8]
    out.append(("target ends", make_case(body, qs, sigma, Ls, Lidx, thr=thr, seedK=8)))
    rep = rand_codes(rng, 12, 4)
    near = np.concatenate([rand_codes(rng, 500, 4)] + [np.concatenate([rep, rand_codes(rng, d, 4)])
                                                       for d in (1, 5, 20, 40, 60, 70, 90, 130, 250, 256, 257, 300)]
                          + [rand_codes(rng, 500, 4)])
    qs = [np.concatenate([rep, rand_codes(rng, 12 * tt, 4)]) for tt in (0, 3, 7, 15, 16, 20)]
    out.append(("neighbouring candidates", make_case(near, qs, 4, 12, 10, thr=[0, 3, 7, 15, 16, 20], seedK=20)))
    out.append(("neighbouring candidates, narrow spread",
                make_case(near, qs, 4, 12, 10, thr=[0, 3, 7, 15, 16, 20], seedK=20, spread=100)))
    # codes >= sigma inside seeds
    qs = []
    for _ in range(12):
        a = rng.randrange(0, len(t) - 150)
        q = t[a:a + 150].copy()
        for _x in range(rng.choice([1, 2, 6])):
            q[rng.randrange(150)] = rng.choice([4, 5, 255])
        qs.append(q)
    out.append(("foreign codes", make_case(t, qs, 4, 12, 10)))
    # numReads not a multiple of the reads per warp or CTA; thr = -1 next to live reads; readList and firstPair
    qs = [t[a:a + rng.choice([60, 100, 150, 250])].copy() for a in rng.sample(range(len(t) - 300), 40)]
    for nr in (1, 3, 5, 9, 17, 33):
        thr = [rng.choice([-1, 0, 2, 5, 9]) if len(qs[i]) >= 24 else -1 for i in range(nr)]
        thr = [min(x, len(qs[i]) // 12 - 1) for i, x in enumerate(thr)]
        out.append(("%d reads" % nr, make_case(t, qs, 4, 12, 10, thr=thr, numReads=nr)))
    rl = rng.sample(range(40), 23)
    out.append(("read list", make_case(t, qs, 4, 12, 10, readList=rl, kBound=6)))
    out.append(("first pair", make_case(t, qs, 4, 12, 10, firstPair=7, seedK=9)))
    return out


def random_cases(seed, count):
    """Random batches over targets shaped like cases.filter_cases: repeats, tandem stretches, protein and two-letter
    alphabets, free and bounded k."""
    rng = random.Random(seed)
    out = []
    for _ in range(count):
        sigma = rng.choice([4, 4, 5, 20, 2])
        Ls = {2: 20, 4: 10, 5: 9, 20: 4}[sigma] - rng.choice([0, 0, 2])
        Lidx = {2: 16, 4: 9, 5: 8, 20: 4}[sigma] + rng.choice([-1, 0, 0])
        shape = rng.random()
        if shape < 0.15:
            unit = rand_codes(rng, rng.choice([5, 13, 31]), sigma)
            t = np.tile(unit, 4000 // len(unit))
            t[rng.sample(range(len(t)), 40)] = rand_codes(rng, 40, sigma)
        else:
            t = rand_codes(rng, rng.choice([3000, 8000, 20000]), sigma)
            if shape < 0.5:
                seg = t[100:100 + rng.choice([200, 600])].copy()
                for _c in range(rng.choice([1, 2, 4])):
                    at = rng.randrange(len(t))
                    t = np.concatenate([t[:at], seg, t[at:]])
        qs = []
        for _ in range(rng.choice([8, 40, 100])):
            L = rng.choice([48, 64, 100, 150, 200, 256])
            a = rng.randrange(0, len(t) - L)
            q = t[a:a + L].copy() if rng.random() < 0.8 else rand_codes(rng, L, sigma)
            for _x in range(rng.choice([0, 1, 3, 8])):
                q[rng.randrange(L)] = rng.randrange(sigma)
            qs.append(q)
        out.append(make_case(t, qs, sigma, Ls, Lidx, kBound=rng.choice([-1, -1, 3, 10, 40]),
                             seedK=rng.choice([20, 20, 12, 40]), maxBucket=rng.choice([64, 256, 2048]),
                             spread=rng.choice([1024, 300])))
    return out


def run_plan_cases(probe, cases):
    """Every case on every instance; returns the instances that ran and how many reads / windows were checked."""
    seen, reads, wins = set(), 0, 0
    for name, case in cases:
        for level, maxLen in instances_of(case):
            try:
                inst, r, w = check_plan(probe, case, level, maxLen)
            except AssertionError as e:
                raise AssertionError("%s: %s" % (name, e)) from None
            seen.add(inst)
            reads += r
            wins += w
    return [list(i) for i in sorted(seen)], reads, wins


def run_overflow_cases(probe, seed):
    """Window caps below the total: winCount stays the total, reads keep their exact windows or are saturated."""
    rng = random.Random(seed)
    checked = 0
    for case in random_cases(seed, 6):
        for level, maxLen in instances_of(case):
            exp = expected_plan(case, 4096 if level >= 2 else 256)
            total = sum(len(w) for _p, s, _t, w in exp if s == R.SEED_WINDOWS)
            if total < 4:
                continue
            for winCap in (total - 1, total // 2, 1):
                check_plan(probe, case, level, maxLen, winCap=winCap)
                checked += 1
    return checked


def lane_group_driver(which, fn, seed):
    """Runs fn(probe, seed) in a subprocess with the planner's lane groups at device width; returns its JSON result."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_seed_stage as T\n"
            "print(json.dumps(T.%s(T.Probe(%r), %d)))\n") % (REPO, TESTS_DIR, fn, which, seed)
    env = dict(os.environ, EDLIB_EMUL_SEED_GROUP="device")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def edges(probe, seed):
    return run_plan_cases(probe, edge_cases(seed))


def randoms(probe, seed):
    return run_plan_cases(probe, [("random batch %d" % i, c) for i, c in enumerate(random_cases(seed, 8))])


def overflows(probe, seed):
    return run_overflow_cases(probe, seed)


ALL_INSTANCES = [[256, 128, 16], [256, 128, 32], [4096, 64, 32]]


# ---------------------------------------------------------------------------------------------------------------
# index cases
# ---------------------------------------------------------------------------------------------------------------

def scan_inputs(count, seed):
    rng = np.random.default_rng(seed + count)
    yield np.zeros(count, dtype=np.int32)
    hi = max(1, min(64, (2 ** 31 - 1) // max(count, 1)))  # counts of an index: the total stays within int32
    yield rng.integers(0, hi, size=count, dtype=np.int32)


def check_scan(probe, count, seed=5):
    for data in scan_inputs(count, seed):
        got = probe.scan(data)
        want = np.zeros(count + 1, dtype=np.int64)
        np.cumsum(data, out=want[1:])
        assert np.array_equal(got, want), (count, np.flatnonzero(got != want)[:5])


def ecoli_codes():
    from edlib_b200 import workloads
    g = workloads.ecoli_genome()
    lut = np.zeros(256, dtype=np.uint8)
    for i, ch in enumerate(b"ACGT"):
        lut[ch] = i
    return lut[g]


def index_targets():
    rng = np.random.default_rng(11)
    yield "5 kbp", rng.integers(0, 4, 5000, dtype=np.uint8), 4
    yield "E. coli", ecoli_codes(), 4
    yield "9 Mbp", rng.integers(0, 4, 9_000_000, dtype=np.uint8), 4
    yield "20 letters", rng.integers(0, 20, 30000, dtype=np.uint8), 20


def check_build_index(probe, name, tcodes, ncodes):
    ok, Lidx, sigma, bs, pos = probe.build_index(tcodes, ncodes)
    assert ok, name
    assert sigma ** Lidx <= max(2 * len(tcodes), 4096) < sigma ** (Lidx + 1) or Lidx == 16, (name, Lidx)
    want, keys = R.index(tcodes, Lidx, sigma)
    assert np.array_equal(bs, want), name
    assert R.same_positions(bs, pos, keys), name
    return Lidx, len(bs) - 1


def check_short_targets(probe):
    """Targets a few symbols longer than Lidx, and seed lengths below, at and above Lidx."""
    rng = np.random.default_rng(3)
    for sigma, Lidx in ((4, 6), (20, 3), (2, 12)):
        for n in (Lidx + 1, Lidx + 3, Lidx + 7):
            t = rng.integers(0, sigma, n, dtype=np.uint8)
            for numPos in (n, n - 2):
                bs, pos = probe.index(t, Lidx, sigma, numPos)
                want, keys = R.index(t, Lidx, sigma, numPos)
                assert np.array_equal(bs, want), (sigma, Lidx, n, numPos)
                assert R.same_positions(bs, pos, keys), (sigma, Lidx, n, numPos)
            for Ls in (Lidx - 2, Lidx, Lidx + 2):  # the reads are the whole target and its pieces
                qs = [t, t[1:], np.concatenate([t, t])]
                thr = [min(1, len(q) // Ls - 1) for q in qs]  # as many seeds as fit (-1: none, the read is left out)
                case = make_case(t, qs, sigma, Ls, Lidx, thr=thr, seedK=1)
                for level, maxLen in instances_of(case):
                    check_plan(probe, case, level, maxLen)


# ---------------------------------------------------------------------------------------------------------------
# CPU: the emulation, serially and with lane groups
# ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def emul():
    return Probe("emul")


@pytest.mark.parametrize("count", SCAN_COUNTS)
def test_scan_emul(emul, count):
    check_scan(emul, count)


def test_index_emul(emul):
    for name, tcodes, ncodes in index_targets():
        if len(tcodes) <= 5_000_000:
            check_build_index(emul, name, tcodes, ncodes)
    check_short_targets(emul)


def test_plan_edges_serial(emul):
    seen, reads, _w = edges(emul, 1)
    assert seen == ALL_INSTANCES and reads > 100


def test_plan_random_serial(emul):
    seen, reads, _w = randoms(emul, 2)
    assert reads > 200


def test_plan_window_overflow_serial(emul):
    assert overflows(emul, 3) > 20


def test_plan_edges_lane_groups():
    seen, reads, _w = lane_group_driver("emul", "edges", 1)
    assert seen == ALL_INSTANCES and reads > 100


def test_plan_random_lane_groups():
    seen, reads, _w = lane_group_driver("emul", "randoms", 4)
    assert reads > 200


def test_plan_window_overflow_lane_groups():
    assert lane_group_driver("emul", "overflows", 3) > 20


# ---------------------------------------------------------------------------------------------------------------
# GPU: the CUDA backend, the same generators
# ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def cuda():
    return Probe("cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("count", SCAN_COUNTS + [1 << 28])  # 2^28: the most keys build_seed_index makes
def test_scan_gpu(cuda, count):
    check_scan(cuda, count)


@pytest.mark.gpu
def test_index_gpu(cuda):
    seen = {}
    for name, tcodes, ncodes in index_targets():
        seen[name] = check_build_index(cuda, name, tcodes, ncodes)
    # E. coli: 4^11 keys, exactly 1024 scan tiles; 9 Mbp: 4^12 keys, 4096 tiles (four per thread of the top level)
    assert seen["E. coli"] == (11, 4 ** 11) and seen["9 Mbp"] == (12, 4 ** 12)
    check_short_targets(cuda)


@pytest.mark.gpu
def test_plan_edges_gpu(cuda):
    seen, reads, wins = edges(cuda, 1)
    print("seed_plan_kernel instances (CAP, THREADS, GW):", seen, "reads with windows:", reads, "windows:", wins)
    assert seen == ALL_INSTANCES and reads > 100


@pytest.mark.gpu
def test_plan_random_gpu(cuda):
    seen, reads, _w = randoms(cuda, 2)
    assert seen == ALL_INSTANCES and reads > 200


@pytest.mark.gpu
def test_plan_window_overflow_gpu(cuda):
    assert overflows(cuda, 3) > 20


# Decisions of the filter per batch, product against emulation: the planner's losses do not show in results (a read it
# drops is decided later, the same way), so the counters are compared too.  The prefix stages are off: their range
# lists depend on the chunking of the sweep, which follows the SM count.  The device-driven first level saturates reads
# whose windows overflow its job arrays in atomic order; its arrays hold reads * 6 + 4096 windows and a read has at
# most 256 candidates there, so batches of at most 16 reads cannot overflow them.
DECISIONS = """
import sys, json, ctypes as C
sys.path.insert(0, %r); sys.path.insert(0, %r)
import cases, parity, test_strands as S
from helpers import product
from test_engine_emul import load_emul
lib = product() if sys.argv[1] == "cuda" else load_emul()
chk = parity.checker()
out = []
for gen, seed, count in (("filter_cases", 26, 12), ("small_k_cases", 101, 8), ("stream_cases", 7, 6)):
    for c in getattr(cases, gen)(seed, count):
        for b in range(0, len(c["qs"]), 16):
            qs, ts = c["qs"][b:b + 16], c["ts"][b:b + 16]
            st, res = lib.align_batch(qs, ts, c["k"], c["mode"], c["task"], c["eqs"])
            assert st == 0
            s = S.Stats()
            lib.lib.edlibB200LastStats(C.byref(s))
            for i, (q, t) in enumerate(zip(qs, ts)):
                assert res[i] == chk.align(q, t, c["k"], c["mode"], c["task"], c["eqs"]), (gen, b + i)
            out.append([s.filterWindows, s.filterDecided, s.filterFallback])
print(json.dumps(out))
""" % (REPO, TESTS_DIR)


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [{}, {"EDLIB_B200_DEVICE_STAGE": "0"}], ids=["device-level", "host-levels"])
def test_filter_decisions_match_the_emulation(extra):
    env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0",
               EDLIB_B200_K1_MIN_GROUP="4", EDLIB_B200_FILTER_K0="0", EDLIB_B200_FILTER_K1="0", **extra)
    got = {}
    for which in ("cuda", "emul"):
        out = subprocess.run([sys.executable, "-c", DECISIONS, which], env=env, capture_output=True, text=True,
                             timeout=900)
        assert out.returncode == 0, out.stderr[-4000:]
        got[which] = json.loads(out.stdout.strip().splitlines()[-1])
    assert len(got["cuda"]) == len(got["emul"]) > 50
    assert sum(w for w, _d, _f in got["cuda"]) > 0
    for i, (a, b) in enumerate(zip(got["cuda"], got["emul"])):
        assert a == b, (i, "filterWindows, filterDecided, filterFallback", a, b)
