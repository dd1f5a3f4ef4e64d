"""All end locations within k (edlibB200FindHits, edlib_b200.find_hits) against a brute-force last row.

The reference below computes the exact HW last row D(c) in numpy, one DP row at a time; every case compares counts,
columns, scores and strands with it exactly.  CPU tests run the engine on the emulated kernels in subprocesses with
forced tunables, and `filterDecided` / `filterFallback` show which route ran (seed windows / whole-target sweep); the
-m gpu tests run the product library, also against the reference build (oracle/_ref)."""
import ctypes as C
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from edlib_b200._ffi import REPO, EdlibLib, Hits, make_config
from helpers import mutate, rand_seq

HERE = os.path.dirname(os.path.abspath(__file__))
EMUL_HITS_DIR = os.path.join(HERE, "emul_hits")


def load_emul_hits():
    """The kernel emulation of tests/emul with the kernels of the hit lists (tests/emul_hits)."""
    subprocess.run(["make", "-s", "-C", EMUL_HITS_DIR], check=True)
    return EdlibLib(os.path.join(EMUL_HITS_DIR, "libedlib_emul_hits.so"), has_batch=True)

_PAIRS = [b"AT", b"CG", b"RY", b"KM", b"BV", b"DH"]
_COMP = bytearray(range(256))
for _a, _b in _PAIRS:
    for _x, _y in ((_a, _b), (_a | 0x20, _b | 0x20)):
        _COMP[_x], _COMP[_y] = _y, _x
_COMP = bytes(_COMP)


def rc(q):
    return bytes(q).translate(_COMP)[::-1]


def last_row(q, t, eqs=None):
    """D(c) for c in 0..n-1: HW (free start in t), the empty substring included (D <= m)."""
    eq = np.eye(256, dtype=bool)
    for a, b in eqs or []:
        eq[a[0], b[0]] = eq[b[0], a[0]] = True
    tv = np.frombuffer(t, dtype=np.uint8)
    n = len(tv)
    j = np.arange(n, dtype=np.int64)
    prev = np.zeros(n, dtype=np.int64)  # row -1: D = 0 in every column
    for r, ch in enumerate(q):
        diag = np.empty(n, dtype=np.int64)
        diag[0] = r  # D[r-1][-1] = r
        diag[1:] = prev[:-1]
        x = np.minimum(diag + (~eq[ch][tv]).astype(np.int64), prev + 1)
        # left dependency: D[r][c] = min_j<=c (X[j] + c - j), and the boundary D[r][-1] = r + 1
        prev = np.minimum(j + np.minimum.accumulate(x - j), r + 2 + j)
    return prev


_rows = {}


def cached_row(q, t, eqs):
    key = (q, len(t), hash(t), repr(eqs))
    if key not in _rows:
        _rows[key] = last_row(q, t, eqs)
    return _rows[key]


def expected(qs, t, k, both, cap, eqs=None):
    out = []
    for q in qs:
        hits = []
        for s, qq in enumerate([q, rc(q)] if both else [q]):
            d = cached_row(qq, t, eqs)
            cols = np.nonzero(d <= k)[0]
            hits += [(int(c), int(d[c]), s) if both else (int(c), int(d[c])) for c in cols]
        out.append({"count": len(hits), "hits": hits[:cap]})
    return out


class Stats(C.Structure):  # include/edlib_b200.h EdlibB200Stats
    _fields_ = [("kernelMs", C.c_double), ("k1Ms", C.c_double), ("launches", C.c_int), ("filterWindows", C.c_int),
                ("h2dBytes", C.c_longlong), ("d2hBytes", C.c_longlong), ("k1Cells", C.c_longlong), ("wCells", C.c_longlong),
                ("filterDecided", C.c_longlong), ("filterFallback", C.c_longlong)]


def stats(lib):
    s = Stats()
    lib.lib.edlibB200LastStats(C.byref(s))
    return s


def check(lib, qs, t, k, both=False, cap=1 << 40, eqs=None):
    """Runs one call, compares with the brute force; returns (decided, fallback, windows) of the call."""
    st, got = lib.find_hits(qs, t, k, both, cap, eqs)
    lib.lib.edlibB200LastError.restype = C.c_char_p
    assert st == 0, lib.lib.edlibB200LastError()
    exp = expected(qs, t, k, both, cap, eqs)
    for i, (g, e) in enumerate(zip(got, exp)):
        assert g == e, dict(query=i, k=k, m=len(qs[i]), n=len(t), both=both, cap=cap, got_count=g["count"],
                            exp_count=e["count"], got=g["hits"][:12], exp=e["hits"][:12])
    s = stats(lib)
    return s.filterDecided, s.filterFallback, s.filterWindows


# ---------------------------------------------------------------------------------------------------------------------
# CPU: emulated kernels under the real engine, one subprocess per set of tunables
# ---------------------------------------------------------------------------------------------------------------------
DRIVER = (
    "import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
    "import test_hits as H\n"
    "lib = H.load_emul_hits()\n"
    "print(json.dumps(H.SCENARIOS[sys.argv[1]](lib)))\n"
) % (REPO, HERE)


def run_scenario(name, env=None):
    e = dict(os.environ, **(env or {}))
    out = subprocess.run([sys.executable, "-c", DRIVER, name], env=e, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def genome(rng, n):
    return rand_seq(rng, n, b"ACGT")


def reads_of(rng, t, count, m, rate):
    out = []
    for _ in range(count):
        a = rng.randrange(0, len(t) - m)
        q = mutate(rng, t[a:a + m], rate, b"ACGT")[:256] or b"A"
        out.append(rc(q) if rng.random() < 0.5 else q)
    return out


def sc_levels(lib):
    """150 bp reads over a 200 kbp target: k at and just above each seed level's threshold, and above every level."""
    rng = random.Random(1)
    t = genome(rng, 200_000)
    qs = reads_of(rng, t, 12, 150, 0.04) + [rand_seq(rng, 150, b"ACGT")]
    res = {}
    for k in (0, 3, 10, 11, 12, 13, 15, 16, 17, 18, 21, 30):
        res[k] = check(lib, qs, t, k, both=(k % 2 == 1))
    return res


def sc_short_target(lib):
    """A target below filterMinTarget: the whole-target sweep only; chunk borders and halos, hits at 0 and n - 1."""
    rng = random.Random(2)
    t = genome(rng, 9_000)
    qs = [t[:40], t[-40:], t[2030:2100], rc(t[4000:4064]), t[1000:1001], t[10:41], t[100:132], t[200:233],
          mutate(rng, t[5000:5256], 0.05, b"ACGT")[:256], b"ACGT" * 16]
    res = {}
    for k in (0, 2, 5):
        res[k] = check(lib, qs, t, k, both=True)
    res["all"] = check(lib, [b"A", b"ACG", t[77:108]], t, 40)  # k >= m: every column
    return res


def sc_equalities(lib):
    """Non-transitive equalities (table path: whole-target sweep) and transitive ones (collapsed: seed route)."""
    rng = random.Random(3)
    t = genome(rng, 120_000)
    t = bytes(c | 0x20 if rng.random() < 0.2 else c for c in t)
    qs = [bytes(c | 0x20 if rng.random() < 0.3 else c for c in q) for q in reads_of(rng, t.upper(), 8, 120, 0.03)]
    fold = [(bytes([c]), bytes([c | 0x20])) for c in b"ACGT"]
    wild = [(b"N", bytes([c])) for c in b"ACGT"]
    qn = [b"".join(b"N" if rng.random() < 0.05 else bytes([c]) for c in q) for q in qs[:4]]
    return {"fold": check(lib, qs, t, 6, eqs=fold), "wild": check(lib, qn + qs[:2], t, 4, eqs=wild)}


def sc_repeats(lib):
    """Homopolymers and tandem repeats (windows with many tied columns), saturated plans, neighbouring occurrences."""
    rng = random.Random(4)
    t = bytearray(genome(rng, 150_000))
    t[1000:3000] = b"A" * 2000
    t[10_000:14_000] = b"ACGTTG" * 666 + b"ACGT"
    unit = genome(rng, 100)
    for a in range(50_000, 50_000 + 40 * 130, 130):  # neighbouring copies whose windows meet
        t[a:a + 100] = mutate(rng, unit, 0.02, b"ACGT")[:100].ljust(100, b"C")
    t = bytes(t)
    qs = [b"A" * 64, b"A" * 150, (b"ACGTTG" * 30)[:150], unit, rc(unit), t[49_990:50_140], b"AC" * 70]
    return {k: check(lib, qs, t, k, both=True) for k in (0, 4, 10)}


def sc_boundaries(lib):
    """m at 1, 31, 32, 33, 64, 256; caps of 0, 1 and exactly the count; palindromes on both strands."""
    rng = random.Random(5)
    t = genome(rng, 100_000)
    qs = [t[5:6], t[70_000:70_031], t[100:132], t[-33:], t[:64], t[8000:8256], mutate(rng, t[3000:3256], 0.02, b"ACGT")[:256],
          b"ACGTTAACGT" * 3 + b"GAATTC"]
    res = {"plain": check(lib, qs, t, 3, both=True)}
    st, full = lib.find_hits(qs, t, 3, True)
    assert st == 0
    for cap in (0, 1, max(r["count"] for r in full)):
        res["cap%d" % cap] = check(lib, qs, t, 3, both=True, cap=cap)
    counts = [r["count"] for r in full]
    res["exact"] = check(lib, qs, t, 3, both=True, cap=min(c for c in counts if c > 0))
    return res


def sc_invalid(lib):
    """Wrong mode / task, k < 0, m = 0, m > 256, NULL hits: EDLIB_STATUS_ERROR, nothing left allocated."""
    fn = lib.lib.edlibB200FindHits
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.c_char_p, C.c_int, type(make_config()[0]),
                   C.c_int, C.c_longlong, C.POINTER(Hits)]
    lib.lib.edlibB200LastError.restype = C.c_char_p
    t = b"ACGT" * 100
    out = {}
    for name, qs, k, mode, task, null in [("mode", [b"ACGT"], 1, 0, 0, False), ("task", [b"ACGT"], 1, 2, 1, False),
                                          ("k", [b"ACGT"], -1, 2, 0, False), ("empty", [b""], 1, 2, 0, False),
                                          ("long", [b"A" * 257], 1, 2, 0, False), ("null", [b"ACGT"], 1, 2, 0, True)]:
        cfg, _ = make_config(k, mode, task)
        h = Hits()
        h.numQueries = 99
        qp = (C.c_char_p * 1)(*qs)
        ql = (C.c_int * 1)(*[len(q) for q in qs])
        st = fn(qp, ql, 1, t, len(t), cfg, 0, 10, None if null else C.byref(h))
        assert st == 1, name
        assert not h.counts and not h.offsets and not h.columns and not h.scores and not h.strands, name
        out[name] = lib.lib.edlibB200LastError().decode()
        assert out[name].startswith("edlibB200FindHits"), out[name]
    st, res = lib.find_hits([], t, 2)
    assert st == 0 and res == []
    return out


SCENARIOS = {"levels": sc_levels, "short_target": sc_short_target, "equalities": sc_equalities, "repeats": sc_repeats,
             "boundaries": sc_boundaries, "invalid": sc_invalid}

FORCED = {"EDLIB_B200_FILTER_MIN_LEVEL_READS": "0"}


def test_brute_force_reference():
    """The numpy last row against the reference's rule on small cases: min(D) and its columns are edlibAlign's."""
    import parity
    rng = random.Random(9)
    chk = parity.checker()
    for _ in range(60):
        t = rand_seq(rng, rng.randrange(1, 300), b"ACG")
        q = rand_seq(rng, rng.randrange(1, 40), b"ACG")
        d = last_row(q, t)
        r = chk.align(q, t, -1, 2, 0)
        assert int(d.min()) == r["editDistance"]
        assert [int(c) for c in np.nonzero(d == d.min())[0]] == [c for c in r["endLocations"] if c >= 0]


def test_seed_levels_emul():
    res = run_scenario("levels", FORCED)
    # (decided, fallback, windows) per k over 13 reads: low k on the seed windows, k above every level swept in full
    assert res["0"][0] > 0 and res["0"][2] > 0
    assert res["10"][0] > 0 and res["17"][0] > 0
    assert res["21"] == [0, 26, 0] and res["30"] == [0, 13, 0]


def test_one_seed_level_emul():
    res = run_scenario("levels", dict(FORCED, EDLIB_B200_DEVICE_STAGE="0", EDLIB_B200_FILTER_SEED_LEVELS="1"))
    assert res["15"] == [0, 26, 0] and res["13"][0] > 0  # level 0 of a 200 kbp target: 10-mers, t <= 14


def test_no_seeds_emul():
    res = run_scenario("levels", dict(FORCED, EDLIB_B200_FILTER_SEED_K="0"))
    assert all(v[0] == 0 and v[2] == 0 for v in res.values())


def test_short_target_emul():
    res = run_scenario("short_target", {"EDLIB_B200_K1_MIN_CHUNK": "256"})
    assert all(v[0] == 0 and v[1] > 0 for v in res.values())


def test_equalities_emul():
    res = run_scenario("equalities", FORCED)
    assert res["fold"][0] == 8 and res["wild"] == [0, 6, 0]


def test_repeats_emul():
    res = run_scenario("repeats", FORCED)
    assert res["10"][1] > 0  # the homopolymer reads saturate their plans
    res = run_scenario("repeats", dict(FORCED, EDLIB_B200_FILTER_SEED_BUCKET="2"))
    assert res["4"][1] > 0


def test_boundaries_emul():
    run_scenario("boundaries", FORCED)


def test_invalid_input_emul():
    res = run_scenario("invalid")
    assert len(res) == 6


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the product library
# ---------------------------------------------------------------------------------------------------------------------
def product_lib():
    from helpers import product
    return product()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_scenarios_gpu(name):
    SCENARIOS[name](product_lib())


@pytest.mark.gpu
def test_python_entry_gpu():
    import edlib_b200
    rng = random.Random(6)
    t = genome(rng, 80_000)
    qs = reads_of(rng, t, 6, 100, 0.03)
    lib = product_lib()
    for strands, both in (("forward", False), ("both", True)):
        got = edlib_b200.find_hits(qs, t, 5, strands=strands, max_hits=7)
        st, raw = lib.find_hits(qs, t, 5, both, 7)
        assert st == 0
        if both:
            raw = [{"count": r["count"], "hits": [(c, s, "-" if d else "+") for c, s, d in r["hits"]]} for r in raw]
        assert got == raw
        assert all(len(r["hits"]) == min(7, r["count"]) for r in got)
    with pytest.raises(Exception):
        edlib_b200.find_hits([b"A" * 300], t, 3)


def ecoli_case(k):
    """The E. coli genome, the reference's reads of at most 256 bp and 200 seeded config-2 reads (150 bp, 3 % errors)."""
    from edlib_b200 import workloads
    genome = workloads.ecoli_genome()
    with open(os.path.join(HERE, "golden", "ecoli_reads.json")) as f:
        fx = json.load(f)
    golden = [r["seq"].encode("ascii") for _, r in sorted(fx["reads"].items()) if 0 < len(r["seq"]) <= 256]
    seeded = [bytes(r) for r in workloads.reads_of(genome, 200, seed=100 + k)]
    return genome.tobytes(), golden + seeded


@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 3, 10, 20])
def test_ecoli_against_reference_gpu(k):
    """The reference's E. coli reads and seeded config-2-style reads over the 4.63 Mbp genome: the least hit score and
    its columns are edlibAlign's distance and end locations (reference build), and single columns match the reversed
    SHW rule of include/edlib_b200.h on a sample."""
    from helpers import have_ref, ref
    if not have_ref():
        pytest.skip("reference build not available")
    genome_bytes, reads = ecoli_case(k)
    lib = product_lib()
    st, got = lib.find_hits(reads, genome_bytes, k, False, 1 << 40)
    assert st == 0
    r = ref()
    rng = random.Random(k)
    for i, q in enumerate(reads):
        e = r.align(q, genome_bytes, k, 2, 0)
        hits = got[i]["hits"]
        assert len(hits) == got[i]["count"]
        if e["editDistance"] < 0:
            assert hits == [], i
            continue
        best = min(s for _, s in hits)
        assert best == e["editDistance"], i
        assert [c for c, s in hits if s == best] == [c for c in e["endLocations"] if c >= 0], i
        assert [c for c, _ in hits] == sorted(set(c for c, _ in hits))
        if i % 25 == 0:  # single columns: D(c) through the reversed SHW alignment of the slice ending at c
            m = len(q)
            present = dict(hits)
            for c0, _ in rng.sample(hits, min(3, len(hits))):
                for c in (c0 - 1, c0, c0 + 1):
                    if not 0 <= c < len(genome_bytes):
                        continue
                    sl = genome_bytes[max(0, c - m - k + 1):c + 1]
                    d = r.align(q[::-1], sl[::-1], -1, 1, 0)["editDistance"]
                    assert min(k + 1, present.get(c, k + 1)) == min(k + 1, d), (i, c)


@pytest.mark.gpu
def test_emulation_matches_gpu():
    """The same seeded batches through the emulation and the H100: identical hit lists."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_hits as H\n"
            "t, qs = H.seeded_batch()\n"
            "st, res = H.load_emul_hits().find_hits(qs, t, 6, True, 50)\n"
            "print(json.dumps(res))\n") % (REPO, HERE)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **FORCED))
    assert out.returncode == 0, out.stderr[-3000:]
    emul = json.loads(out.stdout.strip().splitlines()[-1])
    t, qs = seeded_batch()
    st, res = product_lib().find_hits(qs, t, 6, True, 50)
    assert st == 0
    assert [{"count": r["count"], "hits": [list(h) for h in r["hits"]]} for r in res] == emul


def seeded_batch():
    rng = random.Random(12)
    t = genome(rng, 300_000)
    return t, reads_of(rng, t, 40, 150, 0.03) + reads_of(rng, t, 10, 23, 0.0) + [rand_seq(rng, 150, b"ACGT")]


def test_backend_without_hit_kernels_refuses():
    """A backend that lacks the hit kernels (the plain kernel emulation) fails the call loudly, with nothing allocated."""
    from test_engine_emul import load_emul
    lib = load_emul()
    st, res = lib.find_hits([b"ACGTACGT"], b"ACGT" * 100, 1)
    lib.lib.edlibB200LastError.restype = C.c_char_p
    assert st == 1 and res is None
    assert b"no such kernel" in lib.lib.edlibB200LastError()
