"""All-hits search over a multi-record reference (edlibB200FindRecordHits, edlib_b200.find_hits with a list of records).

The hits of a query over several records are, by definition, its hits on each record.  Every case compares the
records call with the brute-force last row of test_hits.last_row run per record, and, for start locations and paths,
with the single-target calls of edlibB200FindHitAlignments on each record, merged in the stated order (strand, record,
column).  CPU tests run the engine on the emulated kernels (tests/emul_records) in subprocesses with forced tunables;
`filterDecided` / `filterFallback` show which route ran.  The -m gpu tests run the product library."""
import ctypes as C
import json
import mmap
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from edlib_b200._ffi import REPO, EdlibLib, RecordHits, make_config
from helpers import mutate, rand_seq
from test_hits import FORCED, cached_row, genome, rc, reads_of, stats

HERE = os.path.dirname(os.path.abspath(__file__))
EMUL_DIR = os.path.join(HERE, "emul_records")


def load_emul_records():
    """The kernel emulation of tests/emul with every kernel of the all-hits search and of record targets."""
    subprocess.run(["make", "-s", "-C", EMUL_DIR], check=True)
    return EdlibLib(os.path.join(EMUL_DIR, "libedlib_emul_records.so"), has_batch=True)


def expected(qs, recs, k, both, cap, eqs=None):
    """Per query: the brute-force hits of each record, ordered by strand, record, column; the first `cap` listed."""
    out = []
    for q in qs:
        hits = []
        for s, qq in enumerate([q, rc(q)] if both else [q]):
            for r, t in enumerate(recs):
                d = cached_row(qq, t, eqs)
                hits += [(r, int(c), int(d[c]), s) if both else (r, int(c), int(d[c])) for c in np.nonzero(d <= k)[0]]
        out.append({"count": len(hits), "hits": hits[:cap]})
    return out


def error(lib):
    lib.lib.edlibB200LastError.restype = C.c_char_p
    return lib.lib.edlibB200LastError().decode()


def check(lib, qs, recs, k, both=False, cap=1 << 40, eqs=None):
    """Runs one records call, compares with the brute force per record; returns (decided, fallback, windows)."""
    st, got = lib.find_record_hits(qs, recs, k, both, cap, eqs)
    assert st == 0, error(lib)
    s = stats(lib)
    exp = expected(qs, recs, k, both, cap, eqs)
    for i, (g, e) in enumerate(zip(got, exp)):
        assert g == e, dict(query=i, k=k, m=len(qs[i]), records=len(recs), both=both, cap=cap, got_count=g["count"],
                            exp_count=e["count"], got=g["hits"][:12], exp=e["hits"][:12])
    return s.filterDecided, s.filterFallback, s.filterWindows


def merged_single(lib, qs, recs, k, both, cap, eqs, task):
    """The single-target edlibB200FindHitAlignments calls on each record, merged in the order of the records call."""
    per = []
    for t in recs:
        st, res = lib.find_hit_alignments(qs, t, k, both, 1 << 40, eqs, task)
        assert st == 0, error(lib)
        per.append(res)
    out = []
    for i in range(len(qs)):
        items = []
        for s in ((0, 1) if both else (0,)):
            for r, res in enumerate(per):
                d = res[i]
                for j, h in enumerate(d["hits"]):
                    if both and h[2] != s:
                        continue
                    item = [(r,) + tuple(h)]
                    item.append(d["starts"][j] if "starts" in d else None)
                    item.append(d["alignments"][j] if "alignments" in d else None)
                    items.append(item)
        o = {"count": len(items), "hits": [it[0] for it in items[:cap]]}
        if task != 0:
            o["starts"] = [it[1] for it in items[:cap]]
        if task == 2:
            o["alignments"] = [it[2] for it in items[:cap]]
        out.append(o)
    return out


def check_aln(lib, qs, recs, k, both=False, cap=1 << 40, eqs=None, task=2):
    st, got = lib.find_record_hits(qs, recs, k, both, cap, eqs, task)
    assert st == 0, error(lib)
    s = stats(lib)
    exp = merged_single(lib, qs, recs, k, both, cap, eqs, task)
    for i, (g, e) in enumerate(zip(got, exp)):
        assert g == e, dict(query=i, k=k, got=str(g)[:600], exp=str(e)[:600])
    return s.filterDecided, s.filterFallback, s.filterWindows


def cut(t, points):
    """t cut at the given columns into records."""
    edges = [0] + sorted(points) + [len(t)]
    return [t[a:b] for a, b in zip(edges, edges[1:])]


# ---------------------------------------------------------------------------------------------------------------------
# Scenarios (CPU: emulated kernels, one subprocess per set of tunables; GPU: the product library)
# ---------------------------------------------------------------------------------------------------------------------
def sc_cross(lib):
    """A query made of the last 40 symbols of record r and the first 40 of record r + 1 at k = 10: a score-0 hit on the
    plain concatenation, and none (within k) over the records.  Seed route and whole-target sweep."""
    rng = random.Random(21)
    t = genome(rng, 150_000)
    recs = cut(t, [40_000, 90_000, 120_000])
    qs = [recs[r][-40:] + recs[r + 1][:40] for r in range(3)] + reads_of(rng, t, 6, 120, 0.03)
    assert all(int(cached_row(q, t, None).min()) == 0 for q in qs[:3])
    res = {"seeds": check(lib, qs, recs, 10, both=True)}
    st, got = lib.find_record_hits(qs[:3], recs, 10)
    assert st == 0 and all(s > 0 for r in got for _, _, s in r["hits"])
    res["full"] = check(lib, qs, recs, 25)
    return res


def sc_every(lib):
    """k >= m: every column of every record is a hit, no separator column is; counts are the records' total per strand."""
    rng = random.Random(22)
    recs = [genome(rng, n) for n in (1, 7, 300, 2000, 33)]
    qs = [b"A", b"ACGTA", rand_seq(rng, 40, b"ACGT")]
    res = {}
    for k in (40, 60):
        res[k] = check(lib, qs, recs, k, both=True)
        st, got = lib.find_record_hits(qs, recs, k, True)
        assert st == 0 and all(r["count"] == 2 * sum(map(len, recs)) for r in got)
    return res


def sc_edges(lib):
    """Hits at column 0 and at the last column of each record; records of length 1 and shorter than the query; the
    same record object given twice (one pointer)."""
    rng = random.Random(23)
    big = genome(rng, 70_000)
    recs = [big, genome(rng, 5), b"G", genome(rng, 3000), big, genome(rng, 90)]
    qs = []
    for r in recs:
        qs += [r[:30], r[-30:]] if len(r) >= 30 else [r]
    qs += [rand_seq(rng, 64, b"ACGT"), b"T" * 12]
    res = {}
    for k in (0, 2, 6):
        res[k] = check(lib, qs, recs, k, both=(k == 2))
    return res


def sc_many(lib):
    """3,000 records of 20..400 bp, 23-mers at k = 3."""
    rng = random.Random(24)
    recs = [genome(rng, rng.randrange(20, 401)) for _ in range(3000)]
    qs = []
    for _ in range(6):
        r = recs[rng.randrange(len(recs))]
        a = rng.randrange(0, len(r) - 23 + 1)
        qs.append(mutate(rng, r[a:a + 23], 0.04, b"ACGT")[:23] or b"A")
    qs += [recs[5][-23:], recs[6][:23]]
    return {"k3": check(lib, qs, recs, 3, both=True)}


def sc_seed_ends(lib):
    """Queries whose alignment ends one symbol before a record's end, their front mutated so that the seeds at the end
    must find them, at k of every seed level (and above): the index keys must reach past the record end."""
    rng = random.Random(25)
    recs = [genome(rng, n) for n in (60_000, 45_000, 30_001, 50_000)]
    qs = []
    for r in recs:
        e = len(r) - 1
        for m in (150, 100):
            q = bytearray(r[e - m:e])
            for x in range(0, 40, 13):  # substitutions in the front only
                q[x] = b"ACGT"[(b"ACGT".index(q[x]) + 1) % 4]
            qs.append(bytes(q))
        qs.append(r[len(r) - 61:len(r) - 1])
    res = {}
    for k in (0, 3, 4, 6, 10, 13, 17, 21):
        res[k] = check(lib, qs, recs, k)
    return res


def sc_caps(lib):
    """Both strands; caps of 0, 1, exactly a count, one that falls mid-record; k = 0."""
    rng = random.Random(26)
    unit = genome(rng, 30)
    recs = [genome(rng, 20_000) + unit + genome(rng, 500) + unit, unit + genome(rng, 30_000), genome(rng, 9_000) + rc(unit),
            genome(rng, 25_000)]
    qs = [unit, rc(unit), unit[:20], recs[3][100:130]]
    st, full = lib.find_record_hits(qs, recs, 2, True)
    assert st == 0
    res = {"k0": check(lib, qs, recs, 0, both=True)}
    for cap in (0, 1, full[0]["count"], 2):  # unit has 2 hits in record 0 at k = 0: cap 2 stops after record 0
        res["cap%d" % cap] = check(lib, qs, recs, 2, both=True, cap=cap)
        res["cap0_%d" % cap] = check(lib, qs, recs, 0, both=True, cap=cap)
    return res


def sc_equalities(lib):
    """Transitive equalities (collapsed: seed route) and non-transitive ones with a wildcard N in the records (table path:
    whole-target sweep)."""
    rng = random.Random(27)
    t = genome(rng, 140_000)
    t = bytes(c | 0x20 if rng.random() < 0.2 else c for c in t)
    recs = cut(t, [30_000, 70_000, 110_000])
    qs = [bytes(c | 0x20 if rng.random() < 0.3 else c for c in q) for q in reads_of(rng, t.upper(), 6, 120, 0.03)]
    fold = [(bytes([c]), bytes([c | 0x20])) for c in b"ACGT"]
    wild = [(b"N", bytes([c])) for c in b"ACGT"]
    nrecs = [bytes(b"N"[0] if rng.random() < 0.01 else c for c in r.upper()) for r in recs]
    nqs = [q.upper() for q in qs[:4]] + [recs[1][-20:].upper() + b"NNNN"]
    return {"fold": check(lib, qs, recs, 6, eqs=fold), "wild": check(lib, nqs, nrecs, 4, both=True, eqs=wild)}


def sc_alignments(lib):
    """LOC / PATH: a query that begins with an insertion right at a record start takes start 0 in that record (not a
    start in the separator before it), and every start and script is that of the single-record call."""
    rng = random.Random(28)
    recs = [genome(rng, 3_000), genome(rng, 80_000), genome(rng, 700), genome(rng, 12)]
    qs = [b"T" + recs[1][:39], b"GA" + recs[2][:50], recs[0][-30:] + b"C", b"A" + recs[3]]
    qs += reads_of(rng, recs[1], 5, 100, 0.04)
    res = {}
    for k, task in ((3, 1), (3, 2), (12, 2)):
        res["%d_%d" % (k, task)] = check_aln(lib, qs, recs, k, both=(k == 12), task=task)
    st, got = lib.find_record_hits(qs[:2], recs, 3, False, 1 << 40, None, 1)
    assert st == 0
    assert (1, 38, 1) in got[0]["hits"] and got[0]["starts"][got[0]["hits"].index((1, 38, 1))] == 0
    assert (2, 49, 2) in got[1]["hits"] and got[1]["starts"][got[1]["hits"].index((2, 49, 2))] == 0
    return res


def sc_one_record(lib):
    """One record: every array and filterWindows / filterDecided / filterFallback equal edlibB200FindHitAlignments."""
    rng = random.Random(29)
    t = genome(rng, 100_000)
    qs = reads_of(rng, t, 10, 150, 0.03) + [t[:40], t[-25:]]
    out = {}
    for k, task, both in ((3, 0, True), (10, 1, False), (4, 2, True), (30, 0, False)):
        st, one = lib.find_hit_alignments(qs, t, k, both, 1 << 40, None, task)
        s1 = stats(lib)
        st2, rec = lib.find_record_hits(qs, [t], k, both, 1 << 40, None, task)
        s2 = stats(lib)
        assert st == 0 and st2 == 0
        for a, b in zip(one, rec):
            assert [h[1:] for h in b["hits"]] == [tuple(h) for h in a["hits"]] and all(h[0] == 0 for h in b["hits"])
            assert a["count"] == b["count"] and a.get("starts") == b.get("starts")
            assert a.get("alignments") == b.get("alignments")
        got = (s2.filterWindows, s2.filterDecided, s2.filterFallback)
        assert (s1.filterWindows, s1.filterDecided, s1.filterFallback) == got
        out["%d_%d" % (k, task)] = got
    return out


def sc_invalid(lib):
    """Too large a total (records sharing one anonymous read-only mapping: nothing large is allocated or read), a full
    256-code alphabet, NULL and empty records, no records, NULL out: EDLIB_STATUS_ERROR, nothing left allocated."""
    fn = lib.lib.edlibB200FindRecordHits
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int,
                   type(make_config()[0]), C.c_int, C.c_longlong, C.POINTER(RecordHits)]
    q = b"ACGTACGT"
    qp = (C.c_char_p * 1)(q)
    ql = (C.c_int * 1)(len(q))
    libc = C.CDLL(None, use_errno=True)
    libc.mmap.restype = C.c_void_p
    libc.mmap.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_long]
    libc.munmap.argtypes = [C.c_void_p, C.c_size_t]
    size = 1 << 30  # address space only: no page of it is ever touched
    addr = libc.mmap(None, size, mmap.PROT_READ, mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS, -1, 0)
    assert addr not in (None, C.c_void_p(-1).value)
    one = b"ACGTTGCA" * 4
    out = {}
    cases = [("total", [addr] * 3, [size] * 3, 3, 3),
             ("total_gaps", [addr] * 2, [(0x7ffff000 - 2) // 2] * 2, 2, 3),  # the records fit, with the separator not
             ("null", [C.cast(C.c_char_p(one), C.c_void_p).value, None], [len(one), 4], 2, 1),
             ("empty", [C.cast(C.c_char_p(one), C.c_void_p).value] * 2, [len(one), 0], 2, 1),
             ("none", [C.cast(C.c_char_p(one), C.c_void_p).value], [len(one)], 0, 1)]
    for name, ptrs, lens, n, k in cases:
        cfg, _ = make_config(k, 2, 0)
        a = RecordHits()
        st = fn(qp, ql, 1, (C.c_void_p * len(ptrs))(*ptrs), (C.c_int * len(lens))(*lens), n, cfg, 0, 10, C.byref(a))
        assert st == 1, name
        assert not a.aln.hits.counts and not a.aln.hits.offsets and not a.aln.hits.columns and not a.records, name
        out[name] = error(lib)
        assert out[name].startswith("edlibB200FindRecordHits: "), out[name]
    cfg, _ = make_config(2, 2, 0)
    assert fn(qp, ql, 1, (C.c_void_p * 1)(C.cast(C.c_char_p(one), C.c_void_p).value), (C.c_int * 1)(len(one)), 1, cfg,
              0, 10, None) == 1
    out["out"] = error(lib)
    # every byte value: no code is left for the separator of two records, but one record needs none
    allb = bytes(range(256))
    st, res = lib.find_record_hits([b"AC"], [allb, b"ACGT"], 1)
    assert st == 1 and res is None
    out["alphabet"] = error(lib)
    assert out["alphabet"].startswith("edlibB200FindRecordHits: ") and "256" in out["alphabet"]
    st, res = lib.find_record_hits([b"AB"], [allb], 0)
    assert st == 0 and res[0]["hits"] == [(0, 66, 0)]
    # ... and merged codes leave one free: upper / lower case of 26 letters folded
    fold = [(bytes([c]), bytes([c | 0x20])) for c in range(ord("A"), ord("Z") + 1)]
    st, res = lib.find_record_hits([b"ab"], [allb, b"xABx"], 0, equalities=fold)
    assert st == 0, error(lib)
    assert res[0]["hits"] == [(0, 66, 0), (0, 98, 0), (1, 2, 0)]
    st, res = lib.find_record_hits([], [one, one], 2)
    assert st == 0 and res == []
    libc.munmap(addr, size)
    return out


SCENARIOS = {"cross": sc_cross, "every": sc_every, "edges": sc_edges, "many": sc_many, "seed_ends": sc_seed_ends,
             "caps": sc_caps, "equalities": sc_equalities, "alignments": sc_alignments, "one_record": sc_one_record,
             "invalid": sc_invalid}

DRIVER = (
    "import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
    "import test_record_hits as R\n"
    "lib = R.load_emul_records()\n"
    "print(json.dumps(R.SCENARIOS[sys.argv[1]](lib)))\n"
) % (REPO, HERE)


def run_scenario(name, env=None):
    e = dict(os.environ, **(env or {}))
    out = subprocess.run([sys.executable, "-c", DRIVER, name], env=e, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_cross_record_emul():
    res = run_scenario("cross", FORCED)
    assert res["seeds"][0] > 0 and res["full"][1] > 0


def test_every_column_emul():
    run_scenario("every", FORCED)


def test_edges_short_and_repeated_records_emul():
    run_scenario("edges", FORCED)


def test_many_records_emul():
    run_scenario("many", FORCED)


def test_seeds_at_record_ends_emul():
    res = run_scenario("seed_ends", FORCED)
    assert res["0"][0] > 0 and res["10"][0] > 0 and res["17"][0] > 0  # the seed route ran at every level
    assert res["21"][0] == 0 and res["21"][1] > 0


def test_seeds_at_record_ends_one_level_emul():
    res = run_scenario("seed_ends", dict(FORCED, EDLIB_B200_FILTER_SEED_LEVELS="1"))
    assert res["3"][0] > 0


def test_caps_and_strands_emul():
    run_scenario("caps", FORCED)


def test_equalities_emul():
    res = run_scenario("equalities", FORCED)
    assert res["fold"][0] == 6 and res["wild"][0] == 0 and res["wild"][1] > 0


def test_alignments_emul():
    run_scenario("alignments", FORCED)


def test_alignments_sliced_emul():
    run_scenario("alignments", dict(FORCED, EDLIB_B200_SLICE_MB="1"))


def test_one_record_emul():
    res = run_scenario("one_record", FORCED)
    assert res["3_0"][1] > 0 and res["30_0"][2] > 0


def test_invalid_input_emul():
    res = run_scenario("invalid")
    assert "EDLIB_B200_MAX_RECORD_TARGET" in res["total"] and "EDLIB_B200_MAX_RECORD_TARGET" in res["total_gaps"]


def test_backend_without_record_kernels_refuses():
    """A backend without the record kernels (the all-hits emulation of tests/emul_hit_alignments) fails a call of
    several records loudly, with nothing allocated."""
    code = ("import sys, json, ctypes as C; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from test_hit_alignments import load_emul_hit_alignments\n"
            "from edlib_b200._ffi import RecordHits, make_config\n"
            "lib = load_emul_hit_alignments()\n"
            "fn = lib.lib.edlibB200FindRecordHits\n"
            "fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_char_p),\n"
            "               C.POINTER(C.c_int), C.c_int, type(make_config()[0]), C.c_int, C.c_longlong,\n"
            "               C.POINTER(RecordHits)]\n"
            "a = RecordHits()\n"
            "cfg, _ = make_config(1, 2, 0)\n"
            "st = fn((C.c_char_p * 1)(b'ACGTACGT'), (C.c_int * 1)(8), 1, (C.c_char_p * 2)(b'ACGT' * 50, b'TTGCA' * 30),\n"
            "        (C.c_int * 2)(200, 150), 2, cfg, 0, 10, C.byref(a))\n"
            "lib.lib.edlibB200LastError.restype = C.c_char_p\n"
            "print(json.dumps([st, bool(a.aln.hits.counts or a.aln.hits.offsets or a.aln.hits.columns or a.records),\n"
            "                  lib.lib.edlibB200LastError().decode()]))\n") % (REPO, HERE)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-3000:]
    st, allocated, msg = json.loads(out.stdout.strip().splitlines()[-1])
    assert st == 1 and not allocated and "no such kernel" in msg


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


def ecoli_records():
    """The E. coli genome cut at seeded points into 8 records, plus phage P1 as a ninth; the reference's reads of at
    most 256 bp and 200 seeded config-2 reads (150 bp, 3 % errors)."""
    from edlib_b200 import workloads
    g = workloads.ecoli_genome()
    rng = random.Random(31)
    recs = cut(g.tobytes(), rng.sample(range(1000, len(g) - 1000), 7))
    with np.load(os.path.join(HERE, "golden", "phage_1.npz")) as fx:
        recs.append(fx["target"].tobytes())
    with open(os.path.join(HERE, "golden", "ecoli_reads.json")) as f:
        fx = json.load(f)
    golden = [r["seq"].encode("ascii") for _, r in sorted(fx["reads"].items()) if 0 < len(r["seq"]) <= 256]
    seeded = [bytes(r) for r in workloads.reads_of(g, 200, seed=300)]
    return recs, golden + seeded


@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 3, 10, 20])
def test_ecoli_records_gpu(k):
    """The records call equals the single-target calls on each record, merged; k = 20 takes the whole-target route.
    Each record's least score and its columns are edlibAlign's on that record (reference build)."""
    from helpers import have_ref, ref
    recs, reads = ecoli_records()
    lib = product_lib()
    st, got = lib.find_record_hits(reads, recs, k, True, 1 << 40)
    assert st == 0, error(lib)
    s = stats(lib)
    # k = 20 is above every seed level of the 150 bp reads (the longest reference reads still reach it)
    assert s.filterFallback >= 2 * 200 if k == 20 else s.filterDecided > 0
    exp = merged_single(lib, reads, recs, k, True, 1 << 40, None, 0)
    for i, (g, e) in enumerate(zip(got, exp)):
        assert g == e, (i, g["count"], e["count"])
    if not have_ref():
        return
    r = ref()
    for i in range(0, len(reads), 5):
        for ri, t in enumerate(recs):
            e = r.align(reads[i], t, k, 2, 0)
            hits = [(c, sc) for rr, c, sc, strand in got[i]["hits"] if rr == ri and strand == 0]
            if e["editDistance"] < 0:
                assert hits == [], (i, ri)
                continue
            best = min(sc for _, sc in hits)
            assert best == e["editDistance"], (i, ri)
            assert [c for c, sc in hits if sc == best] == [c for c in e["endLocations"] if c >= 0], (i, ri)


@pytest.mark.gpu
def test_ecoli_records_paths_gpu():
    """Start locations and scripts over the E. coli records equal the single-target calls on each record."""
    recs, reads = ecoli_records()
    check_aln(product_lib(), reads[::4], recs, 3, both=True, task=2)


def seeded_batch():
    rng = random.Random(32)
    t = genome(rng, 300_000)
    recs = cut(t, rng.sample(range(100, len(t) - 100), 11)) + [genome(rng, 40), b"ACGTN"]
    qs = reads_of(rng, t, 30, 150, 0.03) + reads_of(rng, t, 10, 23, 0.0) + [rand_seq(rng, 150, b"ACGT")]
    return recs, qs


@pytest.mark.gpu
def test_emulation_matches_gpu():
    """The same seeded batch through the emulation and the H100: identical hit lists, starts and scripts."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_record_hits as R\n"
            "recs, qs = R.seeded_batch()\n"
            "lib = R.load_emul_records()\n"
            "out = [lib.find_record_hits(qs, recs, k, True, 50, None, task)[1] for k, task in ((6, 0), (4, 2))]\n"
            "print(json.dumps(out, default=lambda b: b.hex()))\n") % (REPO, HERE)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **FORCED))
    assert out.returncode == 0, out.stderr[-3000:]
    emul = json.loads(out.stdout.strip().splitlines()[-1])
    recs, qs = seeded_batch()
    lib = product_lib()
    gpu = [lib.find_record_hits(qs, recs, k, True, 50, None, task)[1] for k, task in ((6, 0), (4, 2))]
    assert json.loads(json.dumps(gpu, default=lambda b: b.hex())) == emul


@pytest.mark.gpu
def test_python_entry_gpu():
    """find_hits with a list of records equals the raw call, for str and bytes, on both strands."""
    import edlib_b200
    recs, qs = seeded_batch()
    recs = recs[:6]
    qs = qs[:12]
    lib = product_lib()
    for strands, both in (("forward", False), ("both", True)):
        st, raw = lib.find_record_hits(qs, recs, 5, both, 7)
        assert st == 0
        if both:
            raw = [{"count": r["count"], "hits": [h[:3] + ("-" if h[3] else "+",) for h in r["hits"]]} for r in raw]
        assert edlib_b200.find_hits(qs, recs, 5, strands=strands, max_hits=7) == raw
        assert edlib_b200.find_hits([q.decode() for q in qs], tuple(r.decode() for r in recs), 5, strands=strands,
                                    max_hits=7) == raw
    st, raw = lib.find_record_hits(qs, recs, 4, True, 1 << 40, None, 2)
    got = edlib_b200.find_hits(qs, recs, 4, strands="both", task="path")
    assert [r["starts"] for r in got] == [r["starts"] for r in raw]
    assert [len(r["cigars"]) for r in got] == [len(r["hits"]) for r in raw]
    # a single target behaves as before
    t = b"".join(recs)
    assert edlib_b200.find_hits(qs, t, 3) == lib.find_hits(qs, t, 3)[1]
