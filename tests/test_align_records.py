"""Best-record alignment over a multi-record reference (edlibB200AlignRecords, edlib_b200.align_records).

The rule: for query q, A(r) = edlibAlign(q, records[r], HW); the best record r* is the lowest index among those of
least distance, "none within k" counting as larger than any distance (so r* = 0 when no record has an alignment, and
for an empty query).  The result is A(r*) in every field, the record r*; with both strands, the strand rule of
edlibB200AlignBatchStrands picks between the best records of q and rc(q).  Every case compares every field, the
record and the strand with that rule applied to per-record edlibAlign answers of the checker (the reference build
when oracle/_ref is present, else the oracle restatement).  CPU tests run the engine on the emulated kernels
(tests/emul_records) in subprocesses with forced tunables; `filterDecided` / `filterFallback` show which route ran.
The -m gpu tests run the product library."""
import ctypes as C
import json
import mmap
import os
import random
import subprocess
import sys

import pytest

import parity
from edlib_b200._ffi import REPO, AlignResult, make_config
from helpers import mutate, rand_seq
from test_hits import FORCED, genome, rc, reads_of, stats
from test_record_hits import cut, error, load_emul_records

HERE = os.path.dirname(os.path.abspath(__file__))


def best_of(chk, q, recs, k, task, eqs):
    """(A(r*), r*) by the rule, from one checker call per record."""
    per = [chk.align(q, t, k, 2, task, eqs) for t in recs]
    found = [r for r, a in enumerate(per) if a["editDistance"] >= 0]
    r = min(found, key=lambda x: (per[x]["editDistance"], x)) if found else 0
    return per[r], r


def expected(chk, q, recs, k, task, eqs, both):
    f, rf = best_of(chk, q, recs, k, task, eqs)
    if not both:
        return f, rf, None
    b, rb = best_of(chk, rc(q), recs, k, task, eqs)
    if b["editDistance"] >= 0 and (f["editDistance"] < 0 or b["editDistance"] < f["editDistance"]):
        return b, rb, 1
    return f, rf, 0


def check(lib, qs, recs, k, task=0, both=False, eqs=None):
    """One records call against the rule; returns (decided, fallback, windows) and the records chosen."""
    st, res, rs, ss = lib.align_records(qs, recs, k, task, eqs, both)
    assert st == 0, error(lib)
    s = stats(lib)
    chk = parity.checker()
    for i, q in enumerate(qs):
        exp, r, strand = expected(chk, q, recs, k, task, eqs, both)
        got = (res[i], rs[i], ss[i] if both else None)
        assert got == (exp, r, strand), dict(query=i, k=k, task=task, m=len(q), both=both, got=str(got)[:500],
                                             exp=str((exp, r, strand))[:500])
    return [s.filterDecided, s.filterFallback, s.filterWindows], rs


# ---------------------------------------------------------------------------------------------------------------------
# Scenarios (CPU: emulated kernels, one subprocess per set of tunables; GPU: the product library)
# ---------------------------------------------------------------------------------------------------------------------
def sc_reads(lib):
    """Reads of 100..150 bp drawn from every record with 0..10 edits (and a few unrelated ones), at k = -1, 0, 10 and k
    at and above each seed level's threshold, tasks DISTANCE / LOC / PATH."""
    rng = random.Random(41)
    recs = cut(genome(rng, 180_000), [50_000, 110_000, 150_000]) + [genome(rng, 2_000), genome(rng, 70_000)]
    qs = []
    for r in recs:
        for e in (0, 2, 5, 10):
            m = rng.choice((100, 150))
            a = rng.randrange(0, len(r) - m)
            q = bytearray(r[a:a + m])
            for x in rng.sample(range(m), e):
                q[x] = b"ACGT"[(b"ACGT".index(q[x]) + 1 + rng.randrange(3)) % 4]
            qs.append(bytes(q))
    qs += [rand_seq(rng, 120, b"ACGT") for _ in range(2)]
    res = {}
    for k, task in ((-1, 0), (0, 1), (10, 2), (3, 0), (6, 1), (13, 0), (21, 2), (-1, 2)):
        res["%d_%d" % (k, task)], rs = check(lib, qs, recs, k, task)
        assert set(rs[:4 * len(recs)]) == set(range(len(recs)))
    return res


def sc_ties(lib):
    """The same record twice and a repeat shared by two records (the lower index wins, only its end columns are
    reported); a record ending in the query minus its last symbol (the first separator column ties the best score);
    one inserted symbol before an exact match at the first column of record r > 0 (start 0 of that record); reads
    across a cut between two records."""
    rng = random.Random(42)
    rep = genome(rng, 60)
    a = genome(rng, 30_000)
    q_end = genome(rng, 80)
    recs = [genome(rng, 20_000) + rep + genome(rng, 3_000), a, genome(rng, 9_000) + q_end[:-1], genome(rng, 25_000) + rep,
            a, genome(rng, 700)]
    qs = [rep, a[5_000:5_120], q_end, b"T" + recs[5][:60], b"G" + recs[1][:45], recs[0][-50:] + recs[1][:50],
          recs[2][-40:] + recs[3][:40], recs[3][-30:]]
    res = {}
    for k, task in ((-1, 2), (0, 1), (4, 2), (12, 0)):
        res["%d_%d" % (k, task)], rs = check(lib, qs, recs, k, task)
    st, out, rs, _ = lib.align_records(qs, recs, 4, 2)
    assert st == 0
    assert rs[0] == 0 and out[0]["endLocations"] == [20_059]
    assert rs[1] == 1 and out[1]["endLocations"] == [5_119]
    assert rs[2] == 2 and out[2]["editDistance"] == 1 and out[2]["endLocations"] == [len(recs[2]) - 1]
    assert rs[3] == 5 and out[3]["startLocations"] == [0] and out[3]["editDistance"] == 1
    return res


def sc_none(lib):
    """No record within k: record 0 and record 0's alphabetLength.  Records of different alphabets (N, lower case):
    alphabetLength is that of the query and its own record."""
    rng = random.Random(43)
    recs = [genome(rng, 5_000), genome(rng, 4_000).lower(), genome(rng, 3_000).replace(b"A", b"N"), b"XYZ" * 40]
    qs = [rand_seq(rng, 60, b"ACGT"), recs[1][100:160], recs[2][200:260], recs[3][:30], recs[0][10:70], b"acgtN" * 5]
    res = {}
    for k, task in ((0, 0), (3, 1), (-1, 2), (30, 0)):
        res["%d_%d" % (k, task)], rs = check(lib, qs, recs, k, task)
    st, out, rs, _ = lib.align_records(qs, recs, 0)
    assert st == 0 and rs[0] == 0 and out[0]["editDistance"] == -1
    assert [o["alphabetLength"] for o in out[1:4]] == [4, 4, 3] and rs[1:4] == [1, 2, 3]
    return res


def sc_small(lib):
    """An empty query, records of length 1, records shorter than the query, 3,000 short records."""
    rng = random.Random(44)
    recs = [b"G", genome(rng, 5), genome(rng, 300), b"A", genome(rng, 40)]
    qs = [b"", b"A", b"G", recs[2][:100], recs[1] + b"T", rand_seq(rng, 64, b"ACGT"), recs[4]]
    res = {}
    for k, task in ((-1, 2), (0, 1), (2, 0), (70, 2)):
        res["%d_%d" % (k, task)], rs = check(lib, qs, recs, k, task)
        assert rs[0] == 0
    many = [genome(rng, rng.randrange(20, 401)) for _ in range(3000)]
    mq = []
    for _ in range(6):
        r = many[rng.randrange(len(many))]
        a = rng.randrange(0, len(r) - 23 + 1)
        mq.append(mutate(rng, r[a:a + 23], 0.04, b"ACGT")[:23] or b"A")
    mq += [many[2999][-23:], many[1500][:23]]
    res["many"], rs = check(lib, mq, many, 3, 2)
    assert rs[-2:] == [2999, 1500]
    return res


def sc_strands(lib):
    """Both strands: each strand its own best record, the reverse one only when strictly better; a read whose two
    strands tie takes the forward one."""
    rng = random.Random(45)
    recs = cut(genome(rng, 120_000), [40_000, 85_000]) + [genome(rng, 900)]
    qs = reads_of(rng, recs[1], 4, 120, 0.03) + [rc(x) for x in reads_of(rng, recs[2], 4, 120, 0.03)]
    pal = genome(rng, 30)
    tie = pal + rc(pal)  # its own reverse complement: both strands align equally well
    recs[3] = recs[3][:300] + tie + recs[3][300:]
    qs += [tie, rc(recs[0][1000:1100]), recs[3][:50]]
    res = {}
    for k, task in ((-1, 0), (6, 2), (0, 1)):
        res["%d_%d" % (k, task)], rs = check(lib, qs, recs, k, task, both=True)
    st, out, rs, ss = lib.align_records(qs, recs, 0, 0, None, True)
    assert st == 0 and ss[8] == 0 and rs[8] == 3 and ss[9] == 1 and rs[9] == 0
    return res


def sc_equalities(lib):
    """Transitive equalities (collapsed to one code: the seed route) and non-transitive ones with a wildcard N in the
    records (equality table: the prefix-stage route)."""
    rng = random.Random(46)
    t = genome(rng, 140_000)
    t = bytes(c | 0x20 if rng.random() < 0.2 else c for c in t)
    recs = cut(t, [30_000, 70_000, 110_000])
    qs = [bytes(c | 0x20 if rng.random() < 0.3 else c for c in q) for q in reads_of(rng, t.upper(), 6, 120, 0.03)]
    fold = [(bytes([c]), bytes([c | 0x20])) for c in b"ACGT"]
    wild = [(b"N", bytes([c])) for c in b"ACGT"]
    nrecs = [bytes(b"N"[0] if rng.random() < 0.01 else c for c in r.upper()) for r in recs]
    nqs = [q.upper() for q in qs[:4]] + [recs[1][-20:].upper() + b"NNNN"]
    return {"fold": check(lib, qs, recs, 6, 2, eqs=fold)[0], "wild": check(lib, nqs, nrecs, 4, 1, both=True, eqs=wild)[0],
            "wild_all": check(lib, nqs, nrecs, -1, 0, eqs=wild)[0]}


def sc_long(lib):
    """Queries of 300, 1,100 and 3,000 symbols (the long HW route, start locations of the warp runner); the 3,000
    symbol path takes the Hirschberg route."""
    rng = random.Random(47)
    recs = cut(genome(rng, 150_000), [60_000, 100_000]) + [genome(rng, 5_000)]
    qs = [mutate(rng, recs[1][2_000:2_300], 0.02, b"ACGT"), mutate(rng, recs[2][10_000:11_100], 0.02, b"ACGT"),
          mutate(rng, recs[0][30_000:33_000], 0.01, b"ACGT"), mutate(rng, recs[3][1_000:4_000], 0.02, b"ACGT"),
          recs[0][-500:] + recs[1][:600]]
    res = {}
    for k, task in ((-1, 2), (40, 1), (100, 0)):
        res["%d_%d" % (k, task)], rs = check(lib, qs, recs, k, task)
    return res


def sc_one_record(lib):
    """One record: every field equals edlibAlignBatch against it, every record index is 0."""
    rng = random.Random(48)
    t = genome(rng, 100_000)
    qs = reads_of(rng, t, 10, 150, 0.03) + [t[:40], t[-25:], b"", rand_seq(rng, 90, b"ACGT"),
                                             mutate(rng, t[500:1_000], 0.02, b"ACGT")]
    out = {}
    for k, task in ((-1, 2), (3, 0), (10, 1), (30, 2)):
        st, exp = lib.align_batch(qs, [t] * len(qs), k, 2, task)
        st2, got, rs, _ = lib.align_records(qs, [t], k, task)
        assert st == 0 and st2 == 0
        assert got == exp and rs == [0] * len(qs)
        out["%d_%d" % (k, task)] = True
    return out


def sc_python(lib):
    """edlib_b200.align_records equals align_batch run per record and merged by the rule, for str and bytes and both
    strands."""
    import edlib_b200
    edlib_b200._lib = lib  # the package entry over this library
    lib.lib.edlibB200LastError.restype = C.c_char_p
    rng = random.Random(49)
    recs = cut(genome(rng, 90_000), [30_000, 60_000]) + [genome(rng, 400)]
    qs = reads_of(rng, recs[1], 3, 100, 0.03) + [rc(x) for x in reads_of(rng, recs[2], 3, 100, 0.03)] + [recs[3][:50]]
    for task in ("distance", "locations", "path"):
        for strands in ("forward", "both"):
            per = [edlib_b200.align_batch(qs, t, mode="HW", task=task, k=8, strands=strands) for t in recs]
            exp = []
            for i in range(len(qs)):
                cand = [(per[r][i]["editDistance"], r) for r in range(len(recs)) if per[r][i]["editDistance"] >= 0]
                r = min(cand)[1] if cand else 0
                exp.append(dict(per[r][i], record=r))
            got = edlib_b200.align_records(qs, recs, task=task, k=8, strands=strands)
            got_s = edlib_b200.align_records([q.decode() for q in qs], tuple(r.decode() for r in recs), task=task, k=8,
                                             strands=strands)
            assert got == got_s
            if strands == "forward":
                assert got == exp, task
            else:
                st, raw, rs, ss = lib.align_records(qs, recs, 8, {"distance": 0, "locations": 1, "path": 2}[task], None, True)
                assert [g["record"] for g in got] == rs and [g["strand"] for g in got] == ["-" if s else "+" for s in ss]
                assert [g["editDistance"] for g in got] == [d["editDistance"] for d in raw]
    with pytest.raises(ValueError):
        edlib_b200.align_records(qs, recs, strands="sideways")
    with pytest.raises(Exception):
        edlib_b200.align_records(qs, [])
    return {"ok": True}


def sc_invalid(lib):
    """Invalid input: EDLIB_STATUS_ERROR, a message starting "edlibB200AlignRecords:", error results with no arrays;
    an oversized total is refused before any record byte is read (records sharing one anonymous read-only mapping)."""
    fn = lib.lib.edlibB200AlignRecords
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int,
                   type(make_config()[0]), C.c_int, C.POINTER(AlignResult), C.POINTER(C.c_int), C.POINTER(C.c_ubyte)]
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
    one = C.cast(C.c_char_p(b"ACGTTGCA" * 4), C.c_void_p).value
    out = {}
    rec = (C.c_int * 1)()
    strand = (C.c_ubyte * 1)()
    cases = [("total", [addr] * 3, [size] * 3, 3, 2, 0, 0, True, True),
             ("total_k", [addr] * 2, [(0x7ffff000 - 8) // 2] * 2, 2, -1, 0, 0, True, True),  # gap = longest + 1 = 9
             ("null", [one, None], [32, 4], 2, 1, 0, 0, True, True),
             ("empty", [one] * 2, [32, 0], 2, 1, 0, 0, True, True),
             ("none", [one], [32], 0, 1, 0, 0, True, True),
             ("mode_nw", [one], [32], 1, 1, 0, 0, True, True),
             ("mode_shw", [one], [32], 1, 1, 1, 0, True, True),
             ("records_out", [one], [32], 1, 1, 2, 0, False, True),
             ("strands_out", [one], [32], 1, 1, 2, 1, True, False)]
    for name, ptrs, lens, n, k, mode, both, with_rec, with_strand in cases:
        cfg, _ = make_config(k, {0: 2, 1: 1, 2: 2}[mode] if name != "mode_nw" else 0, 0)
        res = (AlignResult * 1)()
        res[0].editDistance = 77
        st = fn(qp, ql, 1, (C.c_void_p * len(ptrs))(*ptrs), (C.c_int * len(lens))(*lens), n, cfg, both, res,
                rec if with_rec else None, strand if with_strand else None)
        assert st == 1, name
        assert not res[0].endLocations and not res[0].startLocations and not res[0].alignment, name
        assert res[0].status == 1 and res[0].editDistance == -1, name
        out[name] = error(lib)
        assert out[name].startswith("edlibB200AlignRecords: "), out[name]
    libc.munmap(addr, size)
    # every byte value: no code is left for the separator of two records, but one record needs none
    allb = bytes(range(256))
    st, res, rs, _ = lib.align_records([b"AC"], [allb, b"ACGT"], 1)
    assert st == 1 and res is None
    out["alphabet"] = error(lib)
    assert out["alphabet"].startswith("edlibB200AlignRecords: ") and "256" in out["alphabet"]
    st, res, rs, _ = lib.align_records([b"AB"], [allb], 0, 1)
    assert st == 0 and rs == [0] and res[0]["endLocations"] == [66] and res[0]["alphabetLength"] == 256
    # ... and merged codes leave one free: upper / lower case of 26 letters folded
    fold = [(bytes([c]), bytes([c | 0x20])) for c in range(ord("A"), ord("Z") + 1)]
    st, res, rs, _ = lib.align_records([b"xy"], [allb, b"aXYb"], 0, 1, fold)
    assert st == 0, error(lib)
    assert rs == [0] and res[0]["endLocations"] == [89, 121]
    st, res, rs, _ = lib.align_records([], [b"ACGT", b"GG"], 2)
    assert st == 0 and res == []
    return out


SCENARIOS = {"reads": sc_reads, "ties": sc_ties, "none": sc_none, "small": sc_small, "strands": sc_strands,
             "equalities": sc_equalities, "long": sc_long, "one_record": sc_one_record, "python": sc_python,
             "invalid": sc_invalid}

DRIVER = (
    "import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
    "import test_align_records as R\n"
    "lib = R.load_emul_records()\n"
    "print(json.dumps(R.SCENARIOS[sys.argv[1]](lib)))\n"
) % (REPO, HERE)

# every filter stage and the device-driven first level off: the plain sweeps decide every read
NO_FILTERS = {"EDLIB_B200_FILTER_SEED_K": "0", "EDLIB_B200_FILTER_K0": "0", "EDLIB_B200_FILTER_K1": "0",
              "EDLIB_B200_DEVICE_STAGE": "0"}


def run_scenario(name, env=None):
    e = dict(os.environ, **(env or {}))
    out = subprocess.run([sys.executable, "-c", DRIVER, name], env=e, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_reads_from_every_record_emul():
    res = run_scenario("reads", FORCED)
    assert res["0_1"][0] > 0 and res["3_0"][0] > 0 and res["13_0"][0] > 0  # the seed filter decided reads
    assert res["21_2"][1] > 0 or res["-1_0"][1] > 0


def test_reads_without_filters_emul():
    """Every filter stage and the device stage switched off: the same results by the plain sweeps."""
    res = run_scenario("reads", NO_FILTERS)
    assert all(v[0] == 0 and v[2] == 0 for v in res.values())


def test_ties_and_record_edges_emul():
    run_scenario("ties", FORCED)


def test_ties_and_record_edges_without_filters_emul():
    run_scenario("ties", NO_FILTERS)


def test_no_alignment_and_alphabets_emul():
    run_scenario("none", FORCED)


def test_short_and_many_records_emul():
    run_scenario("small", FORCED)


def test_both_strands_emul():
    run_scenario("strands", FORCED)


def test_equalities_emul():
    res = run_scenario("equalities", FORCED)
    # collapsed codes: the seed levels; a table of equalities: no seed index, the prefix stages decide
    assert res["fold"][0] > 0 and res["wild"][0] > 0


def test_long_queries_emul():
    run_scenario("long", FORCED)


def test_one_record_equals_align_batch_emul():
    run_scenario("one_record", FORCED)


def test_python_entry_emul():
    run_scenario("python", FORCED)


def test_invalid_input_emul():
    res = run_scenario("invalid")
    assert "EDLIB_B200_MAX_RECORD_TARGET" in res["total"] and "EDLIB_B200_MAX_RECORD_TARGET" in res["total_k"]
    assert "EDLIB_MODE_HW" in res["mode_nw"] and "EDLIB_MODE_HW" in res["mode_shw"]


def test_backend_without_record_kernels_refuses():
    """A backend without the record kernels (the all-hits emulation of tests/emul_hit_alignments) fails a call of
    several records loudly, with error results and no arrays."""
    code = ("import sys, json, ctypes as C; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from test_hit_alignments import load_emul_hit_alignments\n"
            "lib = load_emul_hit_alignments()\n"
            "st, res, rs, ss = lib.align_records([b'ACGTACGT', b'TTGCA'], [b'ACGT' * 50, b'TTGCA' * 30], 1)\n"
            "lib.lib.edlibB200LastError.restype = C.c_char_p\n"
            "one = lib.align_records([b'ACGTACGT'], [b'ACGT' * 50], 1)\n"
            "print(json.dumps([st, res, lib.lib.edlibB200LastError().decode(), one[0], one[2]]))\n") % (REPO, HERE)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-3000:]
    st, res, msg, st1, rs1 = json.loads(out.stdout.strip().splitlines()[-1])
    assert st == 1 and res is None and "no such kernel" in msg
    assert st1 == 0 and rs1 == [0]  # one record needs no record kernel


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


def ecoli_records(count):
    """The E. coli genome cut at seeded points into 8 records, plus phage P1 as a ninth; `count` config-2 reads of
    150 bp (3 % errors) from the genome, a tenth of them across a cut, and 50 reads from the phage."""
    import numpy as np
    from edlib_b200 import workloads
    g = workloads.ecoli_genome()
    rng = random.Random(51)
    cuts = sorted(rng.sample(range(1000, len(g) - 1000), 7))
    gb = g.tobytes()
    recs = cut(gb, cuts)
    with np.load(os.path.join(HERE, "golden", "phage_1.npz")) as fx:
        phage = fx["target"].tobytes()
    recs.append(phage)
    reads = [bytes(r) for r in workloads.reads_of(g, count - count // 10, seed=301)]
    for x in range(count // 10):
        c = cuts[x % 7] - rng.randrange(20, 130)
        reads.append(mutate(rng, gb[c:c + 150], 0.03, b"ACGT")[:256])
    reads += reads_of(rng, phage, 50, 150, 0.03)
    return recs, reads


def merged_batches(lib, reads, recs, k, task, both):
    """Per-record edlibAlignBatch (or edlibB200AlignBatchStrands per strand) calls merged by the rule."""
    def best(qs):
        per = []
        for t in recs:
            st, res = lib.align_batch(qs, [t] * len(qs), k, 2, task)
            assert st == 0
            per.append(res)
        out = []
        for i in range(len(qs)):
            found = [r for r in range(len(recs)) if per[r][i]["editDistance"] >= 0]
            r = min(found, key=lambda x: (per[x][i]["editDistance"], x)) if found else 0
            out.append((per[r][i], r))
        return out
    f = best(reads)
    if not both:
        return [(a, r, None) for a, r in f]
    b = best([rc(q) for q in reads])
    out = []
    for (fa, fr), (ba, br) in zip(f, b):
        rev = ba["editDistance"] >= 0 and (fa["editDistance"] < 0 or ba["editDistance"] < fa["editDistance"])
        out.append((ba, br, 1) if rev else (fa, fr, 0))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("k", [-1, 10])
@pytest.mark.parametrize("task", [0, 1, 2])
@pytest.mark.parametrize("both", [False, True])
def test_ecoli_records_gpu(k, task, both):
    """About 20,000 reads over the E. coli records plus phage P1 equal the per-record batch calls merged by the rule;
    a sample equals the reference's edlibAlign per record."""
    from helpers import have_ref, ref
    recs, reads = ecoli_records(20_000)
    lib = product_lib()
    st, res, rs, ss = lib.align_records(reads, recs, k, task, None, both)
    assert st == 0, error(lib)
    exp = merged_batches(lib, reads, recs, k, task, both)
    for i, (e, r, s) in enumerate(exp):
        assert (res[i], rs[i], ss[i] if both else None) == (e, r, s), (i, str(res[i])[:300], rs[i], str(e)[:300], r)
    if both:  # the phage reads (of either strand) found their record
        assert sum(1 for r in rs[-50:] if r == 8) >= 45
    if not have_ref():
        return
    chk = ref()
    for i in range(0, len(reads), 397):
        assert (res[i], rs[i], ss[i] if both else None) == expected(chk, reads[i], recs, k, task, None, both), i


def seeded_batch():
    rng = random.Random(52)
    t = genome(rng, 300_000)
    recs = cut(t, rng.sample(range(100, len(t) - 100), 11)) + [genome(rng, 40), b"ACGTN"]
    qs = reads_of(rng, t, 30, 150, 0.03) + reads_of(rng, t, 10, 23, 0.0) + [rand_seq(rng, 150, b"ACGT"), b"",
                                                                            mutate(rng, t[1000:1400], 0.02, b"ACGT")]
    return recs, qs


@pytest.mark.gpu
def test_emulation_matches_gpu():
    """The same seeded batch through the emulation and the H100: identical results, records and strands."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_align_records as R\n"
            "recs, qs = R.seeded_batch()\n"
            "lib = R.load_emul_records()\n"
            "out = [lib.align_records(qs, recs, k, task, None, both) for k, task, both in ((6, 0, True), (-1, 2, False))]\n"
            "print(json.dumps(out, default=lambda b: b.hex()))\n") % (REPO, HERE)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **FORCED))
    assert out.returncode == 0, out.stderr[-3000:]
    emul = json.loads(out.stdout.strip().splitlines()[-1])
    recs, qs = seeded_batch()
    lib = product_lib()
    gpu = [lib.align_records(qs, recs, k, task, None, both) for k, task, both in ((6, 0, True), (-1, 2, False))]
    assert json.loads(json.dumps(gpu, default=lambda b: b.hex())) == emul
