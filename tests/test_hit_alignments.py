"""Start locations and alignment paths of every hit (edlibB200FindHitAlignments, edlib_b200.find_hits(task=...)).

Every stored hit (c, s) of a query q (rc(q) for a strand-1 hit) of m symbols is checked against the per-hit oracle,
the checker of parity.checker() (the reference build when oracle/_ref exists, else the C restatement):
  start  = c - the last end location of align(rev(q), rev(T[max(0, c-m-s+1) .. c]), k = s, SHW, DISTANCE);
  script = align(q, T[start .. c], k = -1, NW, PATH)["alignment"], whose cost is s.
The hit lists themselves must equal edlibB200FindHits for the same arguments.  CPU tests run the engine on the emulated
kernels (tests/emul_hits) in subprocesses with forced tunables; the -m gpu tests run the product library."""
import ctypes as C
import json
import os
import random
import subprocess
import sys

import pytest

from edlib_b200._ffi import REPO, EdlibLib, HitAlignments, make_config
from helpers import mutate, rand_seq
from test_hits import FORCED, load_emul_hits, rc, reads_of, stats

HERE = os.path.dirname(os.path.abspath(__file__))
EMUL_DIR = os.path.join(HERE, "emul_hit_alignments")
LOC, PATH = 1, 2
SHW, NW, HW = 1, 0, 2


def load_emul_hit_alignments():
    """The kernel emulation of tests/emul with every kernel of the all-hits search (tests/emul_hit_alignments)."""
    subprocess.run(["make", "-s", "-C", EMUL_DIR], check=True)
    return EdlibLib(os.path.join(EMUL_DIR, "libedlib_emul_hit_alignments.so"), has_batch=True)


def per_hit(chk, q, t, c, s, eqs=None):
    """(start, script) of the hit (c, s) of q by the per-hit rule."""
    m = len(q)
    sl = t[max(0, c - m - s + 1):c + 1]
    r = chk.align(q[::-1], sl[::-1], s, SHW, 0, eqs)
    assert r["editDistance"] == s, (c, s, r["editDistance"])
    start = c - r["endLocations"][-1]
    return start, chk.align(q, t[start:c + 1], -1, NW, PATH, eqs)["alignment"]


def check(lib, qs, t, k, both=False, cap=1 << 40, eqs=None, task=PATH, sample=None):
    """One call against find_hits and the per-hit oracle (every hit, or every `sample`-th); returns the call's
    (decided, fallback, launches) and its raw result."""
    import parity
    chk = parity.checker()
    st, got = lib.find_hit_alignments(qs, t, k, both, cap, eqs, task)
    lib.lib.edlibB200LastError.restype = C.c_char_p
    assert st == 0, lib.lib.edlibB200LastError()
    s = stats(lib)
    st, plain = lib.find_hits(qs, t, k, both, cap, eqs)
    assert st == 0
    n = 0
    for i, (g, p) in enumerate(zip(got, plain)):
        assert g["count"] == p["count"] and g["hits"] == p["hits"], i
        assert len(g["starts"]) == len(g["hits"])
        if task == PATH:
            assert len(g["alignments"]) == len(g["hits"])
        for h, hit in enumerate(g["hits"]):
            n += 1
            if sample and n % sample:
                continue
            c, sc = hit[0], hit[1]
            qq = rc(qs[i]) if both and hit[2] else qs[i]
            start, script = per_hit(chk, qq, t, c, sc, eqs)
            where = dict(query=i, hit=h, c=c, s=sc, m=len(qq), k=k)
            assert g["starts"][h] == start, dict(where, got=g["starts"][h], exp=start)
            if task == PATH:
                a = g["alignments"][h]
                assert a == script, where
                assert sum(1 for op in a if op != 0) == sc, where
    return [s.filterDecided, s.filterFallback, s.launches], got


# ---------------------------------------------------------------------------------------------------------------------
# Scenarios: each returns what its test asserts on (stats per call)
# ---------------------------------------------------------------------------------------------------------------------
def sc_levels(lib):
    """150 bp reads over a 200 kbp target: the seed route at low k, the whole-target sweep above every seed level."""
    rng = random.Random(21)
    t = rand_seq(rng, 200_000, b"ACGT")
    qs = reads_of(rng, t, 10, 150, 0.04) + [rand_seq(rng, 150, b"ACGT")]
    res = {}
    for k, task, both in ((0, PATH, False), (3, LOC, True), (10, PATH, True), (30, PATH, False)):
        res[k] = check(lib, qs, t, k, both=both, task=task)[0]
    return res


def sc_short_target(lib):
    """A short target (whole-target sweep): hits with c < m, and k >= m where every column is a hit, D(c) = m too."""
    rng = random.Random(22)
    t = rand_seq(rng, 9_000, b"ACGT")
    qs = [t[:40], t[-40:], t[2030:2100], rc(t[4000:4064]), t[1000:1001], t[:33], mutate(rng, t[5000:5256], 0.05, b"ACGT")[:256]]
    res = {k: check(lib, qs, t, k, both=True)[0] for k in (0, 5)}
    small = t[:300]
    res["all"] = check(lib, [b"A", b"ACG", t[77:108], b"TTTTTTTTTT"], small, 40)[0]
    return res


def sc_boundaries(lib):
    """m of 1, 31, 32, 33, 64 and 256 (every word class border); caps of 0, 1 and exactly the count."""
    rng = random.Random(23)
    t = rand_seq(rng, 100_000, b"ACGT")
    qs = [t[5:6], t[70_000:70_031], t[100:132], t[-33:], t[:64], t[8000:8256], mutate(rng, t[3000:3256], 0.02, b"ACGT")[:256],
          t[20:52]]
    res = {"plain": check(lib, qs, t, 3, both=True)[0]}
    st, full = lib.find_hits(qs, t, 3, True)
    assert st == 0
    counts = [r["count"] for r in full]
    for cap in (0, 1, max(counts), min(c for c in counts if c > 0)):
        res["cap%d" % cap] = check(lib, qs, t, 3, both=True, cap=cap, task=LOC if cap == 1 else PATH)[0]
    return res


def sc_repeats(lib):
    """Homopolymers and tandem repeats: many tied columns, where the last column of the best score decides a start."""
    rng = random.Random(24)
    t = bytearray(rand_seq(rng, 60_000, b"ACGT"))
    t[1000:1600] = b"A" * 600
    t[10_000:11_200] = b"ACGTTG" * 200
    t[20_000:20_600] = b"AC" * 300
    t = bytes(t)
    qs = [b"A" * 64, b"A" * 40 + b"C", (b"ACGTTG" * 10)[:50], b"AC" * 30 + b"G", t[9_990:10_040]]
    return {k: check(lib, qs, t, k, both=True)[0] for k in (0, 4)}


def sc_equalities(lib):
    """Transitive equalities (collapsed codes: seed route) and non-transitive ones (equality table)."""
    rng = random.Random(25)
    t = rand_seq(rng, 120_000, b"ACGT")
    t = bytes(c | 0x20 if rng.random() < 0.2 else c for c in t)
    qs = [bytes(c | 0x20 if rng.random() < 0.3 else c for c in q) for q in reads_of(rng, t.upper(), 6, 120, 0.03)]
    fold = [(bytes([c]), bytes([c | 0x20])) for c in b"ACGT"]
    wild = [(b"N", bytes([c])) for c in b"ACGT"]
    qn = [b"".join(b"N" if rng.random() < 0.05 else bytes([c]) for c in q) for q in qs[:3]]
    return {"fold": check(lib, qs, t, 6, eqs=fold)[0], "wild": check(lib, qn + qs[:2], t, 4, eqs=wild)[0]}


def sc_slices(lib):
    """Many hits: with EDLIB_B200_SLICE_MB=1 the scripts are made in several slices; the result is the same."""
    rng = random.Random(26)
    t = rand_seq(rng, 100_000, b"ACGT")
    qs = reads_of(rng, t, 12, 150, 0.03) + reads_of(rng, t, 6, 250, 0.02)
    res, got = check(lib, qs, t, 10, both=True, sample=3)
    return {"stats": res, "got": [{"count": r["count"], "hits": r["hits"], "starts": r["starts"],
                                   "alignments": [a.hex() for a in r["alignments"]]} for r in got]}


def sc_invalid(lib):
    """Wrong mode or task, k < 0, m = 0, m > 256, NULL out: EDLIB_STATUS_ERROR, nothing left allocated; DISTANCE through
    the new entry gives the hit lists alone."""
    fn = lib.lib.edlibB200FindHitAlignments
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.c_char_p, C.c_int, type(make_config()[0]),
                   C.c_int, C.c_longlong, C.POINTER(HitAlignments)]
    lib.lib.edlibB200LastError.restype = C.c_char_p
    t = b"ACGT" * 100
    out = {}
    for name, qs, k, mode, task, null in [("mode", [b"ACGT"], 1, 0, PATH, False), ("task", [b"ACGT"], 1, HW, 3, False),
                                          ("k", [b"ACGT"], -1, HW, LOC, False), ("empty", [b""], 1, HW, PATH, False),
                                          ("long", [b"A" * 257], 1, HW, LOC, False), ("null", [b"ACGT"], 1, HW, PATH, True)]:
        cfg, _ = make_config(k, mode, task)
        a = HitAlignments()
        a.hits.numQueries = 99
        qp = (C.c_char_p * 1)(*qs)
        ql = (C.c_int * 1)(*[len(q) for q in qs])
        st = fn(qp, ql, 1, t, len(t), cfg, 0, 10, None if null else C.byref(a))
        assert st == 1, name
        h = a.hits
        assert not (h.counts or h.offsets or h.columns or h.scores or h.strands), name
        assert not (a.starts or a.alignmentOffsets or a.alignments), name
        out[name] = lib.lib.edlibB200LastError().decode()
        assert out[name].startswith("edlibB200FindHitAlignments:"), out[name]
    for task in (0, LOC, PATH):
        st, res = lib.find_hit_alignments([], t, 2, task=task)
        assert st == 0 and res == []
    st, res = lib.find_hit_alignments([b"ACGTA", b"GGGG"], t, 1, task=0)
    assert st == 0 and all("starts" not in r and "alignments" not in r for r in res)
    assert res == lib.find_hits([b"ACGTA", b"GGGG"], t, 1)[1]
    st, res = lib.find_hit_alignments([b"GGGGGGGG"], t, 1, task=PATH)  # no hits at all
    assert st == 0 and res == [{"count": 0, "hits": [], "starts": [], "alignments": []}]
    return out


SCENARIOS = {"levels": sc_levels, "short_target": sc_short_target, "boundaries": sc_boundaries, "repeats": sc_repeats,
             "equalities": sc_equalities, "slices": sc_slices, "invalid": sc_invalid}

DRIVER = (
    "import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
    "import test_hit_alignments as A\n"
    "lib = A.load_emul_hit_alignments()\n"
    "print(json.dumps(A.SCENARIOS[sys.argv[1]](lib)))\n"
) % (REPO, HERE)


def run_scenario(name, env=None):
    e = dict(os.environ, **(env or {}))
    out = subprocess.run([sys.executable, "-c", DRIVER, name], env=e, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


# ---------------------------------------------------------------------------------------------------------------------
# CPU: emulated kernels under the real engine
# ---------------------------------------------------------------------------------------------------------------------
def test_seed_route_and_whole_target_emul():
    res = run_scenario("levels", FORCED)
    # [decided, fallback, launches]: low k from the seed windows, k = 30 above every seed level swept in full
    assert res["0"][0] > 0 and res["10"][0] > 0
    assert res["30"][:2] == [0, 11]


def test_short_target_emul():
    res = run_scenario("short_target", {"EDLIB_B200_K1_MIN_CHUNK": "256"})
    assert all(v[0] == 0 and v[1] > 0 for v in res.values())


def test_boundaries_and_caps_emul():
    run_scenario("boundaries", FORCED)


def test_repeats_emul():
    run_scenario("repeats", FORCED)


def test_equalities_emul():
    res = run_scenario("equalities", FORCED)
    assert res["fold"][0] == 6 and res["wild"][:2] == [0, 5]


def test_slices_emul():
    """One slice under the default budget, several under 1 MiB: more launches, the same starts and scripts."""
    one = run_scenario("slices", FORCED)
    many = run_scenario("slices", dict(FORCED, EDLIB_B200_SLICE_MB="1"))
    assert many["got"] == one["got"]
    assert many["stats"][2] > one["stats"][2] + 20


def test_invalid_input_emul():
    assert len(run_scenario("invalid")) == 6


def test_backend_without_hit_kernels_refuses():
    """The plain kernel emulation lacks the hit kernels: the new entry fails loudly, with nothing allocated."""
    from test_engine_emul import load_emul
    lib = load_emul()
    for task in (0, LOC, PATH):
        st, res = lib.find_hit_alignments([b"ACGTACGT"], b"ACGT" * 100, 1, task=task)
        lib.lib.edlibB200LastError.restype = C.c_char_p
        assert st == 1 and res is None
        assert b"no such kernel" in lib.lib.edlibB200LastError()


def test_backend_without_hit_res_kernel_refuses_loc_and_path():
    """A backend with the hit-list kernels but without hit_res_kernel (tests/emul_hits) gives the hit lists for task
    DISTANCE and refuses LOC / PATH loudly, with nothing allocated."""
    lib = load_emul_hits()
    lib.lib.edlibB200LastError.restype = C.c_char_p
    q, t = [b"ACGTACGT"], b"ACGT" * 100
    st, res = lib.find_hit_alignments(q, t, 1, task=0)
    assert st == 0 and res == lib.find_hits(q, t, 1)[1]
    for task in (LOC, PATH):
        st, res = lib.find_hit_alignments(q, t, 1, task=task)
        assert st == 1 and res is None
        assert b"hit_res: no such kernel" in lib.lib.edlibB200LastError()


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
def test_slices_gpu():
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_hit_alignments as A\n"
            "from helpers import product\n"
            "print(json.dumps(A.sc_slices(product())))\n") % (REPO, HERE)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                         env=dict(os.environ, EDLIB_B200_SLICE_MB="1"))
    assert out.returncode == 0, out.stderr[-3000:]
    many = json.loads(out.stdout.strip().splitlines()[-1])
    one = json.loads(json.dumps(sc_slices(product_lib())))  # hits as lists, as they come back from the subprocess
    assert many["got"] == one["got"] and many["stats"][2] > one["stats"][2] + 20


@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 3, 10])
def test_ecoli_against_reference_gpu(k):
    """E. coli reads over the 4.63 Mbp genome: the starts of the least-score columns are edlibAlign's HW LOC
    startLocations, the script of the first is its HW PATH alignment, and a sample of the other hits follows the
    per-hit rule."""
    from helpers import have_ref, ref
    from test_hits import ecoli_case
    if not have_ref():
        pytest.skip("reference build not available")
    genome, reads = ecoli_case(k)
    lib = product_lib()
    st, got = lib.find_hit_alignments(reads, genome, k, False, 1 << 40, None, PATH)
    assert st == 0
    st, plain = lib.find_hits(reads, genome, k, False, 1 << 40)
    assert st == 0 and [(g["count"], g["hits"]) for g in got] == [(p["count"], p["hits"]) for p in plain]
    r = ref()
    rng = random.Random(k)
    for i, q in enumerate(reads):
        hits = got[i]["hits"]
        if not hits:
            continue
        best = min(s for _, s in hits)
        idx = [h for h, (_, s) in enumerate(hits) if s == best]
        loc = r.align(q, genome, k, HW, LOC)
        assert loc["editDistance"] == best, i
        assert [got[i]["starts"][h] for h in idx] == loc["startLocations"], i
        assert [hits[h][0] for h in idx] == loc["endLocations"], i
        assert got[i]["alignments"][idx[0]] == r.align(q, genome, k, HW, PATH)["alignment"], i
        for h in rng.sample(range(len(hits)), min(2, len(hits))):
            c, s = hits[h]
            start, script = per_hit(r, q, genome, c, s)
            assert (got[i]["starts"][h], got[i]["alignments"][h]) == (start, script), (i, h)


@pytest.mark.gpu
def test_emulation_matches_gpu():
    """One seeded batch, both strands, task PATH, through the emulation and the H100: identical output."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_hit_alignments as A\n"
            "t, qs = A.seeded_batch()\n"
            "st, res = A.load_emul_hit_alignments().find_hit_alignments(qs, t, 6, True, 50, None, 2)\n"
            "print(json.dumps(A.plain(res)))\n") % (REPO, HERE)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **FORCED))
    assert out.returncode == 0, out.stderr[-3000:]
    emul = json.loads(out.stdout.strip().splitlines()[-1])
    t, qs = seeded_batch()
    st, res = product_lib().find_hit_alignments(qs, t, 6, True, 50, None, PATH)
    assert st == 0
    assert plain(res) == emul


def seeded_batch():
    rng = random.Random(27)
    t = rand_seq(rng, 300_000, b"ACGT")
    return t, reads_of(rng, t, 40, 150, 0.03) + reads_of(rng, t, 10, 23, 0.0) + [rand_seq(rng, 150, b"ACGT")]


def plain(res):
    return [{"count": r["count"], "hits": [list(h) for h in r["hits"]], "starts": r["starts"],
             "alignments": [a.hex() for a in r["alignments"]]} for r in res]


@pytest.mark.gpu
def test_python_entry_gpu():
    import edlib_b200
    rng = random.Random(28)
    t = rand_seq(rng, 80_000, b"ACGT")
    qs = reads_of(rng, t, 6, 100, 0.03)
    lib = product_lib()
    for strands, both in (("forward", False), ("both", True)):
        base = edlib_b200.find_hits(qs, t, 5, strands=strands, max_hits=7)
        loc = edlib_b200.find_hits(qs, t, 5, strands=strands, max_hits=7, task="locations")
        path = edlib_b200.find_hits(qs, t, 5, strands=strands, max_hits=7, task="path")
        st, raw = lib.find_hit_alignments(qs, t, 5, both, 7, None, PATH)
        assert st == 0
        for b, lo, pa, r in zip(base, loc, path, raw):
            assert set(b) == {"count", "hits"} and set(lo) == {"count", "hits", "starts"}
            assert lo["hits"] == b["hits"] == pa["hits"] and lo["starts"] == pa["starts"] == r["starts"]
            assert pa["cigars"] == [lib.cigar(a) for a in r["alignments"]]
    # the least-score hit of a forward query: the same locations and CIGAR as align(..., "HW", "path")
    q = t[5000:5100]
    one = edlib_b200.find_hits([q], t, 5, task="path")[0]
    best = min(s for _, s in one["hits"])
    h = [i for i, (_, s) in enumerate(one["hits"]) if s == best]
    a = edlib_b200.align(q, t, mode="HW", task="path", k=5)
    assert a["locations"] == [(one["starts"][i], one["hits"][i][0]) for i in h]
    assert a["cigar"] == one["cigars"][h[0]]
    with pytest.raises(ValueError):
        edlib_b200.find_hits(qs, t, 3, task="cigar")
