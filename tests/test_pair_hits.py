"""All-hits search over query-target pairs (edlibB200FindPairHits, edlib_b200.find_pair_hits).

Pair i searches query i in its own target i only.  Every case compares the hit lists with the brute-force HW last row of
test_hits.last_row per pair, exactly; with task LOC / PATH every entry is also compared with a single-target
edlibB200FindHitAlignments call of the pair's query over its target on the same library, and every script's cost must
be its hit's score.  CPU tests run the engine on the emulated kernels (tests/emul_pair_hits) in subprocesses with
forced tunables; `filterDecided` / `filterFallback` show which route ran.  The -m gpu tests run the product library."""
import ctypes as C
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from edlib_b200._ffi import REPO, EdlibLib, HitAlignments, make_config
from helpers import mutate, rand_seq
from test_hits import FORCED, cached_row, genome, rc, stats

HERE = os.path.dirname(os.path.abspath(__file__))
EMUL_DIR = os.path.join(HERE, "emul_pair_hits")


def load_emul_pair_hits():
    """The kernel emulation of tests/emul with every kernel of tests/emul_records plus the per-pair hit sweep."""
    subprocess.run(["make", "-s", "-C", EMUL_DIR], check=True)
    return EdlibLib(os.path.join(EMUL_DIR, "libedlib_emul_pair_hits.so"), has_batch=True)


def error(lib):
    lib.lib.edlibB200LastError.restype = C.c_char_p
    return lib.lib.edlibB200LastError().decode()


def expected(qs, ts, k, both, cap, eqs=None):
    """Per pair: the brute-force hits of its query (and rc) over its own target, forward first; the first `cap` listed."""
    out = []
    for q, t in zip(qs, ts):
        hits = []
        for s, qq in enumerate([q, rc(q)] if both else [q]):
            if not t:
                continue
            d = cached_row(qq, t, eqs)
            hits += [(int(c), int(d[c]), s) if both else (int(c), int(d[c])) for c in np.nonzero(d <= k)[0]]
        out.append({"count": len(hits), "hits": hits[:cap]})
    return out


def single(lib, q, t, k, both, cap, eqs, task):
    """The pair's entry as a single-target edlibB200FindHitAlignments call gives it (an empty target: no hits)."""
    if not t:
        d = {"count": 0, "hits": []}
        if task:
            d["starts"] = []
        if task == 2:
            d["alignments"] = []
        return d
    st, res = lib.find_hit_alignments([q], t, k, both, cap, eqs, task)
    assert st == 0, error(lib)
    return res[0]


def check(lib, qs, ts, k, both=False, cap=1 << 40, eqs=None, task=0, singles=None):
    """One pair call against the brute force (and, task LOC / PATH, the single-target calls of the pairs in `singles`,
    default all); returns (decided, fallback, windows) of the pair call."""
    st, got = lib.find_pair_hits(qs, ts, k, both, cap, eqs, task)
    assert st == 0, error(lib)
    s = stats(lib)
    res = (s.filterDecided, s.filterFallback, s.filterWindows)
    assert len(got) == len(qs)
    exp = expected(qs, ts, k, both, cap, eqs)
    for i, (g, e) in enumerate(zip(got, exp)):
        assert {"count": g["count"], "hits": g["hits"]} == e, dict(
            pair=i, k=k, m=len(qs[i]), n=len(ts[i]), both=both, cap=cap, got_count=g["count"], exp_count=e["count"],
            got=g["hits"][:12], exp=e["hits"][:12])
    if task:
        for i in (range(len(qs)) if singles is None else singles):
            g = got[i]
            assert g == single(lib, qs[i], ts[i], k, both, cap, eqs, task), dict(pair=i, k=k, got=str(g)[:600])
            if task == 2:
                for h, a in zip(g["hits"], g["alignments"]):
                    assert sum(1 for op in a if op != 0) == h[1], (i, h)  # EDLIB_EDOP_MATCH == 0
    return res


def planted(rng, n, q, copies, rate):
    """A random target of n symbols with `copies` mutated copies of q (at most ~n / 2 columns each apart)."""
    t = bytearray(genome(rng, n))
    for _ in range(copies):
        c = mutate(rng, q, rate, b"ACGT")
        a = rng.randrange(0, max(1, n - len(c)))
        t[a:a + len(c)] = c[:n - a]
    return bytes(t)


# ---------------------------------------------------------------------------------------------------------------------
# Scenarios (CPU: emulated kernels, one subprocess per set of tunables; GPU: the product library)
# ---------------------------------------------------------------------------------------------------------------------
def word_class_case(seed=21):
    """m = 1, 31, 32, 33, 64, 256 (and a palindrome), each over targets of 0, 1, < m, = m symbols, 3 kbp and ~100 kbp
    with planted copies; the 100 kbp target is one object shared by the queries' pairs (one group below k1MinGroup)."""
    rng = random.Random(seed)
    qs0 = [genome(rng, m) for m in (1, 31, 32, 33, 64, 256)] + [b"ACGTTAACGT" * 3 + b"GAATTC"]
    big = bytearray(genome(rng, 100_000))
    for j, q in enumerate(qs0):
        for c in range(3):
            a = 4_000 + 14_000 * j + 3_000 * c
            big[a:a + len(q)] = mutate(rng, q, 0.02 * c, b"ACGT")[:len(q)].ljust(len(q), b"G")
    big = bytes(big)
    qs, ts = [], []
    for q in qs0:
        m = len(q)
        mid = planted(rng, 3_000, q, 4, 0.03)
        for t in (b"", q[:1], q[:max(1, m // 2)], bytes(q), mid, big):
            qs.append(q)
            ts.append(t)
    return qs, ts


def sc_word_classes(lib):
    qs, ts = word_class_case()
    res = {}
    for k in (0, 3, 12):
        res["k%d" % k] = check(lib, qs, ts, k, both=(k == 3))
    res["all"] = check(lib, qs[:18], ts[:18], 40)  # k >= m for m <= 32: every column of every non-empty target
    big = [i for i, t in enumerate(ts) if len(t) >= 100_000]
    other = [i for i in range(len(ts)) if i not in big]
    for task in (1, 2):
        # the 100 kbp target at k = 3 with a cap (m = 1: every column a hit); the others in full
        res["task%d" % task] = check(lib, qs, ts, 3, both=True, cap=40, task=task)
        res["task%d_all" % task] = check(lib, [qs[i] for i in other], [ts[i] for i in other], 5, both=(task == 2),
                                         task=task)
    return res


def sc_caps(lib):
    """Caps of 0, 1, exactly a pair's count and above it, both strands (forward hits first)."""
    qs, ts = word_class_case(seed=22)
    st, full = lib.find_pair_hits(qs, ts, 4, True, 1 << 40)
    assert st == 0, error(lib)
    counts = [r["count"] for r in full]
    exact = min(c for c in counts if c > 0)
    res = {}
    for cap in (0, 1, exact, max(counts), max(counts) + 5):
        res["cap%d" % cap] = check(lib, qs, ts, 4, both=True, cap=cap, task=1 if cap == exact else 0)
    return res


def sc_chunks(lib):
    """Dense hits all over long targets (tandem copies of the query, and k >= m): with a tiny EDLIB_B200_K1_MIN_CHUNK every
    chunk border and halo holds hits."""
    rng = random.Random(23)
    unit = genome(rng, 40)
    tandem = b"".join(mutate(rng, unit, 0.05, b"ACGT") for _ in range(600))
    qs = [unit, rc(unit), unit[:17], genome(rng, 70), unit * 2]
    ts = [tandem, tandem, tandem, planted(rng, 30_000, qs[3], 20, 0.03), tandem[:9_000]]
    res = {}
    for k in (0, 4, 9):
        res["k%d" % k] = check(lib, qs, ts, k, both=(k == 4))
    res["all"] = check(lib, [unit[:20], unit], [tandem[:5_000], tandem[:3_001]], 45)
    res["path"] = check(lib, qs[:3], ts[:3], 4, cap=300, task=2)
    return res


def mixed_case(seed=24):
    """Queries shared by many pairs; one 120 kbp target shared by 40 queries (group route, seed windows), one 20 kbp
    target shared by 36 (group route, whole-target sweep), targets shared by 3 pairs (per-pair route), unique targets
    and empty ones, interleaved in one call."""
    rng = random.Random(seed)
    g1 = genome(rng, 120_000)
    g2 = genome(rng, 20_000)
    primers = [genome(rng, 20), genome(rng, 24), genome(rng, 45)]
    reads = []
    for _ in range(30):
        r = bytearray(genome(rng, rng.randrange(200, 4_000)))
        for _ in range(rng.randrange(0, 4)):
            p = mutate(rng, rng.choice(primers), 0.05, b"ACGT")
            a = rng.randrange(0, len(r) - len(p))
            r[a:a + len(p)] = p
        reads.append(bytes(r))
    qs, ts = [], []
    for i in range(40):  # a group over g1
        a = rng.randrange(0, len(g1) - 150)
        qs.append(mutate(rng, g1[a:a + 150], 0.03, b"ACGT")[:150] or b"A")
        ts.append(g1)
        if i % 3 == 0:  # each read of the per-pair route with its three primers
            r = reads[i % len(reads)]
            for p in primers:
                qs.append(p)
                ts.append(r)
        if i % 5 == 0:
            qs.append(primers[i % 3])
            ts.append(b"")
        if i < 36:  # a group over g2
            a = rng.randrange(0, len(g2) - 60)
            qs.append(g2[a:a + 60])
            ts.append(g2)
        if i % 4 == 1:  # unique targets
            qs.append(primers[1])
            ts.append(reads[(i + 7) % len(reads)][:] + b"A")
    return qs, ts


def sc_mixed(lib):
    qs, ts = mixed_case()
    res = {}
    for k in (2, 6):
        res["k%d" % k] = check(lib, qs, ts, k, both=(k == 6))
    singles = list(range(0, len(qs), 7))
    res["path"] = check(lib, qs, ts, 4, both=True, cap=25, task=2, singles=singles)
    return res


def sc_equalities(lib):
    """Transitive equalities (collapsed codes) and non-transitive ones (an equality table) with wildcards in the
    targets, on the per-pair route and on a group."""
    rng = random.Random(25)
    g = genome(rng, 30_000)
    g = bytes(c | 0x20 if rng.random() < 0.2 else c for c in g)
    reads = [b"".join(b"N" if rng.random() < 0.03 else bytes([c]) for c in genome(rng, rng.randrange(300, 3_000)))
             for _ in range(10)]
    qs, ts = [], []
    for i in range(40):
        a = rng.randrange(0, len(g) - 80)
        qs.append(bytes(c | 0x20 if rng.random() < 0.3 else c for c in g[a:a + 80].upper()))
        ts.append(g)
    for r in reads:
        a = rng.randrange(0, len(r) - 30)
        qs += [r[a:a + 30].replace(b"N", b"A"), genome(rng, 25)]
        ts += [r, r]
    fold = [(bytes([c]), bytes([c | 0x20])) for c in b"ACGTN"]
    wild = [(b"N", bytes([c])) for c in b"ACGT"]
    return {"fold": check(lib, qs, ts, 5, eqs=fold), "wild": check(lib, qs[40:], ts[40:], 3, eqs=wild, task=2),
            "wild_both": check(lib, qs[40:], ts[40:], 2, both=True, eqs=wild)}


def sc_one_target(lib):
    """Pairs that all share one target: the same arrays and filter counters as edlibB200FindHitAlignments over it, for
    a group below and above k1MinGroup, on the seed route and the whole-target sweep."""
    rng = random.Random(26)
    out = {}
    for name, n, count in (("few", 100_000, 5), ("many", 100_000, 40), ("short", 5_000, 40)):
        t = genome(rng, n)
        qs = []
        for i in range(count):
            a = rng.randrange(0, n - 120)
            qs.append(mutate(rng, t[a:a + 120], 0.03, b"ACGT")[:120] or b"A")
        for k, both, task in ((3, False, 0), (8, True, 2)):
            st, single_res = lib.find_hit_alignments(qs, t, k, both, 30, None, task)
            assert st == 0, error(lib)
            s1 = stats(lib)
            st, pair_res = lib.find_pair_hits(qs, [t] * count, k, both, 30, None, task)
            assert st == 0, error(lib)
            s2 = stats(lib)
            assert pair_res == single_res, (name, k)
            c1 = (s1.filterDecided, s1.filterFallback, s1.filterWindows)
            assert c1 == (s2.filterDecided, s2.filterFallback, s2.filterWindows), (name, k)
            out["%s_k%d" % (name, k)] = c1
    return out


def call_raw(lib, qs, ts, n, k=2, mode=2, task=0, null_out=False, lengths=None, cap=10):
    fn = lib.lib.edlibB200FindPairHits
    fn.restype = C.c_int
    fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int,
                   type(make_config()[0]), C.c_int, C.c_longlong, C.POINTER(HitAlignments)]
    cfg, keep = make_config(k, mode, task)
    qp = (C.c_char_p * max(len(qs), 1))(*qs)
    ql = (C.c_int * max(len(qs), 1))(*[len(q) if q is not None else 4 for q in qs])
    tp = (C.c_char_p * max(len(ts), 1))(*ts)
    tl = (C.c_int * max(len(ts), 1))(*(lengths if lengths is not None else [len(t) if t else 0 for t in ts]))
    a = HitAlignments()
    a.hits.numQueries = 99
    st = fn(qp, ql, tp, tl, n, cfg, 0, cap, None if null_out else C.byref(a))
    del keep
    empty = not (a.hits.counts or a.hits.offsets or a.hits.columns or a.hits.scores or a.hits.strands or a.starts
                 or a.alignmentOffsets or a.alignments)
    return st, empty


def sc_invalid(lib):
    """Invalid input: EDLIB_STATUS_ERROR, a message starting "edlibB200FindPairHits:", nothing allocated."""
    t = b"ACGT" * 100
    out = {}
    for name, kw in [("empty", dict(qs=[b""], ts=[t], n=1)), ("long", dict(qs=[b"A" * 257], ts=[t], n=1)),
                     ("k", dict(qs=[b"ACGT"], ts=[t], n=1, k=-1)), ("nw", dict(qs=[b"ACGT"], ts=[t], n=1, mode=0)),
                     ("shw", dict(qs=[b"ACGT"], ts=[t], n=1, mode=1)), ("null_query", dict(qs=[None], ts=[t], n=1)),
                     ("null_target", dict(qs=[b"ACGT"], ts=[None], n=1, lengths=[5])),
                     ("negative", dict(qs=[b"ACGT"], ts=[t], n=1, lengths=[-1])),
                     ("null_out", dict(qs=[b"ACGT"], ts=[t], n=1, null_out=True)),
                     ("pairs", dict(qs=[b"ACGT"], ts=[t], n=-1)), ("cap", dict(qs=[b"ACGT"], ts=[t], n=1, cap=-1)),
                     ("task", dict(qs=[b"ACGT"], ts=[t], n=1, task=3))]:
        st, empty = call_raw(lib, **kw)
        assert st == 1 and empty, name
        out[name] = error(lib)
        assert out[name].startswith("edlibB200FindPairHits: "), (name, out[name])
    # accepted: no pairs, and NULL targets of length 0
    st, res = lib.find_pair_hits([], [], 2)
    assert st == 0 and res == []
    st, empty = call_raw(lib, [b"ACGT", b"AC"], [None, None], 2, task=2)
    assert st == 0 and not empty
    return out


SCENARIOS = {"word_classes": sc_word_classes, "caps": sc_caps, "chunks": sc_chunks, "mixed": sc_mixed,
             "equalities": sc_equalities, "one_target": sc_one_target, "invalid": sc_invalid}

DRIVER = (
    "import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
    "import test_pair_hits as P\n"
    "lib = P.load_emul_pair_hits()\n"
    "print(json.dumps(P.SCENARIOS[sys.argv[1]](lib)))\n"
) % (REPO, HERE)


def run_scenario(name, env=None):
    e = dict(os.environ, **(env or {}))
    out = subprocess.run([sys.executable, "-c", DRIVER, name], env=e, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-4000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_word_classes_emul():
    res = run_scenario("word_classes", FORCED)
    # 7 queries x 5 non-empty targets, every pair on the per-pair route; no seed windows
    assert res["k0"] == [0, 35, 0] and res["k3"] == [0, 70, 0]


def test_word_classes_small_chunks_emul():
    run_scenario("word_classes", dict(FORCED, EDLIB_B200_K1_MIN_CHUNK="16"))


def test_caps_emul():
    run_scenario("caps", FORCED)


def test_chunks_emul():
    for chunk in ("16", "1024"):
        res = run_scenario("chunks", dict(FORCED, EDLIB_B200_K1_MIN_CHUNK=chunk))
        assert res["k0"][0] == 0 and res["k0"][1] == 5


def test_mixed_routes_emul():
    res = run_scenario("mixed", FORCED)
    # seed windows decide the 120 kbp group; the rest is swept, its own target or the group's
    assert res["k2"][0] > 0 and res["k2"][2] > 0 and res["k2"][1] > 0


def test_mixed_routes_launch_groups_emul():
    """Launch groups of three reads: several per route and word class, the same hits."""
    res = run_scenario("mixed", dict(FORCED, EDLIB_B200_HIT_RUN_READS="3", EDLIB_B200_K1_MIN_CHUNK="16"))
    assert res["k2"][0] > 0


def test_equalities_emul():
    res = run_scenario("equalities", FORCED)
    assert res["wild"][0] == 0 and res["wild"][1] == 20


def test_one_target_emul():
    res = run_scenario("one_target", FORCED)
    assert res["few_k3"][0] > 0 and res["many_k3"][0] > 0  # seed windows even for a few pairs over one target
    assert res["short_k3"][0] == 0 and res["short_k3"][1] == 40


def test_invalid_input_emul():
    res = run_scenario("invalid")
    assert len(res) == 12


def test_backend_without_lane_hits_refuses():
    """A backend without lane_hits (tests/emul_records) refuses a call that needs the per-pair route, with nothing
    allocated, and still runs one whose pairs share one target."""
    from test_record_hits import load_emul_records
    lib = load_emul_records()
    st, res = lib.find_pair_hits([b"ACGTACGT", b"ACGT"], [b"ACGT" * 100, b"ACGT" * 50], 1)
    assert st == 1 and res is None
    assert "no such kernel" in error(lib)
    st, empty = call_raw(lib, [b"ACGTACGT", b"ACGT"], [b"ACGT" * 100, b"CGTA" * 100], 2)
    assert st == 1 and empty
    t = b"ACGT" * 100
    st, res = lib.find_pair_hits([b"ACGTACGT", b"ACGA"], [t, t], 1)
    assert st == 0 and res == expected([b"ACGTACGT", b"ACGA"], [t, t], 1, False, 1 << 40)


def test_python_entry_validation():
    import edlib_b200
    with pytest.raises(ValueError):
        edlib_b200.find_pair_hits([b"ACGT"], [b"ACGT", b"AC"], 1)
    with pytest.raises(ValueError):
        edlib_b200.find_pair_hits([b"ACGT"], [b"ACGT"], 1, strands="reverse")
    with pytest.raises(ValueError):
        edlib_b200.find_pair_hits([b"ACGT"], [b"ACGT"], 1, task="cigar")


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
def test_emulation_matches_gpu():
    """The same seeded mixed call through the emulation and the H100: identical entries, starts and scripts included."""
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_pair_hits as P\n"
            "qs, ts = P.mixed_case(31)\n"
            "st, res = P.load_emul_pair_hits().find_pair_hits(qs, ts, 5, True, 40, None, 2)\n"
            "assert st == 0\n"
            "for r in res: r['alignments'] = [a.hex() for a in r['alignments']]\n"
            "print(json.dumps(res))\n") % (REPO, HERE)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **FORCED))
    assert out.returncode == 0, out.stderr[-3000:]
    emul = json.loads(out.stdout.strip().splitlines()[-1])
    qs, ts = mixed_case(31)
    st, res = product_lib().find_pair_hits(qs, ts, 5, True, 40, None, 2)
    assert st == 0
    for r in res:
        r["alignments"] = [a.hex() for a in r["alignments"]]
        r["hits"] = [list(h) for h in r["hits"]]
    assert res == emul


def ecoli_pairs(rate_max=0.10):
    """The reads of tests/golden/ecoli_reads.json (50 bp - 10 kbp) as targets, each with primer- and adapter-like
    queries planted 0-3 times at seeded places with 0-10 % edits, plus queries that were not planted."""
    with open(os.path.join(HERE, "golden", "ecoli_reads.json")) as f:
        fx = json.load(f)
    reads = [r["seq"].encode("ascii") for _, r in sorted(fx["reads"].items())]
    rng = random.Random(40)
    adapters = [genome(rng, 30), genome(rng, 20), genome(rng, 22), genome(rng, 58)]
    qs, ts = [], []
    for r in reads:
        t = bytearray(r)
        for a in adapters:
            for _ in range(rng.randrange(0, 4)):
                c = mutate(rng, a, rng.random() * rate_max, b"ACGT")
                at = rng.randrange(0, max(1, len(t) - len(c)))
                t[at:at + len(c)] = c[:len(t) - at]
        t = bytes(t)
        for a in adapters:
            qs.append(a)
            ts.append(t)
    return qs, ts


@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 3, 6])
def test_ecoli_reads_gpu(k):
    qs, ts = ecoli_pairs()
    lib = product_lib()
    check(lib, qs, ts, k, both=(k == 3))
    check(lib, qs, ts, k, both=True, cap=20, task=2, singles=range(0, len(qs), 9))


@pytest.mark.gpu
def test_scripts_against_reference_gpu():
    """A sample of scripts: edlibAlign(q, T[start..c], NW, PATH) of the reference build gives the same script."""
    from helpers import have_ref, ref
    if not have_ref():
        pytest.skip("reference build not available")
    qs, ts = ecoli_pairs()
    st, got = product_lib().find_pair_hits(qs, ts, 6, True, 50, None, 2)
    assert st == 0
    r = ref()
    rng = random.Random(41)
    seen = 0
    for i in rng.sample(range(len(qs)), 120):
        g = got[i]
        for (c, s, strand), st0, aln in list(zip(g["hits"], g["starts"], g["alignments"]))[:6]:
            q = rc(qs[i]) if strand else qs[i]
            e = r.align(q, ts[i][st0:c + 1], -1, 0, 2)
            assert e["editDistance"] == s and e["alignment"] == aln, (i, c)
            seen += 1
    assert seen > 50


@pytest.mark.gpu
def test_python_entry_gpu():
    import edlib_b200
    qs, ts = mixed_case(32)
    lib = product_lib()
    for strands, both in (("forward", False), ("both", True)):
        for task, code in (("distance", 0), ("path", 2)):
            got = edlib_b200.find_pair_hits(qs, ts, 4, strands=strands, max_hits=9, task=task)
            st, raw = lib.find_pair_hits(qs, ts, 4, both, 9, None, code)
            assert st == 0
            for r in raw:
                if both:
                    r["hits"] = [h[:-1] + ("-" if h[-1] else "+",) for h in r["hits"]]
                if "alignments" in r:
                    r["cigars"] = [lib.cigar(a) for a in r.pop("alignments")]
            assert got == raw
    # str sequences, and a repeated object shares one target
    t = "ACGTTGCA" * 40
    got = edlib_b200.find_pair_hits(["TTGCA", "ACGTT"], [t, t], 0)
    assert [r["count"] for r in got] == [40, 40]
    with pytest.raises(Exception):
        edlib_b200.find_pair_hits([b"A" * 300], [b"ACGT"], 3)
