"""Both strands of a read set in one call (edlibB200AlignBatchStrands, edlibB200BatchPrepareStrands, align_batch(...,
strands="both")): every field of every result, and the strand, against the reference build run on the read and on its
reverse complement, with the rule of include/edlib_b200.h (the reverse strand wins only with a strictly smaller
distance).  CPU tests run the engine on the emulated kernels in subprocesses with forced tunables; the -m gpu tests
run the product library."""
import ctypes as C
import json
import os
import random
import subprocess

import pytest

import parity
from edlib_b200._ffi import REPO, AlignConfig, AlignResult, make_config, result_to_dict
from helpers import mutate, rand_seq

HERE = os.path.dirname(os.path.abspath(__file__))

_PAIRS = [b"AT", b"CG", b"RY", b"KM", b"BV", b"DH"]
_COMP = bytearray(range(256))
for _a, _b in _PAIRS:
    for x, y in ((_a, _b), (_a | 0x20, _b | 0x20)):
        _COMP[x], _COMP[y] = y, x
_COMP = bytes(_COMP)


def rc(q):
    return bytes(q).translate(_COMP)[::-1]


def expected(chk, q, t, k, mode, task, eqs):
    f = chk.align(q, t, k, mode, task, eqs)
    r = chk.align(rc(q), t, k, mode, task, eqs)
    if f.get("status", 0) == 0 and r["editDistance"] >= 0 and (f["editDistance"] < 0 or r["editDistance"] < f["editDistance"]):
        return r, 1
    return f, 0


def run_cases(lib, cases):
    chk = parity.checker()
    n = 0
    for c in cases:
        st, res, strands = lib.align_batch_strands(c["qs"], c["ts"], c["k"], c["mode"], c["task"], c["eqs"])
        assert st == 0
        for i, (q, t) in enumerate(zip(c["qs"], c["ts"])):
            exp, s = expected(chk, q, t, c["k"], c["mode"], c["task"], c["eqs"])
            assert (res[i], strands[i]) == (exp, s), dict(pair=i, k=c["k"], mode=c["mode"], task=c["task"], m=len(q), n=len(t),
                                                         q=q[:80], got=str(res[i])[:300], exp=str(exp)[:300], strand=strands[i])
            n += 1
    return n


SPICE = b"NNacgtRYKMBVDHSWX#"


def read_from(rng, t, m, rate):
    """A read of about m bytes from either strand of t: errors, unrelated reads, N / lowercase / IUPAC / foreign bytes."""
    a = rng.randrange(0, len(t) - m)
    q = mutate(rng, t[a:a + m], rate, b"ACGT")[:256] or b"A"
    if rng.random() < 0.1:
        q = rand_seq(rng, m, b"ACGT")
    if rng.random() < 0.2:
        q = bytearray(q)
        for _ in range(rng.randrange(1, 4)):
            q[rng.randrange(len(q))] = rng.choice(SPICE)
        q = bytes(q)
    return rc(q) if rng.random() < 0.5 else q


def random_cases(seed, count, lengths=(20_000, 50_000, 200_000), reads=(80, 60, 24)):
    rng = random.Random(seed)
    for i in range(count):
        j = i % len(lengths)
        t = rand_seq(rng, lengths[j], b"ACGT")
        qs = [read_from(rng, t, rng.randrange(20, 257), rng.choice([0, 0.01, 0.03, 0.08, 0.15])) for _ in range(reads[j])]
        yield dict(qs=qs, ts=[t] * len(qs), k=rng.choice([-1, 0, 3, 12, 40]), mode=2, task=i % 3, eqs=None)


def shape_cases(seed):
    rng = random.Random(seed)
    t = rand_seq(rng, 6000, b"ACGT")
    for mode in (0, 1):  # NW and SHW, per-pair targets
        qs, ts = [], []
        for _ in range(40):
            a = rng.randrange(0, 5000)
            x = t[a:a + rng.randrange(30, 300)]
            q = mutate(rng, x, 0.05, b"ACGT")
            qs.append(rc(q) if rng.random() < 0.5 else q)
            ts.append(x)
        for task in (0, 1, 2):
            yield dict(qs=qs, ts=ts, k=rng.choice([-1, 20]), mode=mode, task=task, eqs=None)
    # long queries over a long target: the seeded long-query path (LONG_HW_MIN_TARGET lowered)
    lt = rand_seq(rng, 12000, b"ACGT")
    qs = []
    for _ in range(6):
        a = rng.randrange(0, 11000)
        q = mutate(rng, lt[a:a + rng.randrange(300, 900)], 0.04, b"ACGT")
        qs.append(rc(q) if rng.random() < 0.5 else q)
    for k in (-1, 30):
        yield dict(qs=qs, ts=[lt] * len(qs), k=k, mode=2, task=1, eqs=None)
    # equalities: case folding (transitive: collapsed to one code per group) and a wildcard (non-transitive)
    mixed = [bytes(ch | 0x20 if rng.random() < 0.3 else ch for ch in q) for q in qs[:3]]
    short = [read_from(rng, t, rng.randrange(40, 200), 0.03) for _ in range(30)]
    short = [bytes(ch | 0x20 if rng.random() < 0.3 else ch for ch in q) for q in short]
    fold = [(bytes([c]), bytes([c | 0x20])) for c in b"ACGT"]
    wild = [(b"N", bytes([c])) for c in b"ACGT"]
    for eqs in (fold, wild):
        yield dict(qs=short + mixed, ts=[t] * (len(short) + 3), k=-1, mode=2, task=2, eqs=eqs)
    # empty reads, palindromes (tie: forward), both strands beyond k (forward, -1)
    pal = b"ACGTTAACGT"
    odd = [b"", pal, t[100:180], rc(t[300:400]), rand_seq(rng, 60, b"ACGT"), b"GAATTC" * 5, rc(b"GAATTC" * 5)]
    for mode in (0, 1, 2):
        for k in (-1, 2):
            yield dict(qs=odd, ts=[t] * len(odd), k=k, mode=mode, task=2, eqs=None)


DRIVER = (
    "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
    "import test_strands as S, test_engine_emul as T\n"
    "lib = T.load_emul()\n"
    "print(S.run_cases(lib, GEN))\n"
) % (REPO, HERE)

FORCED = dict(EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_K1_MIN_GROUP="4")


def run_driver(gen, extra):
    env = dict(os.environ, **FORCED, **extra)
    out = subprocess.run(["python", "-c", DRIVER.replace("GEN", gen)], env=env, check=True, capture_output=True, text=True)
    return int(out.stdout.strip().splitlines()[-1]), out.stderr


def test_complement_table_on_every_byte():
    from test_engine_emul import load_emul
    rng = random.Random(3)
    q = bytearray(range(1, 256))
    rng.shuffle(q)
    q = bytes(q)
    assert rc(rc(q)) == q
    assert rc(b"AaCcRrKkBbDdNSW#") == b"#WSNhHvVmMyYgGtT"
    lib = load_emul()
    st, res, strands = lib.align_batch_strands([q], [rc(q)], -1, 0, 2)
    assert st == 0 and strands == [1] and res[0]["editDistance"] == 0
    assert res[0] == parity.checker().align(rc(q), rc(q), -1, 0, 2)


def test_reads_longer_than_one_presence_item():
    """Reads above 65536 bytes are cut into several presence-set work items; each piece writes its part of the reverse
    complement (and of its presence set), next to short reads of the same batch."""
    from test_engine_emul import load_emul
    rng = random.Random(4)
    big = rand_seq(rng, 70000, b"ACGTN")
    t1 = rc(mutate(rng, big, 0.001, b"ACGT"))
    short = rand_seq(rng, 120, b"ACGT")
    t2 = mutate(rng, short, 0.05, b"ACGT")
    case = dict(qs=[short, big, rc(short)], ts=[t2, t1, t2], k=-1, mode=0, task=0, eqs=None)
    assert run_cases(load_emul(), [case]) == 3


@pytest.mark.parametrize("extra",[{}, {"EDLIB_B200_DEVICE_STAGE": "0"}, {"EDLIB_B200_FILTER_SEED_K": "0"},
                                   {"EDLIB_B200_FILTER_SEED_LEVELS": "1", "EDLIB_B200_SLICE_READS": "64"},
                                   {"EDLIB_B200_FILTER_SEED_BUCKET": "2"}],
                         ids=["default", "host-driven", "no-seeds", "one-level-slices", "tight-bucket"])
def test_random_read_sets_forced_filter(extra):
    n, _ = run_driver("S.random_cases(11, 6)", extra)
    assert n >= 300


def test_other_shapes():
    n, _ = run_driver("S.shape_cases(5)", {"EDLIB_B200_LONG_HW_MIN_TARGET": "2000"})
    assert n >= 300


class Stats(C.Structure):  # include/edlib_b200.h EdlibB200Stats
    _fields_ = [("kernelMs", C.c_double), ("k1Ms", C.c_double), ("launches", C.c_int), ("filterWindows", C.c_int),
                ("h2dBytes", C.c_longlong), ("d2hBytes", C.c_longlong), ("k1Cells", C.c_longlong), ("wCells", C.c_longlong),
                ("filterDecided", C.c_longlong), ("filterFallback", C.c_longlong)]


BOUND_CODE = """
import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)
import ctypes as C, random
import test_strands as S, test_engine_emul as T
from helpers import mutate, rand_seq
lib = T.load_emul()
rng = random.Random(8)
t = rand_seq(rng, 200_000, b"ACGT")
M, N = int(sys.argv[1]), int(sys.argv[2])
true = []
for _ in range(N):
    a = rng.randrange(0, len(t) - M - 10)
    true.append(mutate(rng, t[a:a + M], rng.choice([0, 0.01, 0.02, 0.03]), b"ACGT")[:M])
mixed = [S.rc(q) if i %% 2 else q for i, q in enumerate(true)]
def fallback():
    s = S.Stats()
    lib.lib.edlibB200LastStats(C.byref(s))
    return s.filterFallback
st, fwd = lib.align_batch(true, [t] * N, -1, 2, 1)
assert st == 0
f = fallback()
st, res, strands = lib.align_batch_strands(mixed, [t] * N, -1, 2, 1)
assert st == 0
b = fallback()
for i in range(N):
    assert res[i]["editDistance"] == fwd[i]["editDistance"] and strands[i] == (1 if i %% 2 else 0), i
print(f, b)
""" % (REPO, HERE)


def test_the_other_strand_bounds_the_filter():
    """Reads of <= 3 %% error from both strands: the losing strand is settled by the winner's distance, so the strand batch
    sends no more reads to the plain full sweep than a forward-only batch of the truly oriented reads; 10 kbp reads never
    take the chunked sweep of the whole target."""
    out = subprocess.run(["python", "-c", BOUND_CODE, "150", "200"], check=True, capture_output=True, text=True)
    f, b = map(int, out.stdout.split())
    assert b <= f
    env = dict(os.environ, EDLIB_B200_TRACE="1")
    out = subprocess.run(["python", "-c", BOUND_CODE, "10000", "4"], env=env, check=True, capture_output=True, text=True)
    assert "long HW queries, seed threshold" in out.stderr
    assert "long HW queries, chunked sweeps" not in out.stderr


def bind_staged(L):
    L.edlibB200BatchPrepareStrands.restype = C.c_void_p
    L.edlibB200BatchPrepare.restype = C.c_void_p
    args = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, AlignConfig]
    L.edlibB200BatchPrepareStrands.argtypes = args
    L.edlibB200BatchPrepare.argtypes = args
    L.edlibB200BatchCompute.argtypes = [C.c_void_p, C.c_void_p]
    L.edlibB200BatchResults.argtypes = [C.c_void_p, C.POINTER(AlignResult)]
    L.edlibB200BatchStrands.argtypes = [C.c_void_p, C.POINTER(C.c_ubyte)]
    L.edlibB200BatchFree.argtypes = [C.c_void_p]


def test_staged_strand_batches():
    from test_engine_emul import load_emul
    lib = load_emul()
    L = lib.lib
    bind_staged(L)
    c = next(random_cases(21, 1, lengths=(30_000,), reads=(90,)))
    qs, t, n = c["qs"], c["ts"][0], len(c["qs"])
    tb = C.create_string_buffer(t, len(t))
    arrs = ((C.c_char_p * n)(*qs), (C.c_int * n)(*[len(q) for q in qs]), (C.c_char_p * n)(*[C.cast(tb, C.c_char_p)] * n),
            (C.c_int * n)(*[len(t)] * n))
    cfg, keep = make_config(12, 2, 2, None)
    h = L.edlibB200BatchPrepareStrands(*arrs, n, cfg)
    assert h
    strands = (C.c_ubyte * n)()
    assert L.edlibB200BatchStrands(h, strands) == 1  # not computed yet
    outs = []
    for _ in range(2):
        assert L.edlibB200BatchCompute(h, None) == 0
        res = (AlignResult * n)()
        assert L.edlibB200BatchResults(h, res) == 0
        assert L.edlibB200BatchStrands(h, strands) == 0
        outs.append(([result_to_dict(res[i]) for i in range(n)], list(strands)))
        for i in range(n):
            lib.free(res[i])
    L.edlibB200BatchFree(h)
    st, one, s1 = lib.align_batch_strands(qs, [t] * n, 12, 2, 2)
    assert st == 0 and outs[0] == outs[1] == (one, s1)
    assert 0 < sum(s1) < n
    plain = L.edlibB200BatchPrepare(*arrs, n, cfg)
    assert plain and L.edlibB200BatchCompute(plain, None) == 0
    assert L.edlibB200BatchStrands(plain, strands) == 1
    L.edlibB200BatchFree(plain)
    del keep


def test_python_mirror_strands(monkeypatch):
    import edlib_b200
    from test_engine_emul import load_emul
    lib = load_emul()
    lib.lib.edlibB200LastError.restype = C.c_char_p
    monkeypatch.setattr(edlib_b200, "_lib", lib)
    t = "ACGTTGCAATGCCGTAAGGCTTAACGGATCCA" * 20
    qs = ["TTGCAATGC", rc(b"AAGGCTTAACGG").decode(), "GGGGGGGG", ""]
    got = edlib_b200.align_batch(qs, t, mode="HW", task="path", strands="both")
    assert [g["strand"] for g in got] == ["+", "-", "+", "+"]
    assert got[1]["editDistance"] == 0
    fwd = edlib_b200.align_batch(qs, t, mode="HW", task="path")
    assert "strand" not in fwd[0] and {k: v for k, v in got[0].items() if k != "strand"} == fwd[0]
    with pytest.raises(ValueError):
        edlib_b200.align_batch([[1, 2, 3]], [1, 2, 3, 4], strands="both")
    with pytest.raises(ValueError):
        edlib_b200.align_batch(["ты"], "ACGT", strands="both")


# ---- GPU -------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_random_read_sets_on_gpu():
    from helpers import product
    lib = product()
    assert lib.lib.edlibB200Available() == 1
    assert run_cases(lib, random_cases(31, 6, lengths=(200_000, 1_000_000), reads=(3000, 2000))) >= 10000
    assert run_cases(lib, shape_cases(7)) >= 300


def ecoli():
    from edlib_b200 import workloads
    with open(os.path.join(HERE, "golden", "ecoli_reads.json")) as f:
        fx = json.load(f)
    return workloads.ecoli_genome().tobytes(), fx["reads"]


@pytest.mark.gpu
def test_ecoli_reads_and_their_reverse_complements_on_gpu():
    from helpers import product
    lib = product()
    genome, reads = ecoli()
    names = sorted(n for n in reads if 0 < len(reads[n]["seq"]) <= 500)
    seqs = [reads[n]["seq"].encode("ascii") for n in names]
    seqs = seqs + [rc(q) for q in seqs]
    assert run_cases(lib, [dict(qs=seqs, ts=[genome] * len(seqs), k=-1, mode=2, task=1, eqs=None)]) == len(seqs)


@pytest.mark.gpu
def test_ecoli_long_reads_reverse_complemented_on_gpu():
    from helpers import product
    lib = product()
    genome, reads = ecoli()
    names = sorted(n for n in reads if len(reads[n]["seq"]) > 5000 and reads[n]["editDistance"] <= 0.2 * len(reads[n]["seq"]))
    assert names
    seqs = [rc(reads[n]["seq"].encode("ascii")) for n in names]
    st, res, strands = lib.align_batch_strands(seqs, [genome] * len(seqs), -1, 2, 1)
    assert st == 0 and strands == [1] * len(seqs)
    for n, r in zip(names, res):
        exp = reads[n]
        assert (r["editDistance"], r["endLocations"], r["startLocations"], r["alphabetLength"]) == \
               (exp["editDistance"], exp["endLocations"], exp["startLocations"], exp["alphabetLength"]), n
