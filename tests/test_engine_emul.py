"""CPU tests of the host engine + kernel LOGIC: the real planner (eb_engine.cpp and the eb_pass_*.cpp / eb_wrunner.cpp units) drives the real
kernel bodies (eb_core.h) through the host SIMT emulation backend (tests/emul/), and every
result field is compared with the reference build / oracle.  No GPU involved; the product
library is not used here (its CUDA path is covered by the -m gpu tests)."""
import os
import subprocess

import pytest

import parity
from edlib_b200._ffi import REPO, EdlibLib

EMUL_DIR = os.path.join(REPO, "tests", "emul")


def load_emul(env=None):
    subprocess.run(["make", "-s", "-C", EMUL_DIR], check=True)
    return EdlibLib(os.path.join(EMUL_DIR, "libedlib_emul.so"), has_batch=True)


@pytest.fixture(scope="module")
def emul():
    return load_emul()


def test_known_and_golden(emul):
    parity.run_known(emul)
    assert parity.run_golden(emul) > 200


def test_single_pairs(emul):
    assert parity.run_single(emul, 11, 1500) == 1500


def test_batches_shared_targets(emul):
    assert parity.run_batches(emul, 12, 30) > 1000


def test_pairwise_batches_with_own_targets(emul):
    import cases
    assert parity.run_batches(emul, 17, 40, gen=cases.pairwise_cases) > 1500


def test_long_queries(emul):
    import cases
    assert parity.run_single(emul, 13, 40, gen=cases.long_cases) == 40


def test_banded_nw_of_long_queries_on_the_band_kernel():
    """k-banded NW sweeps of long queries: thread-per-alignment band kernel (several window sizes in one batch), and the
    same batches on the warp kernel's sliding window (EDLIB_B200_BAND_KERNEL=0)."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 61, 10, gen=cases.band_cases))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    for extra, want in (({}, True), ({"EDLIB_B200_BAND_KERNEL": "0"}, False)):
        env = dict(os.environ, EDLIB_B200_TRACE="1", **extra)
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) >= 30
        assert ("band kernel:" in out.stderr) == want


def test_chunked_sweeps_and_overflow_retry():
    """Same batches with tiny chunk / overflow limits so that target chunking with halo, the
    overflow list and its exact-size second pass are all exercised (separate process: the
    tunables are read once per process)."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 14, 30))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    env = dict(os.environ, EDLIB_B200_K1_MIN_CHUNK="64", EDLIB_EMUL_SMS="64", EDLIB_B200_OVF_CAP="3",
               EDLIB_B200_K1_MIN_GROUP="4", EDLIB_B200_SLICE_MB="1")
    out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
    assert int(out.stdout.strip().splitlines()[-1]) > 1000


def test_paths_beyond_the_stored_matrix_rule(emul):
    import cases
    assert parity.run_single(emul, 15, 60, gen=cases.path_cases) == 60


def test_candidate_filter_all_branches():
    """Seed stage + prefix stages + window verification + fallbacks, forced on for small targets
    (separate processes: tunables are read once), under settings that push reads through every branch
    (tight thresholds / spread / window and bucket limits, single stages alone)."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 16, 25, gen=cases.filter_cases))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    for extra in ({}, {"EDLIB_B200_FILTER_K0": "4", "EDLIB_B200_FILTER_K1": "2", "EDLIB_B200_FILTER_SPREAD": "64",
                       "EDLIB_B200_FILTER_MAX_WINDOWS": "2", "EDLIB_B200_K1_MIN_CHUNK": "64", "EDLIB_EMUL_SMS": "64"},
                  {"EDLIB_B200_FILTER_K1": "0", "EDLIB_B200_FILTER_SEED_K": "3", "EDLIB_B200_FILTER_SEED_BUCKET": "2",
                   "EDLIB_B200_FILTER_SKIP_REPEATS": "0"},
                  {"EDLIB_B200_FILTER_K0": "0", "EDLIB_B200_FILTER_K1": "12", "EDLIB_B200_FILTER_SEED_K": "0"},
                  {"EDLIB_B200_WINDOW_CHECK": "0"}, {"EDLIB_B200_WINDOW_CHECK": "-1", "EDLIB_B200_FILTER_SEED_LEVELS": "2"},
                  {"EDLIB_B200_FILTER_K0": "0", "EDLIB_B200_FILTER_K1": "0", "EDLIB_B200_FILTER_SEED_K": "40",
                   "EDLIB_B200_FILTER_SEED_LEVELS": "3", "EDLIB_B200_FILTER_SEED_SLACK": "100000"},
                  {"EDLIB_B200_DEVICE_STAGE": "0"},                                   # every stage host-driven
                  {"EDLIB_B200_TINY_SWEEP_READS": "8", "EDLIB_B200_FILTER_SEED_K": "2"},  # few undecided reads: (read, chunk) lane jobs
                  {"EDLIB_B200_SLICE_READS": "64", "EDLIB_B200_FILTER_SEED_LEVELS": "1"}):  # many slices, one seed level
        prefix_only = extra.get("EDLIB_B200_FILTER_SEED_K") == "0"
        env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_K1_MIN_GROUP="4", **extra)
        if prefix_only:
            env["EDLIB_B200_TRACE"] = "1"
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) > 500
        if prefix_only:
            assert "filter stage P=" in out.stderr  # the prefix stages ran


def test_tightest_bounds_through_every_filter_path():
    """k = 0, 1, 2 (thresholds t = 0, 1, 2): exact and nearly exact reads through the device-driven seed level (staged and
    streamed), the host-driven seed levels, the prefix stages alone and the plain sweep."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 101, 12, gen=cases.small_k_cases))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    for extra in ({}, {"EDLIB_B200_STREAM_MIN_PAIRS": "8"}, {"EDLIB_B200_DEVICE_STAGE": "0"},
                  {"EDLIB_B200_FILTER_SEED_K": "0"}, {"EDLIB_B200_FILTER_SEED_K": "0", "EDLIB_B200_FILTER_K0": "0", "EDLIB_B200_FILTER_K1": "0"},
                  {"EDLIB_B200_WINDOW_CHECK": "0"}, {"EDLIB_B200_WINDOW_CHECK": "-1"}, {"EDLIB_B200_TINY_SWEEP_READS": "8"}):
        env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_K1_MIN_GROUP="4", **extra)
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) > 400


def test_reads_that_tie_on_many_end_columns():
    """Homopolymer / tandem stretches: windows with more end columns than a record holds inline (overflow list of the
    window sweeps), through the device-driven first seed level (streamed and staged), the host-driven seed levels and
    the prefix stages alone."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 51, 8, gen=cases.tied_ends_cases))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    for extra in ({"EDLIB_B200_STREAM_MIN_PAIRS": "8"}, {"EDLIB_B200_DEVICE_STAGE": "0"},
                  {"EDLIB_B200_FILTER_SEED_K": "0", "EDLIB_B200_FILTER_K1": "12"},
                  {"EDLIB_B200_STREAM_MIN_PAIRS": "8", "EDLIB_B200_SLICE_READS": "64", "EDLIB_B200_FILTER_SEED_BUCKET": "4096"}):
        prefix_only = extra.get("EDLIB_B200_FILTER_SEED_K") == "0"
        env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_K1_MIN_GROUP="4", **extra)
        if prefix_only:
            env["EDLIB_B200_TRACE"] = "1"
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) > 300
        if prefix_only:
            assert "filter stage P=" in out.stderr  # the prefix stages ran


def test_start_locations_and_paths_driven_from_the_device():
    """LOC / PATH of short queries: jobs derived on the device from the per-pair results (shared and per-pair targets,
    several word classes per batch, slices of a few pairs).  What the device route does not take runs through the job
    runner: NW paths of short queries over targets longer than a device-driven path slice (word classes with enough
    pairs for the lane kernel and with too few), and the short-row Hirschberg leaves of batches of long paths."""
    head = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    device = head + (
        "a = parity.run_batches(lib, 71, 25)\n"
        "b = parity.run_batches(lib, 72, 25, gen=cases.pairwise_cases)\n"
        "c = parity.run_batches(lib, 73, 12, gen=cases.stream_cases)\n"
        "print(a + b + c)\n"
    )
    host = head + (
        "a = parity.run_batches(lib, 74, 6, gen=cases.long_target_path_cases)\n"
        "b = parity.run_batches(lib, 76, 4, gen=cases.path_batch_cases)\n"
        "print(a + b)\n"
    )
    for code, extra, least, marks in ((device, {}, 2500, ("device-driven lane sweeps", "device-driven leaf sweeps")),
                                      (device, {"EDLIB_B200_SLICE_MB": "1", "EDLIB_B200_K1_MIN_GROUP": "4"}, 2500,
                                       ("device-driven lane sweeps", "device-driven leaf sweeps")),
                                      (host, {}, 300, ("paths: leaf sweeps + tracebacks",))):
        env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_STREAM_MIN_PAIRS="8", EDLIB_B200_TRACE="1", **extra)
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) > least
        assert all(mark in out.stderr for mark in marks)


def test_read_sets_with_additional_equalities():
    """Case-folding equalities collapse to one code per group (seed filter and lane kernels without the table), a
    wildcard keeps the table; also with the collapse switched off."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 91, 9, gen=cases.equality_read_cases))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    for extra, seeds in (({}, True), ({"EDLIB_B200_COLLAPSE_EQUALITIES": "0"}, False)):
        env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_K1_MIN_GROUP="4", EDLIB_B200_TRACE="1", **extra)
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) > 300
        assert ("filter seed stage" in out.stderr or "device stage" in out.stderr) == seeds


DIRECT_UPLOAD_CODE = """
import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)
import ctypes as C, random
import numpy as np
import parity
from edlib_b200._ffi import AlignResult, make_config, result_to_dict
from helpers import mutate, rand_seq
lib = LOAD
chk = parity.checker()
rng = random.Random(5)
total = 0
for mode, task, shared in ((2, 1, True), (2, 0, True), (0, 0, False), (2, 2, False)):
    n, m = 300, 150
    t = rand_seq(rng, 6000, b"ACGT")
    reads = ALLOC((n, m))          # ONE block: query i starts where query i-1 ends
    for i in range(n):
        a = rng.randrange(0, len(t) - m - 20)
        q = (mutate(rng, t[a:a + m + 10], 0.03, b"ACGT") + b"A" * m)[:m]
        reads[i] = np.frombuffer(q, dtype=np.uint8)
    tb = [C.create_string_buffer(t, len(t))] if shared else [C.create_string_buffer(t[i %% 50:], len(t) - i %% 50) for i in range(n)]
    tl = [len(t)] * n if shared else [len(t) - i %% 50 for i in range(n)]
    qptr = (C.c_char_p * n)(*[C.cast(reads.ctypes.data + i * m, C.c_char_p) for i in range(n)])
    qlen = (C.c_int * n)(*[m] * n)
    tptr = (C.c_char_p * n)(*[C.cast(tb[0 if shared else i], C.c_char_p) for i in range(n)])
    tlen = (C.c_int * n)(*tl)
    cfg, keep = make_config(-1, mode, task, None)
    res = (AlignResult * n)()
    assert lib.lib.edlibAlignBatch(qptr, qlen, tptr, tlen, n, cfg, res) == 0
    for i in range(n):
        got = result_to_dict(res[i])
        lib.free(res[i])
        tt = t if shared else t[i %% 50:]
        assert got == chk.align(reads[i].tobytes(), tt, -1, mode, task, None), (mode, task, i)
    total += n
print(total)
"""


def test_queries_in_one_pinned_block_are_uploaded_directly():
    """Queries that lie back to back in page-locked caller memory skip the staging copy (streamed read sets and grouped
    batches); the emulation backend is told to treat every host buffer as pinned."""
    code = (DIRECT_UPLOAD_CODE % (REPO, os.path.join(REPO, "tests"))).replace("LOAD", "__import__('test_engine_emul').load_emul()") \
        .replace("ALLOC", "(lambda shape: np.zeros(shape, dtype=np.uint8))")
    for extra in ({"EDLIB_EMUL_PINNED": "1"}, {"EDLIB_EMUL_PINNED": "1", "EDLIB_B200_PACK_PARALLEL_KB": "16", "EDLIB_B200_HOST_THREADS": "4"},
                  {"EDLIB_EMUL_PINNED": "1", "EDLIB_B200_DIRECT_UPLOAD": "0"}):
        env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_STREAM_MIN_PAIRS="8", EDLIB_B200_DIRECT_MIN_KB="1", **extra)
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) == 1200


TARGET_HANDLE_CODE = """
import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)
import ctypes as C, random
import parity, cases
from edlib_b200._ffi import AlignResult, make_config, result_to_dict
lib = LOAD
L = lib.lib
L.edlibB200TargetPrepare.restype = C.c_void_p
L.edlibB200TargetPrepare.argtypes = [C.c_char_p, C.c_int]
L.edlibB200TargetFree.argtypes = [C.c_void_p]
chk = parity.checker()
total = 0
for c in cases.stream_cases(81, 6):
    t = c["ts"][0]
    tb = C.create_string_buffer(t, len(t))
    n = len(c["qs"])
    qptr = (C.c_char_p * n)(*c["qs"]); qlen = (C.c_int * n)(*[len(q) for q in c["qs"]])
    tptr = (C.c_char_p * n)(*[C.cast(tb, C.c_char_p)] * n); tlen = (C.c_int * n)(*[len(t)] * n)
    cfg, keep = make_config(c["k"], c["mode"], c["task"], None)
    outs = []
    for use_handle in (False, True, True):
        h = L.edlibB200TargetPrepare(C.cast(tb, C.c_char_p), len(t)) if use_handle else None
        assert (h is not None and h != 0) == use_handle
        res = (AlignResult * n)()
        assert L.edlibAlignBatch(qptr, qlen, tptr, tlen, n, cfg, res) == 0
        outs.append([result_to_dict(res[i]) for i in range(n)])
        for i in range(n):
            lib.free(res[i])
        if h:
            L.edlibB200TargetFree(h)
    assert outs[0] == outs[1] == outs[2]
    for i in range(0, n, 7):
        assert outs[1][i] == chk.align(c["qs"][i], t, c["k"], c["mode"], c["task"], None)
    total += n
print(total)
"""


def test_target_handle():
    """edlibB200TargetPrepare: batches against a target kept resident (encoded bytes + seed index reused) give what
    the same call gives without a handle, handle after handle."""
    code = (TARGET_HANDLE_CODE % (REPO, os.path.join(REPO, "tests"))).replace("LOAD", "__import__('test_engine_emul').load_emul()")
    env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_STREAM_MIN_PAIRS="8", EDLIB_B200_TRACE="1")
    out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
    assert int(out.stdout.strip().splitlines()[-1]) > 500
    assert "stream: slices enqueued" in out.stderr


def test_streamed_batches():
    """edlibAlignBatch on read-set-shaped HW batches goes through the streamed path (slices packed and uploaded
    under the kernels of earlier slices, results assembled on the device, result structs built per slice): the
    size limits are lowered so that small batches take it, with one host thread, several, and slices of 64 reads."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 31, 18, gen=cases.stream_cases))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    for extra in ({"EDLIB_B200_HOST_THREADS": "1"}, {"EDLIB_B200_HOST_THREADS": "5", "EDLIB_B200_SLICE_READS": "64"},
                  {"EDLIB_B200_HOST_THREADS": "3", "EDLIB_B200_SLICE_READS": "100", "EDLIB_B200_FILTER_SEED_BUCKET": "2",
                   "EDLIB_B200_FILTER_SEED_K": "5"}):
        env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_STREAM_MIN_PAIRS="8", EDLIB_B200_TRACE="1", **extra)
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) > 2000
        assert "stream: slices enqueued" in out.stderr  # the streamed path really ran


def test_long_queries_hw_over_long_targets():
    """HW, queries above 256 rows over a long target: seed levels with doubling thresholds + sliding warp windows, then
    chunked sweeps with 2m halos (eb_pass_results.cpp: long_hw_distance); limits lowered so that small targets take it.
    Also with seeds off (chunks only) and with a tiny seed-threshold cap."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 41, 9, gen=cases.long_hw_cases))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    for extra in ({}, {"EDLIB_B200_LONG_SEED_MAX_K": "0"}, {"EDLIB_B200_LONG_SEED_MAX_K": "70", "EDLIB_B200_FILTER_SEED_BUCKET": "1"}):
        env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_LONG_HW_MIN_TARGET="2000", **extra)
        out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) >= 27


def test_large_batch_uses_the_threaded_host_paths():
    """> 131072 pairs: packing + upload, classification, seed-stage outcomes and end-location assembly run
    on several host threads; every result still equals the reference's."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 3, 1, gen=lambda seed, count: [cases.big_batch_case(seed)]))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    env = dict(os.environ, EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_PACK_PARALLEL_KB="1024")
    out = subprocess.run(["python", "-c", code], env=env, check=True, capture_output=True, text=True)
    assert int(out.stdout.strip().splitlines()[-1]) == 140000


def test_sequences_longer_than_one_presence_item(emul):
    """Queries and targets above 65536 bytes are split into several presence-set work items
    (alphabetLength) and sweep as usual."""
    import random
    from helpers import mutate, rand_seq
    chk = parity.checker()
    rng = random.Random(9)
    q = rand_seq(rng, 70000, b"ACGTN")
    t = mutate(rng, q, 0.001, b"ACGT")
    assert emul.align(q, t, -1, 0, 0) == chk.align(q, t, -1, 0, 0)
    pairs = [(q, t), (b"ACGT" * 10, t), (q[:66000], b"AXY")]
    st, res = emul.align_batch([a for a, _ in pairs], [b for _, b in pairs], -1, 2, 0)
    assert st == 0
    for (a, b), r in zip(pairs, res):
        assert r == chk.align(a, b, -1, 2, 0)


def test_bad_input_in_a_large_batch_is_an_error_not_a_crash(emul):
    """A negative length is found by a worker thread of the host pool: the call returns EDLIB_STATUS_ERROR with
    every result marked, and the engine keeps working afterwards."""
    import ctypes as C
    from edlib_b200._ffi import AlignResult, make_config
    n = 140000
    q = C.create_string_buffer(b"ACGTACGTAC", 10)
    t = C.create_string_buffer(b"ACGTTCGTACGGA", 13)
    qptr = (C.c_char_p * n)(*[C.cast(q, C.c_char_p)] * n)
    tptr = (C.c_char_p * n)(*[C.cast(t, C.c_char_p)] * n)
    qlen = (C.c_int * n)(*[10] * n)
    tlen = (C.c_int * n)(*[13] * n)
    qlen[n - 7] = -3
    cfg, keep = make_config(-1, 2, 0, None)
    res = (AlignResult * n)()
    assert emul.lib.edlibAlignBatch(qptr, qlen, tptr, tlen, n, cfg, res) == 1
    assert res[0].status == 1 and res[n - 1].status == 1
    qlen[n - 7] = 10
    assert emul.lib.edlibAlignBatch(qptr, qlen, tptr, tlen, n, cfg, res) == 0
    exp = emul.align(b"ACGTACGTAC", b"ACGTTCGTACGGA", -1, 2, 0)
    assert res[5].editDistance == exp["editDistance"] and res[n - 7].editDistance == exp["editDistance"]
    for i in range(n):
        emul.free(res[i])
    del keep


def test_staged_batches_are_independent(emul):
    """edlibB200BatchPrepare / Compute / Results: two batches alive at once, computed out of order and twice;
    each yields what the one-shot call yields."""
    import ctypes as C
    import random
    from edlib_b200._ffi import AlignConfig, AlignResult, make_config, result_to_dict
    from helpers import mutate, rand_seq
    L = emul.lib
    L.edlibB200BatchPrepare.restype = C.c_void_p
    L.edlibB200BatchPrepare.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                                        C.c_int, AlignConfig]
    L.edlibB200BatchCompute.argtypes = [C.c_void_p, C.c_void_p]
    L.edlibB200BatchResults.argtypes = [C.c_void_p, C.POINTER(AlignResult)]
    L.edlibB200BatchFree.argtypes = [C.c_void_p]
    rng = random.Random(77)

    def make(nq, tlen, mode, task):
        t = rand_seq(rng, tlen, b"ACGT")
        qs = [mutate(rng, t[a:a + 60], 0.05, b"ACGT") for a in (rng.randrange(0, tlen - 60) for _ in range(nq))]
        n = len(qs)
        tb = C.create_string_buffer(t, len(t))
        arrs = ((C.c_char_p * n)(*qs), (C.c_int * n)(*[len(q) for q in qs]),
                (C.c_char_p * n)(*[C.cast(tb, C.c_char_p)] * n), (C.c_int * n)(*[len(t)] * n))
        cfg, keep = make_config(-1, mode, task, None)
        return dict(qs=qs, t=t, arrs=arrs, cfg=cfg, keep=(keep, tb), mode=mode, task=task, n=n)

    def results(b, handle):
        res = (AlignResult * b["n"])()
        assert L.edlibB200BatchResults(handle, res) == 0
        out = [result_to_dict(res[i]) for i in range(b["n"])]
        for i in range(b["n"]):
            emul.free(res[i])
        return out

    a, b = make(50, 900, 2, 1), make(70, 500, 0, 0)
    ha = L.edlibB200BatchPrepare(*a["arrs"], a["n"], a["cfg"])
    hb = L.edlibB200BatchPrepare(*b["arrs"], b["n"], b["cfg"])
    assert ha and hb
    assert L.edlibB200BatchCompute(hb, None) == 0
    assert L.edlibB200BatchCompute(ha, None) == 0
    assert L.edlibB200BatchCompute(hb, None) == 0
    for batch, h in ((a, ha), (b, hb)):
        st, exp = emul.align_batch(batch["qs"], [batch["t"]] * batch["n"], -1, batch["mode"], batch["task"])
        assert st == 0 and results(batch, h) == exp
    L.edlibB200BatchFree(ha)
    L.edlibB200BatchFree(hb)


def test_staged_api_misuse_is_an_error_not_a_crash(emul):
    """Results requested from a batch that was never computed (after another batch went through the engine, so that
    recycled storage is in play) return EDLIB_STATUS_ERROR; the batch still computes fine afterwards."""
    import ctypes as C
    from edlib_b200._ffi import AlignConfig, AlignResult, make_config, result_to_dict
    L = emul.lib
    L.edlibB200BatchPrepare.restype = C.c_void_p
    L.edlibB200BatchPrepare.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                                        C.c_int, AlignConfig]
    L.edlibB200BatchCompute.argtypes = [C.c_void_p, C.c_void_p]
    L.edlibB200BatchResults.argtypes = [C.c_void_p, C.POINTER(AlignResult)]
    L.edlibB200BatchFree.argtypes = [C.c_void_p]
    L.edlibB200LastError.restype = C.c_char_p
    st, _ = emul.align_batch([b"ACGTACGT"] * 5, [b"ACGTTTACGT"] * 5, -1, 2, 1)
    assert st == 0
    qs = [b"ACGTAC", b"TTTT", b"ACGGGT"] * 7
    n = len(qs)
    t = C.create_string_buffer(b"ACGTACGGGTTTACG", 15)
    arrs = ((C.c_char_p * n)(*qs), (C.c_int * n)(*[len(q) for q in qs]), (C.c_char_p * n)(*[C.cast(t, C.c_char_p)] * n),
            (C.c_int * n)(*[15] * n))
    cfg, keep = make_config(-1, 2, 1, None)
    h = L.edlibB200BatchPrepare(*arrs, n, cfg)
    assert h
    res = (AlignResult * n)()
    assert L.edlibB200BatchResults(h, res) == 1
    assert b"not" in L.edlibB200LastError()
    assert L.edlibB200BatchCompute(h, None) == 0
    assert L.edlibB200BatchResults(h, res) == 0
    got = [result_to_dict(res[i]) for i in range(n)]
    for i in range(n):
        emul.free(res[i])
    assert got == [emul.align(q, t.raw, -1, 2, 1) for q in qs]
    L.edlibB200BatchFree(h)
    del keep


def test_concurrent_small_calls_and_a_large_batch(emul):
    """Single calls from several threads go to the side engines (round robin, each behind its own lock) while a large
    batch runs on the main engine; every result still equals the reference's."""
    import random
    from concurrent.futures import ThreadPoolExecutor
    from helpers import mutate, rand_seq
    chk = parity.checker()
    rng = random.Random(6)
    t = rand_seq(rng, 2500, b"ACGT")
    qs = [mutate(rng, t[a:a + 100], 0.05, b"ACGT") for a in range(0, 2000, 50)]
    big_q = [mutate(rng, t[a % 2300:a % 2300 + 150], 0.03, b"ACGT") for a in range(0, 9000, 7)]
    with ThreadPoolExecutor(7) as ex:
        fb = ex.submit(lambda: emul.align_batch(big_q, [t] * len(big_q), -1, 2, 1))
        got = list(ex.map(lambda q: emul.align(q, t, -1, 2, 2), qs * 3))
        st, res = fb.result()
    assert st == 0 and res[::31] == [chk.align(q, t, -1, 2, 1) for q in big_q[::31]]
    assert got == [chk.align(q, t, -1, 2, 2) for q in qs] * 3


def test_many_end_locations(emul):
    """Repeats: every column is an end location (ref runTests-style 'A*64 vs B*70' shapes)."""
    chk = parity.checker()
    for q, t, mode in [(b"A" * 64, b"B" * 70, 2), (b"A" * 10, b"A" * 300, 2), (b"AC" * 20, b"AC" * 200, 2),
                       (b"A" * 33, b"A" * 100, 1), (b"A" * 5, b"C" * 9, 2)]:
        for task in (0, 1, 2):
            assert emul.align(q, t, -1, mode, task) == chk.align(q, t, -1, mode, task)
    qs = [b"A" * 10] * 40
    t = b"A" * 500
    st, res = emul.align_batch(qs, [t] * 40, -1, 2, 1)
    exp = chk.align(qs[0], t, -1, 2, 1)
    assert st == 0 and all(r == exp for r in res)


def test_very_large_bounds_and_full_byte_alphabets(emul):
    """k far above any possible distance (single calls and batches), byte values 0..255, hundreds of equality pairs.  Up to
    INT_MAX - 64 the reference's band arithmetic stays inside an int (edlib.cpp:563, 610, 634: k + 1, k + WORD_SIZE) and
    every field must agree with it; above that its result is undefined, and "at most k" must give what k = -1 gives."""
    import random
    chk = parity.checker()
    rng = random.Random(77)

    def rs(n, alphabet=b"ACGT"):
        return bytes(rng.choice(alphabet) for _ in range(n))

    int_max = 2**31 - 1
    pairs = [(rs(10), rs(30)), (rs(150), rs(3000)), (rs(300), rs(300)), (rs(700), rs(900)), (rs(70), b""), (b"", rs(20)), (rs(33), rs(31))]
    for q, t in pairs:
        for mode in (0, 1, 2):
            for task in (0, 1, 2):
                for k in (int_max - 64, 2**30 + 5, 2**24, 65536):
                    assert emul.align(q, t, k, mode, task) == chk.align(q, t, k, mode, task), (len(q), len(t), k, mode, task)
                free = emul.align(q, t, -1, mode, task)
                for k in (int_max, int_max - 1, int_max - 63):
                    assert emul.align(q, t, k, mode, task) == free, (len(q), len(t), k, mode, task)
    t = rs(3000)
    qs = [rs(rng.randrange(1, 300)) for _ in range(150)]
    for mode in (0, 1, 2):
        for task in (0, 1, 2):
            st, res = emul.align_batch(qs, [t] * len(qs), int_max - 64, mode, task)
            assert st == 0 and res == [chk.align(q, t, int_max - 64, mode, task) for q in qs]
            st, top = emul.align_batch(qs, [t] * len(qs), int_max, mode, task)
            assert st == 0 and top == res
    full = bytes(range(256))
    for mode in (0, 1, 2):
        for task in (0, 1, 2):
            q = bytes(rng.randrange(256) for _ in range(400))
            t = bytes(rng.randrange(256) for _ in range(900))
            eqs = [(bytes([rng.randrange(256)]), bytes([rng.randrange(256)])) for _ in range(300)]
            for args in ((q, t, -1, mode, task), (full, full[::-1], -1, mode, task), (q, t, -1, mode, task, eqs), (q, t, 5, mode, task, eqs)):
                assert emul.align(*args) == chk.align(*args), (mode, task, len(args))


def test_lengths_on_word_boundaries_in_mixed_batches():
    """Query and target lengths on the 32/64-bit word boundaries, alphabets of 1..256 symbols, every mode, task and bound, in
    batches over one shared or many targets: with the default thresholds and with the filter / streamed paths forced on."""
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "import parity, cases, test_engine_emul as T\n"
        "lib = T.load_emul()\n"
        "print(parity.run_batches(lib, 7, 60, gen=cases.boundary_mix_cases))\n"
    ) % (REPO, os.path.join(REPO, "tests"))
    forced = dict(EDLIB_B200_FILTER_MIN_TARGET="128", EDLIB_B200_FILTER_MIN_LEVEL_READS="0", EDLIB_B200_K1_MIN_GROUP="4",
                  EDLIB_B200_STREAM_MIN_PAIRS="64", EDLIB_B200_LONG_HW_MIN_TARGET="2000")
    for extra in ({}, forced):
        out = subprocess.run(["python", "-c", code], env=dict(os.environ, **extra), check=True, capture_output=True, text=True)
        assert int(out.stdout.strip().splitlines()[-1]) > 3000


def test_batch_helpers_for_results_and_cigar_strings(emul):
    """edlibB200AlignmentsToCigar / edlibB200FreeCigars / edlibB200FreeResults over the raw result structs of one
    edlibAlignBatch (HW, PATH): every CIGAR string (both formats) equals the reference's edlibAlignmentToCigar of the
    reference's own alignment; results without an alignment (bound exceeded) give NULL strings."""
    import ctypes as C
    import numpy as np
    import bench
    from edlib_b200 import workloads
    from edlib_b200._ffi import AlignResult, make_config
    L = emul.lib
    target, reads = workloads.reads_vs_target(num_reads=600, read_len=150, target_len=20_000, seed=5)
    reads = reads.copy()
    reads[::50] = workloads.random_dna(150, 3)  # unrelated reads: beyond the bound, no alignment
    qptr, qlen, tptr, tlen = bench.pointer_arrays(reads, target)
    cfg, _ = make_config(30, 2, 2)
    res = np.zeros(len(reads), dtype=bench.RESULT_DTYPE)
    assert L.edlibAlignBatch(bench.as_pp(qptr), bench.as_pi(qlen), bench.as_pp(tptr), bench.as_pi(tlen), len(reads), cfg,
                             C.cast(res.ctypes.data, C.POINTER(AlignResult))) == 0
    chk = parity.checker()
    t = target.tobytes()
    exp = [chk.align(reads[i].tobytes(), t, 30, 2, 2) for i in range(len(reads))]
    assert [bench.gpu_result_dict(res, i) for i in range(len(reads))] == exp
    assert sum(e["editDistance"] < 0 for e in exp) >= 10
    L.edlibB200AlignmentsToCigar.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.edlibB200FreeCigars.argtypes = [C.c_void_p, C.c_int]
    L.edlibB200FreeResults.argtypes = [C.c_void_p, C.c_int]
    for fmt in (0, 1):
        cg = (C.c_void_p * len(reads))()
        assert L.edlibB200AlignmentsToCigar(res.ctypes.data, len(reads), fmt, cg) == 0
        for i, e in enumerate(exp):
            if e["alignment"] is None:
                assert not cg[i]
            else:
                assert C.string_at(cg[i]).decode() == chk.cigar(e["alignment"], fmt), (i, fmt)
        L.edlibB200FreeCigars(cg, len(reads))
        assert not any(cg)  # pointers are cleared
    L.edlibB200FreeResults(res.ctypes.data, len(reads))
    assert not res["endLocations"].any() and not res["alignment"].any()
