"""ctypes view of the edlib C ABI (include/edlib.h).

`EdlibLib` binds any shared object that exports the ABI under a symbol prefix; the package
itself only ever loads the product library edlib_b200/lib/libedlib_b200.so (prefix "edlib").
The test-suite re-uses the class to bind its checkers; that wiring lives in tests/, not here.
"""
import ctypes as C
import os

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EDLIB_STATUS_OK, EDLIB_STATUS_ERROR = 0, 1
EDLIB_MODE_NW, EDLIB_MODE_SHW, EDLIB_MODE_HW = 0, 1, 2
EDLIB_TASK_DISTANCE, EDLIB_TASK_LOC, EDLIB_TASK_PATH = 0, 1, 2
EDLIB_CIGAR_STANDARD, EDLIB_CIGAR_EXTENDED = 0, 1
MODES = {"NW": 0, "SHW": 1, "HW": 2}
TASKS = {"distance": 0, "locations": 1, "path": 2}


class EqualityPair(C.Structure):          # include/edlib.h EdlibEqualityPair (2 bytes)
    _fields_ = [("first", C.c_char), ("second", C.c_char)]


class AlignConfig(C.Structure):           # include/edlib.h EdlibAlignConfig (32 bytes)
    _fields_ = [("k", C.c_int), ("mode", C.c_int), ("task", C.c_int),
                ("additionalEqualities", C.POINTER(EqualityPair)),
                ("additionalEqualitiesLength", C.c_int)]


class AlignResult(C.Structure):           # include/edlib.h EdlibAlignResult (48 bytes)
    _fields_ = [("status", C.c_int), ("editDistance", C.c_int),
                ("endLocations", C.POINTER(C.c_int)), ("startLocations", C.POINTER(C.c_int)),
                ("numLocations", C.c_int), ("alignment", C.POINTER(C.c_ubyte)),
                ("alignmentLength", C.c_int), ("alphabetLength", C.c_int)]


class Hits(C.Structure):                  # include/edlib_b200.h EdlibB200Hits (48 bytes)
    _fields_ = [("numQueries", C.c_int), ("counts", C.POINTER(C.c_longlong)), ("offsets", C.POINTER(C.c_longlong)),
                ("columns", C.POINTER(C.c_int)), ("scores", C.POINTER(C.c_int)), ("strands", C.POINTER(C.c_ubyte))]


class HitAlignments(C.Structure):         # include/edlib_b200.h EdlibB200HitAlignments (72 bytes)
    _fields_ = [("hits", Hits), ("starts", C.POINTER(C.c_int)), ("alignmentOffsets", C.POINTER(C.c_longlong)),
                ("alignments", C.POINTER(C.c_ubyte))]


class RecordHits(C.Structure):            # include/edlib_b200.h EdlibB200RecordHits (80 bytes)
    _fields_ = [("aln", HitAlignments), ("records", C.POINTER(C.c_int))]


assert C.sizeof(EqualityPair) == 2 and C.sizeof(AlignConfig) == 32 and C.sizeof(AlignResult) == 48
assert C.sizeof(Hits) == 48 and C.sizeof(HitAlignments) == 72 and C.sizeof(RecordHits) == 80


def _hit_dicts(a, n, both, records):
    """Per query of an EdlibB200HitAlignments: {"count", "hits"} and, when present, "starts" / "alignments"; hits are
    (column, score[, strand]), prefixed by the record when `records` is given."""
    h = a.hits
    out = []
    for i in range(n):
        lo, hi = h.offsets[i], h.offsets[i + 1]
        cols = [list(h.columns[lo:hi]), list(h.scores[lo:hi])]
        if both:
            cols.append(list(h.strands[lo:hi]))
        if records is not None:
            cols.insert(0, list(records[lo:hi]))
        r = {"count": h.counts[i], "hits": list(zip(*cols))}
        if a.starts:
            r["starts"] = a.starts[lo:hi]
        if a.alignments:
            off, base = a.alignmentOffsets, C.cast(a.alignments, C.c_void_p).value
            r["alignments"] = [C.string_at(base + off[j], off[j + 1] - off[j]) for j in range(lo, hi)]
        out.append(r)
    return out


def make_config(k=-1, mode=EDLIB_MODE_NW, task=EDLIB_TASK_DISTANCE, equalities=None):
    """Returns (config, keepalive) -- keepalive owns the equality array."""
    cfg = AlignConfig()
    cfg.k, cfg.mode, cfg.task = int(k), int(mode), int(task)
    keep = None
    if equalities:
        keep = (EqualityPair * len(equalities))()
        for i, (a, b) in enumerate(equalities):
            keep[i].first = a if isinstance(a, bytes) else bytes([a])
            keep[i].second = b if isinstance(b, bytes) else bytes([b])
        cfg.additionalEqualities = C.cast(keep, C.POINTER(EqualityPair))
        cfg.additionalEqualitiesLength = len(equalities)
    else:
        cfg.additionalEqualities = None
        cfg.additionalEqualitiesLength = 0
    return cfg, keep


def result_to_dict(r):
    """Copies every field of an AlignResult into plain Python (None for NULL arrays)."""
    d = {"status": r.status, "editDistance": r.editDistance, "numLocations": r.numLocations,
         "alignmentLength": r.alignmentLength, "alphabetLength": r.alphabetLength}
    if r.status != EDLIB_STATUS_OK:
        return {"status": r.status}
    d["endLocations"] = [r.endLocations[i] for i in range(r.numLocations)] if r.endLocations else None
    d["startLocations"] = [r.startLocations[i] for i in range(r.numLocations)] if r.startLocations else None
    d["alignment"] = bytes(bytearray(r.alignment[i] for i in range(r.alignmentLength))) if r.alignment else None
    return d


class EdlibLib:
    """One loaded implementation of the edlib ABI; `prefix` is the exported symbol prefix."""

    def __init__(self, path, prefix="edlib", has_batch=False):
        self.path = path
        self.lib = C.CDLL(path)
        self._align = getattr(self.lib, prefix + "Align")
        self._align.restype = AlignResult
        self._align.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, AlignConfig]
        self._free = getattr(self.lib, prefix + "FreeAlignResult")
        self._free.restype = None
        self._free.argtypes = [AlignResult]
        self._cigar = getattr(self.lib, prefix + "AlignmentToCigar")
        self._cigar.restype = C.c_void_p
        self._cigar.argtypes = [C.POINTER(C.c_ubyte), C.c_int, C.c_int]
        self._libc = C.CDLL(None)
        self._libc.free.argtypes = [C.c_void_p]
        self._batch = None
        if has_batch:
            self._batch = self.lib.edlibAlignBatch
            self._batch.restype = C.c_int
            self._batch.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                                    C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                                    C.c_int, AlignConfig, C.POINTER(AlignResult)]

    def align_raw(self, q, t, cfg):
        return self._align(q, len(q), t, len(t), cfg)

    def free(self, r):
        self._free(r)

    def align(self, q, t, k=-1, mode=EDLIB_MODE_NW, task=EDLIB_TASK_DISTANCE, equalities=None):
        cfg, keep = make_config(k, mode, task, equalities)
        r = self.align_raw(q, t, cfg)
        d = result_to_dict(r)
        if r.status == EDLIB_STATUS_OK:
            self.free(r)
        del keep
        return d

    def cigar(self, alignment, fmt=EDLIB_CIGAR_EXTENDED):
        n = len(alignment)
        buf = (C.c_ubyte * max(n, 1))(*alignment)
        p = self._cigar(buf, n, fmt)
        if not p:
            return None
        s = C.string_at(p).decode("ascii")
        self._libc.free(p)
        return s

    def align_batch(self, queries, targets, k=-1, mode=EDLIB_MODE_NW, task=EDLIB_TASK_DISTANCE,
                    equalities=None):
        """queries/targets: lists of bytes (targets may repeat the SAME bytes object to share it).
        Returns (status, [dict])."""
        assert self._batch is not None
        return self._run_batch(self._batch, queries, targets, k, mode, task, equalities)

    def align_batch_strands(self, queries, targets, k=-1, mode=EDLIB_MODE_NW, task=EDLIB_TASK_DISTANCE,
                            equalities=None):
        """edlibB200AlignBatchStrands: each query and its reverse complement, the better strand reported.
        Returns (status, [dict], [strand]) with strand 0 (forward) or 1 (reverse complement)."""
        assert self._batch is not None
        fn = self.lib.edlibB200AlignBatchStrands
        fn.restype = C.c_int
        fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                       C.c_int, AlignConfig, C.POINTER(AlignResult), C.POINTER(C.c_ubyte)]
        strands = (C.c_ubyte * max(len(queries), 1))()
        st, out = self._run_batch(lambda *a: fn(*a, strands), queries, targets, k, mode, task, equalities)
        return st, out, [strands[i] for i in range(len(queries))]

    def find_hits(self, queries, target, k, both=False, max_hits=(1 << 62), equalities=None,
                  mode=EDLIB_MODE_HW, task=EDLIB_TASK_DISTANCE):
        """edlibB200FindHits over one shared target.  Returns (status, [{"count": int, "hits": [...]}]) with hits
        (column, score), or (column, score, strand) when both strands were searched; status != 0: (status, None)."""
        fn = self.lib.edlibB200FindHits
        fn.restype = C.c_int
        fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.c_char_p, C.c_int, AlignConfig, C.c_int,
                       C.c_longlong, C.POINTER(Hits)]
        self.lib.edlibB200FreeHits.restype = None
        self.lib.edlibB200FreeHits.argtypes = [C.POINTER(Hits)]
        n = len(queries)
        cfg, keep = make_config(k, mode, task, equalities)
        qptr = (C.c_char_p * max(n, 1))(*queries)
        qlen = (C.c_int * max(n, 1))(*[len(q) for q in queries])
        h = Hits()
        st = fn(qptr, qlen, n, target, len(target), cfg, 1 if both else 0, max_hits, C.byref(h))
        del keep
        if st != EDLIB_STATUS_OK:
            return st, None
        out = []
        for i in range(n):
            a, b = h.offsets[i], h.offsets[i + 1]
            cols, scores = h.columns[a:b], h.scores[a:b]
            hits = list(zip(cols, scores, h.strands[a:b])) if both else list(zip(cols, scores))
            out.append({"count": h.counts[i], "hits": hits})
        self.lib.edlibB200FreeHits(C.byref(h))
        return st, out

    def find_hit_alignments(self, queries, target, k, both=False, max_hits=(1 << 62), equalities=None,
                            task=EDLIB_TASK_DISTANCE, mode=EDLIB_MODE_HW):
        """edlibB200FindHitAlignments over one shared target.  Returns (status, [dict]) as find_hits; with task LOC /
        PATH each dict also has "starts" (one per stored hit), with PATH "alignments" (bytes of EDLIB_EDOP_* codes,
        one per stored hit); status != 0: (status, None)."""
        fn = self.lib.edlibB200FindHitAlignments
        fn.restype = C.c_int
        fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.c_char_p, C.c_int, AlignConfig, C.c_int,
                       C.c_longlong, C.POINTER(HitAlignments)]
        self.lib.edlibB200FreeHitAlignments.restype = None
        self.lib.edlibB200FreeHitAlignments.argtypes = [C.POINTER(HitAlignments)]
        n = len(queries)
        cfg, keep = make_config(k, mode, task, equalities)
        qptr = (C.c_char_p * max(n, 1))(*queries)
        qlen = (C.c_int * max(n, 1))(*[len(q) for q in queries])
        a = HitAlignments()
        st = fn(qptr, qlen, n, target, len(target), cfg, 1 if both else 0, max_hits, C.byref(a))
        del keep
        if st != EDLIB_STATUS_OK:
            return st, None
        out = _hit_dicts(a, n, both, None)
        self.lib.edlibB200FreeHitAlignments(C.byref(a))
        return st, out

    def find_pair_hits(self, queries, targets, k, both=False, max_hits=(1 << 62), equalities=None,
                       task=EDLIB_TASK_DISTANCE, mode=EDLIB_MODE_HW):
        """edlibB200FindPairHits: query i searched in targets[i] only (repeat the SAME bytes object to share a target).
        Returns (status, [dict]) as find_hit_alignments, one dict per pair; status != 0: (status, None)."""
        fn = self.lib.edlibB200FindPairHits
        fn.restype = C.c_int
        fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int,
                       AlignConfig, C.c_int, C.c_longlong, C.POINTER(HitAlignments)]
        self.lib.edlibB200FreeHitAlignments.restype = None
        self.lib.edlibB200FreeHitAlignments.argtypes = [C.POINTER(HitAlignments)]
        n = len(queries)
        cfg, keep = make_config(k, mode, task, equalities)
        qptr = (C.c_char_p * max(n, 1))(*queries)
        qlen = (C.c_int * max(n, 1))(*[len(q) for q in queries])
        bufs = {}  # one buffer per distinct object: identical objects share a pointer, hence a target
        for t in targets:
            if id(t) not in bufs:
                bufs[id(t)] = C.create_string_buffer(bytes(t), max(len(t), 1))
        tptr = (C.c_char_p * max(n, 1))(*[C.cast(bufs[id(t)], C.c_char_p) for t in targets])
        tlen = (C.c_int * max(n, 1))(*[len(t) for t in targets])
        a = HitAlignments()
        st = fn(qptr, qlen, tptr, tlen, n, cfg, 1 if both else 0, max_hits, C.byref(a))
        del keep, bufs
        if st != EDLIB_STATUS_OK:
            return st, None
        out = _hit_dicts(a, n, both, None)
        self.lib.edlibB200FreeHitAlignments(C.byref(a))
        return st, out

    def find_record_hits(self, queries, records, k, both=False, max_hits=(1 << 62), equalities=None,
                         task=EDLIB_TASK_DISTANCE, mode=EDLIB_MODE_HW):
        """edlibB200FindRecordHits over a list of records.  Returns (status, [dict]) as find_hit_alignments, with
        hits (record, column, score) or (record, column, score, strand); status != 0: (status, None)."""
        fn = self.lib.edlibB200FindRecordHits
        fn.restype = C.c_int
        fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                       C.c_int, AlignConfig, C.c_int, C.c_longlong, C.POINTER(RecordHits)]
        self.lib.edlibB200FreeRecordHits.restype = None
        self.lib.edlibB200FreeRecordHits.argtypes = [C.POINTER(RecordHits)]
        n, r = len(queries), len(records)
        cfg, keep = make_config(k, mode, task, equalities)
        qptr = (C.c_char_p * max(n, 1))(*queries)
        qlen = (C.c_int * max(n, 1))(*[len(q) for q in queries])
        rptr = (C.c_char_p * max(r, 1))(*records)
        rlen = (C.c_int * max(r, 1))(*[len(x) for x in records])
        a = RecordHits()
        st = fn(qptr, qlen, n, rptr, rlen, r, cfg, 1 if both else 0, max_hits, C.byref(a))
        del keep
        if st != EDLIB_STATUS_OK:
            return st, None
        out = _hit_dicts(a.aln, n, both, a.records)
        self.lib.edlibB200FreeRecordHits(C.byref(a))
        return st, out

    def align_records(self, queries, records, k=-1, task=EDLIB_TASK_DISTANCE, equalities=None, both=False,
                      mode=EDLIB_MODE_HW):
        """edlibB200AlignRecords: each query against a list of records, the result of its best record.  Returns
        (status, [dict], [record], [strand] or None) with the dicts of align_batch; status != 0: (status, None, None,
        None)."""
        fn = self.lib.edlibB200AlignRecords
        fn.restype = C.c_int
        fn.argtypes = [C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                       C.c_int, AlignConfig, C.c_int, C.POINTER(AlignResult), C.POINTER(C.c_int), C.POINTER(C.c_ubyte)]
        n, r = len(queries), len(records)
        cfg, keep = make_config(k, mode, task, equalities)
        qptr = (C.c_char_p * max(n, 1))(*queries)
        qlen = (C.c_int * max(n, 1))(*[len(q) for q in queries])
        rptr = (C.c_char_p * max(r, 1))(*records)
        rlen = (C.c_int * max(r, 1))(*[len(x) for x in records])
        res = (AlignResult * max(n, 1))()
        recs = (C.c_int * max(n, 1))()
        strands = (C.c_ubyte * max(n, 1))()
        st = fn(qptr, qlen, n, rptr, rlen, r, cfg, 1 if both else 0, res, recs, strands)
        del keep
        if st != EDLIB_STATUS_OK:
            return st, None, None, None
        out = []
        for i in range(n):
            out.append(result_to_dict(res[i]))
            self.free(res[i])
        return st, out, list(recs[:n]), (list(strands[:n]) if both else None)

    def _run_batch(self, call, queries, targets, k, mode, task, equalities):
        n = len(queries)
        cfg, keep = make_config(k, mode, task, equalities)
        qptr = (C.c_char_p * n)(*queries)
        qlen = (C.c_int * n)(*[len(q) for q in queries])
        # identical bytes objects must map to identical pointers: build one buffer per distinct object
        bufs = {}
        tptr_vals, tlen_vals = [], []
        for t in targets:
            key = id(t)
            if key not in bufs:
                bufs[key] = C.create_string_buffer(t, len(t)) if len(t) else C.create_string_buffer(1)
            tptr_vals.append(C.cast(bufs[key], C.c_char_p))
            tlen_vals.append(len(t))
        tptr = (C.c_char_p * n)(*tptr_vals)
        tlen = (C.c_int * n)(*tlen_vals)
        res = (AlignResult * n)()
        st = call(qptr, qlen, tptr, tlen, n, cfg, res)
        out = []
        for i in range(n):
            out.append(result_to_dict(res[i]))
            if res[i].status == EDLIB_STATUS_OK:
                self.free(res[i])
        del keep, bufs
        return st, out


def product_path():
    return os.path.join(REPO, "edlib_b200", "lib", "libedlib_b200.so")
