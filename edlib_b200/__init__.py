"""edlib_b200 -- H100-native batched edit-distance engine behind the edlib C ABI.

Python host mirror of the reference's binding (bindings/python/edlib.pyx): `align()` takes the same
arguments and returns the same dict (edlib.pyx:56-155), `getNiceAlignment()` is edlib.pyx:157-238,
`align_batch()` is the batched form over `edlibAlignBatch`.  All computation happens in the CUDA library
edlib_b200/lib/libedlib_b200.so; importing this package without it (or without a GPU) works, calling
`align*` then raises.
"""
import ctypes as _C
import re as _re

from ._ffi import (EDLIB_CIGAR_EXTENDED, EDLIB_CIGAR_STANDARD, EDLIB_STATUS_OK, MODES, TASKS, EdlibLib,
                   product_path)

__all__ = ["align", "align_batch", "align_many", "align_records", "find_hits", "find_pair_hits", "getNiceAlignment",
           "library"]

_lib = None


def library():
    """The loaded product library (raises OSError if it has not been built)."""
    global _lib
    if _lib is None:
        _lib = EdlibLib(product_path(), prefix="edlib", has_batch=True)
        _lib.lib.edlibB200LastError.restype = _C.c_char_p
    return _lib


def _is_plain(s):
    """bytes, or str whose UTF-8 form has one byte per character (edlib.pyx:11-19)."""
    return isinstance(s, (bytes, bytearray)) or (isinstance(s, str) and len(s.encode("utf-8")) == len(s))


def _plain_bytes(s):
    return bytes(s) if isinstance(s, (bytes, bytearray)) else s.encode("utf-8")


def _map_to_bytes(seqs, additional_equalities):
    """Sequences of hashables -> byte strings (edlib.pyx:22-53): ASCII str / bytes pass through,
    anything else is recoded over the joint alphabet (at most 256 distinct values)."""
    if all(_is_plain(s) for s in seqs):
        eqs = None
        if additional_equalities is not None:
            eqs = [(_plain_bytes(a)[:1], _plain_bytes(b)[:1]) for a, b in additional_equalities]
        return [_plain_bytes(s) for s in seqs], eqs
    alphabet = set()
    for s in seqs:
        alphabet.update(s)
    if len(alphabet) > 256:
        raise ValueError("query and target combined have more than 256 unique values, this is not supported.")
    code = {c: bytes([i]) for i, c in enumerate(alphabet)}
    eqs = None
    if additional_equalities is not None:
        eqs = [(code[a], code[b]) for a, b in additional_equalities if a in code and b in code]
    return [b"".join(code[c] for c in s) for s in seqs], eqs


def _result(d, want_cigar):
    if d["status"] != EDLIB_STATUS_OK:
        raise Exception("There was an error. (" + library().lib.edlibB200LastError().decode() + ")")
    locations = []
    if d["endLocations"] is not None:
        starts = d["startLocations"] or [None] * d["numLocations"]
        locations = list(zip(starts, d["endLocations"]))
    cigar = library().cigar(d["alignment"], EDLIB_CIGAR_EXTENDED) if (want_cigar and d["alignment"] is not None) else None
    return {"editDistance": d["editDistance"], "alphabetLength": d["alphabetLength"],
            "locations": locations, "cigar": cigar}


def align(query, target, mode="NW", task="distance", k=-1, additionalEqualities=None):
    """Same contract as the reference's `edlib.align` (edlib.pyx:56-155)."""
    (q, t), eqs = _map_to_bytes([query, target], additionalEqualities)
    d = library().align(q, t, -1 if k is None else k, MODES.get(mode, 0), TASKS.get(task, 0), eqs)
    return _result(d, True)


def align_batch(queries, targets, mode="NW", task="distance", k=-1, additionalEqualities=None, strands="forward"):
    """Batched `align`: `targets` is one sequence shared by all queries, or one per query (repeat the
    same object to share its upload).  Returns one dict per query.

    strands="both": every query is aligned as given and as its reverse complement (DNA reads from either strand,
    IUPAC codes complemented, case kept); each dict is the better strand's result (ties: the forward one) and gains
    "strand": "+" or "-".  Sequences must then be bytes or ASCII str: recoding them would destroy the complement."""
    if strands not in ("forward", "both"):
        raise ValueError("strands must be 'forward' or 'both'")
    queries = list(queries)
    shared = isinstance(targets, (bytes, bytearray, str))
    tlist = [targets] if shared else list(targets)
    distinct, index = [], {}
    for t in tlist:
        if id(t) not in index:
            index[id(t)] = len(distinct)
            distinct.append(t)
    if strands == "both" and not all(_is_plain(s) for s in queries + distinct):
        raise ValueError("strands='both' needs bytes or ASCII str sequences")
    mapped, eqs = _map_to_bytes(queries + distinct, additionalEqualities)
    qs, ts = mapped[:len(queries)], mapped[len(queries):]
    per_query = [ts[0]] * len(qs) if shared else [ts[index[id(t)]] for t in tlist]
    args = (qs, per_query, -1 if k is None else k, MODES.get(mode, 0), TASKS.get(task, 0), eqs)
    if strands == "both":
        st, res, chosen = library().align_batch_strands(*args)
    else:
        (st, res), chosen = library().align_batch(*args), None
    if st != EDLIB_STATUS_OK:
        raise Exception("There was an error. (" + library().lib.edlibB200LastError().decode() + ")")
    out = [_result(d, True) for d in res]
    if chosen is not None:
        for r, s in zip(out, chosen):
            r["strand"] = "-" if s else "+"
    return out


align_many = align_batch  # the name SURVEY.md 8f proposes for the batched binding entry


def align_records(queries, records, task="distance", k=-1, additionalEqualities=None, strands="forward"):
    """Each query aligned (HW mode) against a reference of several records (chromosomes, plasmids, contigs) in one
    call, with the result of its best record: the lowest-index record among those of least edit distance (record 0
    when none is within k).  Returns one dict per query, that of `align_batch(query, records[r], mode="HW", ...)` for
    that record r, plus "record": r.  Locations count from the start of the record, and "alphabetLength" covers the
    query and that record only.

    strands="both": the query and its reverse complement each get their best record; the reverse one is reported only
    when strictly better, and the dict gains "strand" as for `align_batch`.  The sequence rules are those of
    `align_batch`."""
    if strands not in ("forward", "both"):
        raise ValueError("strands must be 'forward' or 'both'")
    if task not in TASKS:
        raise ValueError("task must be 'distance', 'locations' or 'path'")
    queries, records = list(queries), list(records)
    if strands == "both" and not all(_is_plain(s) for s in queries + records):
        raise ValueError("strands='both' needs bytes or ASCII str sequences")
    mapped, eqs = _map_to_bytes(queries + records, additionalEqualities)
    both = strands == "both"
    lib = library()
    st, res, chosen, strand = lib.align_records(mapped[:len(queries)], mapped[len(queries):], -1 if k is None else k,
                                                TASKS[task], eqs, both)
    if st != EDLIB_STATUS_OK:
        raise Exception("There was an error. (" + lib.lib.edlibB200LastError().decode() + ")")
    out = [_result(d, True) for d in res]
    for i, r in enumerate(out):
        r["record"] = chosen[i]
        if both:
            r["strand"] = "-" if strand[i] else "+"
    return out


def find_hits(queries, target, k, strands="forward", max_hits=None, additionalEqualities=None, task="distance"):
    """Every place where each query occurs in `target` with at most k edits (HW mode; queries of 1..256 symbols).

    Returns one dict per query: {"count": number of hits, "hits": [(column, score), ...]}, where the hits are every
    end column c of `target` whose best alignment of the query ending there has score <= k, in ascending columns.
    At most `max_hits` hits are listed per query (None: all); "count" is always the full number.
    strands="both": the reverse complement is searched too; its hits follow the forward ones and every hit becomes
    (column, score, "+" or "-").  The sequence rules are those of `align_batch`.

    task="locations" adds "starts", one per listed hit: the first target column of the hit's alignment (the smallest
    start whose alignment to [start, column] still has the hit's score).  task="path" adds "cigars" as well: the
    extended CIGAR of that alignment, as `align(..., task="path")` gives it; a "-" hit's CIGAR aligns the reverse
    complement.  For the columns of a query's least score these are exactly `align(query, target, "HW", task, k)`'s
    locations, and its CIGAR is the one of the first of them.

    `target` given as a non-empty list or tuple of sequences (str, bytes, or lists / tuples of symbols; so a list of
    single characters counts as records of one symbol) searches them as the records of one reference (chromosomes,
    contigs) in one call.  The hits of a query on record r are exactly those of find_hits(query, target[r]): every hit
    becomes (record, column, score) or (record, column, score, "+"/"-"), its column and "starts" count from the start
    of its record, no hit spans two records, and hits are ordered by strand, then record, then column."""
    if strands not in ("forward", "both"):
        raise ValueError("strands must be 'forward' or 'both'")
    if task not in ("distance", "locations", "path"):
        raise ValueError("task must be 'distance', 'locations' or 'path'")
    queries = list(queries)
    is_seq = lambda s: isinstance(s, (str, bytes, bytearray, list, tuple))  # noqa: E731
    records = list(target) if isinstance(target, (list, tuple)) and target and all(map(is_seq, target)) else None
    targets = records if records is not None else [target]
    if strands == "both" and not all(_is_plain(s) for s in queries + targets):
        raise ValueError("strands='both' needs bytes or ASCII str sequences")
    mapped, eqs = _map_to_bytes(queries + targets, additionalEqualities)
    queries, targets = mapped[:len(queries)], mapped[len(queries):]
    both = strands == "both"
    cap = (1 << 62) if max_hits is None else max_hits
    lib = library()
    if records is not None:
        st, res = lib.find_record_hits(queries, targets, k, both, cap, eqs, TASKS[task])
    elif task == "distance":
        st, res = lib.find_hits(queries, targets[0], k, both, cap, eqs)
    else:
        st, res = lib.find_hit_alignments(queries, targets[0], k, both, cap, eqs, TASKS[task])
    if st != EDLIB_STATUS_OK:
        raise Exception("There was an error. (" + lib.lib.edlibB200LastError().decode() + ")")
    for r in res:
        if both:
            r["hits"] = [h[:-1] + ("-" if h[-1] else "+",) for h in r["hits"]]
        if "alignments" in r:
            r["cigars"] = [lib.cigar(a, EDLIB_CIGAR_EXTENDED) for a in r.pop("alignments")]
    return res


def find_pair_hits(queries, targets, k, strands="forward", max_hits=None, additionalEqualities=None, task="distance"):
    """Every place where queries[i] occurs in its own targets[i] with at most k edits, for every pair i in one call
    (HW mode; queries of 1..256 symbols): a read's candidate region, its amplicon, the locus a guide is assigned to.

    Returns one dict per pair, that of `find_hits([queries[i]], targets[i], ...)` for its one query: {"count", "hits":
    [(column, score[, "+"/"-"]), ...]} and, for task "locations" / "path", "starts" / "cigars"; columns and starts count
    from the start of targets[i].  An empty target has no hits.  The sequence rules and target sharing are those of
    `align_batch`: repeating the same object shares its upload, and many pairs over one target are searched together."""
    if strands not in ("forward", "both"):
        raise ValueError("strands must be 'forward' or 'both'")
    if task not in ("distance", "locations", "path"):
        raise ValueError("task must be 'distance', 'locations' or 'path'")
    queries, tlist = list(queries), list(targets)
    if len(queries) != len(tlist):
        raise ValueError("queries and targets must have the same length")
    distinct, index = [], {}
    for t in tlist:
        if id(t) not in index:
            index[id(t)] = len(distinct)
            distinct.append(t)
    if strands == "both" and not all(_is_plain(s) for s in queries + distinct):
        raise ValueError("strands='both' needs bytes or ASCII str sequences")
    mapped, eqs = _map_to_bytes(queries + distinct, additionalEqualities)
    qs, ts = mapped[:len(queries)], mapped[len(queries):]
    both = strands == "both"
    cap = (1 << 62) if max_hits is None else max_hits
    lib = library()
    st, res = lib.find_pair_hits(qs, [ts[index[id(t)]] for t in tlist], k, both, cap, eqs, TASKS[task])
    if st != EDLIB_STATUS_OK:
        raise Exception("There was an error. (" + lib.lib.edlibB200LastError().decode() + ")")
    for r in res:
        if both:
            r["hits"] = [h[:-1] + ("-" if h[-1] else "+",) for h in r["hits"]]
        if "alignments" in r:
            r["cigars"] = [lib.cigar(a, EDLIB_CIGAR_EXTENDED) for a in r.pop("alignments")]
    return res


def getNiceAlignment(alignResult, query, target, gapSymbol="-"):
    """Human-readable three-line view of an `align(..., task='path')` result (edlib.pyx:157-238):
    dict with 'query_aligned', 'matched_aligned' ('|' match, '.' mismatch, gap symbol for indels) and
    'target_aligned'."""
    if not isinstance(alignResult, dict):
        raise Exception("The object alignResult is expected to be a python dictionary. Please check the input alignResult.")
    if "locations" not in alignResult:
        raise Exception("The object alignResult is expected to contain a field 'locations'. Please check the input alignResult.")
    if "cigar" not in alignResult:
        raise Exception("The object alignResult is expected to contain a CIGAR string. Please check the input alignResult.")
    cigar = alignResult["cigar"]
    if not cigar:
        raise Exception("The object alignResult contains an empty CIGAR string. Users must run align() with task='path'. "
                        "Please check the input alignResult.")
    tpos = alignResult["locations"][0][0] or 0
    qpos = 0
    t_aln, m_aln, q_aln = [], [], []
    for count, op in _re.findall(r"(\d+)(\D)", cigar):
        n = int(count)
        if op in "=X":
            t_aln.append(target[tpos:tpos + n])
            q_aln.append(query[qpos:qpos + n])
            m_aln.append(("|" if op == "=" else ".") * n)
            tpos += n
            qpos += n
        elif op == "D":
            t_aln.append(target[tpos:tpos + n])
            q_aln.append(gapSymbol * n)
            m_aln.append(gapSymbol * n)
            tpos += n
        elif op == "I":
            t_aln.append(gapSymbol * n)
            q_aln.append(query[qpos:qpos + n])
            m_aln.append(gapSymbol * n)
            qpos += n
        else:
            raise Exception("The CIGAR string from alignResult contains a symbol not '=', 'X', 'D', 'I'. "
                            "Please check the validity of alignResult and alignResult.cigar")
    return {"query_aligned": "".join(q_aln), "matched_aligned": "".join(m_aln), "target_aligned": "".join(t_aln)}
