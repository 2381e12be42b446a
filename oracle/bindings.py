"""ctypes bindings for the checkers under oracle/ — TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this.
  ref_*    -> oracle/_ref/libracon_ref.so   (unmodified reference sources, built by oracle/Makefile)
  oracle_* -> oracle/_build/libpoa_oracle.so (the restated CPU oracle, oracle/poa_oracle.cpp)
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(HERE, "_ref", "libracon_ref.so")
ORACLE_SO = os.path.join(HERE, "_build", "libpoa_oracle.so")

_ref = None
_oracle = None

_CONS_ARGS = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
              C.c_void_p, C.c_void_p, C.c_int8, C.c_int8, C.c_int8, C.c_uint32, C.c_int, C.c_uint32,
              C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]


def have_ref():
    return os.path.exists(REF_SO)


def ref_lib():
    global _ref
    if _ref is None:
        lib = C.CDLL(REF_SO)
        lib.ref_poa_consensus.restype = C.c_double
        lib.ref_poa_consensus.argtypes = _CONS_ARGS
        lib.ref_edlib_cigar.restype = C.c_int64
        lib.ref_edlib_cigar.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_void_p,
                                        C.c_uint64, C.c_void_p]
        _ref = lib
    return _ref


def oracle_lib():
    global _oracle
    if _oracle is None:
        srcs = [os.path.join(HERE, f) for f in ("poa_oracle.cpp", "myers_oracle.cpp", "bp_oracle.cpp")]
        stale = not os.path.exists(ORACLE_SO) or any(
            os.path.exists(f) and os.path.getmtime(f) > os.path.getmtime(ORACLE_SO) for f in srcs)
        if stale:
            import subprocess
            subprocess.check_call(["make", "-C", HERE, "oracle"], stdout=subprocess.DEVNULL)
        lib = C.CDLL(ORACLE_SO)
        lib.oracle_poa_consensus.restype = C.c_double
        lib.oracle_poa_consensus.argtypes = _CONS_ARGS + [C.c_void_p]
        lib.oracle_poa_stats.restype = None
        lib.oracle_poa_stats.argtypes = [C.c_void_p]
        if hasattr(lib, "oracle_myers_cigar"):
            lib.oracle_myers_cigar.restype = C.c_int64
            lib.oracle_myers_cigar.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_void_p,
                                               C.c_uint64, C.c_void_p, C.c_uint64]
            lib.oracle_myers_tree.restype = C.c_int64
            lib.oracle_myers_tree.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint64, C.c_void_p,
                                              C.c_uint64]
        lib.oracle_graph_shape.restype = C.c_int
        lib.oracle_graph_shape.argtypes = _CONS_ARGS[:13] + [C.c_uint32, C.c_void_p, C.c_uint32] + [C.c_void_p, C.c_uint32] + \
            [C.c_void_p] * 3
        lib.oracle_poa_set_tie_rules.restype = None
        lib.oracle_poa_set_tie_rules.argtypes = [C.c_uint32]
        lib.oracle_poa_trace_begin.restype = None
        lib.oracle_poa_trace_begin.argtypes = []
        lib.oracle_poa_trace_end.restype = C.c_uint64
        lib.oracle_poa_trace_end.argtypes = [C.c_void_p, C.c_uint64]
        if hasattr(lib, "oracle_breaking_points"):
            lib.oracle_breaking_points.restype = C.c_int64
            lib.oracle_breaking_points.argtypes = [C.c_char_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32,
                                                   C.c_uint32, C.c_void_p, C.c_uint64]
        _oracle = lib
    return _oracle


def _ptr(a):
    return None if a is None else a.ctypes.data


def _max_nodes_bound(ws):
    # consensus length <= number of graph nodes <= total bases of the window
    lens = np.diff(ws.seq_off.astype(np.int64))
    per_win = np.add.reduceat(lens, ws.win_first[:-1].astype(np.int64)) if ws.n_windows else np.zeros(0)
    return int(per_win.max()) if len(per_win) else 1


def _run(fn, ws, m, x, g, window_length, trim, threads, extra=()):
    n = ws.n_windows
    stride = max(16, _max_nodes_bound(ws))
    out = np.zeros((n, stride), dtype=np.uint8)
    out_len = np.zeros(n, dtype=np.uint32)
    polished = np.zeros(n, dtype=np.uint8)
    secs = fn(n, _ptr(ws.bases), _ptr(ws.quals), _ptr(ws.seq_off), _ptr(ws.seq_has_qual),
              _ptr(ws.seq_begin), _ptr(ws.seq_end), _ptr(ws.win_first), _ptr(ws.win_type),
              m, x, g, window_length, 1 if trim else 0, threads, out.ctypes.data, stride,
              out_len.ctypes.data, polished.ctypes.data, *extra)
    if secs < 0:
        raise RuntimeError("checker failed (code %r)" % secs)
    cons = [out[w, :out_len[w]].tobytes() for w in range(n)]
    return cons, polished.astype(bool), secs


def ref_consensus(ws, m=3, x=-5, g=-4, window_length=500, trim=True, threads=1):
    """The reference itself: Window::generate_consensus over every window."""
    return _run(ref_lib().ref_poa_consensus, ws, m, x, g, window_length, trim, threads)


def oracle_consensus(ws, m=3, x=-5, g=-4, window_length=500, trim=True, threads=1, want_coverage=False):
    """The restated oracle.  With want_coverage also returns per-window uint32 coverage (untrimmed
    consensus coordinates are not exposed; coverage is for the returned, trimmed consensus)."""
    n = ws.n_windows
    stride = max(16, _max_nodes_bound(ws))
    cov = np.zeros((n, stride), dtype=np.uint32)
    cons, pol, secs = _run(oracle_lib().oracle_poa_consensus, ws, m, x, g, window_length, trim, threads,
                           extra=(cov.ctypes.data,))
    if want_coverage:
        return cons, pol, secs, [cov[w, :len(cons[w])].copy() for w in range(n)]
    return cons, pol, secs


# spoa's tie rules, one bit each: oracle_poa_set_tie_rules(bit) replaces that rule by its opposite
TIE_RULES = {
    "first_in_edge_diagonal": 1 << 0,   # traceback, diagonal step: predecessors in in-edge order, the first match wins
    "vertical_before_horizontal": 1 << 1,
    "first_tied_sink": 1 << 2,          # equal best scores in the last column: the first sink in rank order wins
    "bundle_tie_le": 1 << 3,            # heaviest bundle, equal edge weights: scores[pred] <= scores[tail] takes the tail
    "first_best_node": 1 << 4,          # heaviest bundle: the strict maximum keeps the first best node in rank order
}


def oracle_poa_set_tie_rules(mask):
    """TESTS ONLY: every later oracle call breaks ties with the opposite of each rule set in `mask` (TIE_RULES); 0, the
    default, is spoa.  It exists to show that a test's windows reach a rule, never to check a result."""
    oracle_lib().oracle_poa_set_tie_rules(mask)


def oracle_consensus_with_tie_rules(ws, mask, *args, **kw):
    """oracle_consensus with the tie rules of `mask` flipped, then spoa's rules again"""
    oracle_poa_set_tie_rules(mask)
    try:
        return oracle_consensus(ws, *args, **kw)
    finally:
        oracle_poa_set_tie_rules(0)


def oracle_matrix_ranges(ws, m=3, x=-5, g=-4, window_length=500, trim=True):
    """Per window, an (alignments, 5) int64 array: read length, graph rows, lowest column-0 value, lowest and highest
    cell of each of the window's int32 score matrices, in the order the oracle aligned its layers."""
    lib = oracle_lib()
    out = []
    for w in range(ws.n_windows):
        sub = ws.subset([w])
        lib.oracle_poa_trace_begin()
        try:
            _run(lib.oracle_poa_consensus, sub, m, x, g, window_length, trim, 1, extra=(None,))
        finally:
            cap = int(ws.win_first[w + 1] - ws.win_first[w])
            rec = np.zeros((cap, 5), np.int64)
            n = lib.oracle_poa_trace_end(rec.ctypes.data, cap)
        out.append(rec[:min(n, cap)])
    return out


def oracle_graph_shape(ws, m=3, x=-5, g=-4, window_length=500, threads=1):
    """Per window, (nodes, max in-degree, max aligned-set size) of the oracle's graph: nodes = uint32 array of the node
    count after the backbone and after each aligned layer, in the order the oracle aligned its layers (sorted by begin;
    empty for windows of fewer than 3 sequences); the two maxima are those of the final graph."""
    n = ws.n_windows
    stride = max(16, _max_nodes_bound(ws))
    out = np.zeros((n, stride), dtype=np.uint8)
    per_win = np.diff(ws.win_first.astype(np.int64))
    nstride = max(1, int(per_win.max()) if n else 1)
    nodes = np.zeros((n, nstride), np.uint32)
    n_nodes, indeg, aligned = (np.zeros(n, np.uint32) for _ in range(3))
    r = oracle_lib().oracle_graph_shape(n, _ptr(ws.bases), _ptr(ws.quals), _ptr(ws.seq_off), _ptr(ws.seq_has_qual),
                                        _ptr(ws.seq_begin), _ptr(ws.seq_end), _ptr(ws.win_first), _ptr(ws.win_type),
                                        m, x, g, window_length, threads, out.ctypes.data, stride, nodes.ctypes.data,
                                        nstride, n_nodes.ctypes.data, indeg.ctypes.data, aligned.ctypes.data)
    if r != 0:
        raise RuntimeError("oracle graph shape failed (%d)" % r)
    return [(nodes[w, :n_nodes[w]].copy(), int(indeg[w]), int(aligned[w])) for w in range(n)]


def ref_edlib_cigar(q, t):
    cap = 4 * (len(q) + len(t)) + 64
    buf = C.create_string_buffer(cap)
    ed = C.c_int32(0)
    n = ref_lib().ref_edlib_cigar(q, len(q), t, len(t), buf, cap, C.byref(ed))
    if n < 0:
        raise RuntimeError("edlib failed (%d)" % n)
    return buf.raw[:n].decode(), ed.value


EDLIB_RULE = 1 << 20   # edlib traces a node back below this many bytes of alignment data, and splits it above


def edlib_data_bytes(ql, tl):
    """The alignment data edlib's rule weighs for a (ql x tl) node (edlib.cpp:1155-1157)."""
    return 20 * ((ql + 63) // 64) * tl + 8 * tl


def oracle_myers_cigar(q, t, rule=EDLIB_RULE):
    """(CIGAR, edit distance) edlib returns, restated; with another `rule` (bytes), what it would return if its 1 MiB
    rule were moved there."""
    cap = 4 * (len(q) + len(t)) + 64
    buf = C.create_string_buffer(cap)
    ed = C.c_int32(0)
    n = oracle_lib().oracle_myers_cigar(q, len(q), t, len(t), buf, cap, C.byref(ed), rule)
    if n < 0:
        raise RuntimeError("oracle myers failed (%d)" % n)
    return buf.raw[:n].decode(), ed.value


def oracle_myers_tree(q, t, rule=EDLIB_RULE):
    """edlib's node tree for the pair: an (nodes, 4) int64 array of (query length, target length, score, leaf) in
    pre-order, leaf = 1 for a traceback node and 0 for a Hirschberg split; nodes with an empty side are left out."""
    cap = 2 * (len(q) + len(t)) + 8
    out = np.zeros((cap, 4), np.int32)
    n = oracle_lib().oracle_myers_tree(q, len(q), t, len(t), rule, out.ctypes.data, cap)
    if n < 0:
        raise RuntimeError("oracle myers tree failed (%d)" % n)
    return out[:n].astype(np.int64)


def oracle_breaking_points(cigar, t_begin, t_end, q_start, window_length):
    """(n, 2) uint32 array of (t, q) breaking points, two rows per window with a match (overlap.cpp:226-292)."""
    if isinstance(cigar, str):
        cigar = cigar.encode()
    cap = 2 * ((t_end - t_begin) // max(1, window_length) + 3)
    out = np.zeros((cap, 2), np.uint32)
    n = oracle_lib().oracle_breaking_points(cigar, len(cigar), t_begin, t_end, q_start, window_length,
                                            out.ctypes.data, cap)
    if n < 0:
        raise RuntimeError("oracle breaking points failed (%d)" % n)
    return out[:n].copy()


CUDAPOA_SO = os.path.join(HERE, "_ref", "libref_cudapoa.so")


def have_ref_cudapoa():
    return os.path.exists(CUDAPOA_SO)


def ref_cudapoa_consensus(ws, match=3, mismatch=-5, gap=-4, banded=False, max_depth=200, device=0, mem_fraction=0.5):
    """The reference's own GPU path (GenomeWorks cudapoa, unmodified; oracle/ref_cudapoa_harness.cu) on a window set.
    Returns (list of consensus bytes — b"" where cudapoa rejected the window —, n_ok, wall seconds, GPU-call seconds).
    Timing only: cudapoa's consensus is not spoa's."""
    lib = C.CDLL(CUDAPOA_SO)
    lib.ref_cudapoa_consensus.restype = C.c_int64
    lib.ref_cudapoa_consensus.argtypes = [C.c_uint32] + [C.c_void_p] * 6 + [C.c_int8, C.c_int8, C.c_int8, C.c_int,
                                                                            C.c_uint32, C.c_int, C.c_double, C.c_void_p,
                                                                            C.c_uint32, C.c_void_p, C.c_void_p]
    n = ws.n_windows
    stride = 2048
    out = np.zeros((n, stride), np.uint8)
    out_len = np.zeros(n, np.uint32)
    times = np.zeros(2, np.float64)
    seq_off = np.ascontiguousarray(ws.seq_off, dtype=np.uint64)
    ok = lib.ref_cudapoa_consensus(n, _ptr(ws.bases), _ptr(ws.quals), _ptr(seq_off), _ptr(ws.seq_has_qual),
                                   _ptr(ws.seq_begin), _ptr(ws.win_first), match, mismatch, gap, 1 if banded else 0,
                                   max_depth, device, mem_fraction, _ptr(out), stride, _ptr(out_len), _ptr(times))
    if ok < 0:
        raise RuntimeError("reference cudapoa failed (%d)" % ok)
    return [out[i, :out_len[i]].tobytes() for i in range(n)], int(ok), float(times[0]), float(times[1])



def ref_cudapoa_multi(ws, match=3, mismatch=-5, gap=-4, banded=False, max_depth=200, n_devices=1, batches_per_device=2):
    """The reference's own multi-GPU driver shape (CUDAPolisher::polish, cudapolisher.cpp:226-345) over GenomeWorks
    cudapoa, unmodified: `batches_per_device` batch objects on each of the first n_devices GPUs, one host thread each.
    Returns (windows reported ok, wall seconds).  Timing only."""
    lib = C.CDLL(CUDAPOA_SO)
    lib.ref_cudapoa_multi.restype = C.c_int64
    lib.ref_cudapoa_multi.argtypes = [C.c_uint32] + [C.c_void_p] * 6 + [C.c_int8, C.c_int8, C.c_int8, C.c_int,
                                                                       C.c_uint32, C.c_int, C.c_int, C.c_void_p]
    seq_off = ws.seq_off.astype(np.uint64)
    times = np.zeros(2, np.float64)
    ok = lib.ref_cudapoa_multi(ws.n_windows, _ptr(ws.bases), _ptr(ws.quals), _ptr(seq_off), _ptr(ws.seq_has_qual),
                               _ptr(ws.seq_begin), _ptr(ws.win_first), match, mismatch, gap, 1 if banded else 0,
                               max_depth, n_devices, batches_per_device, times.ctypes.data)
    if ok < 0:
        raise RuntimeError("reference cudapoa (multi) failed (%d)" % ok)
    return int(ok), float(times[0])
