"""ctypes access to the TEST-ONLY host simulation of the device code (racon_b200/lib/libracon_sim.so)."""
import ctypes as C

import numpy as np

from racon_b200 import build

_lib = None


def lib():
    global _lib
    if _lib is None:
        l = C.CDLL(build.build_sim())
        l.rp_sim_poa.restype = C.c_int
        l.rp_sim_poa.argtypes = [C.c_uint32] + [C.c_void_p] * 8 + [C.c_int8, C.c_int8, C.c_int8, C.c_int,
                                                                    C.c_void_p, C.c_void_p, C.c_uint32,
                                                                    C.c_void_p, C.c_void_p, C.c_void_p,
                                                                    C.c_void_p, C.c_void_p]
        l.rp_sim_aln.restype = C.c_int
        l.rp_sim_aln.argtypes = [C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                                                    C.c_void_p, C.c_void_p, C.c_void_p]
        l.rp_sim_aln_bp.restype = C.c_int
        l.rp_sim_aln_bp.argtypes = [C.c_uint32] + [C.c_void_p] * 5 + [C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32,
                                                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32,
                                                                       C.c_void_p]
        _lib = l
    return _lib


def _ptr(a):
    return None if a is None else a.ctypes.data


def sim_consensus(ws, m=3, x=-5, g=-4, trim=True, nmax=4096, lmax=1535, ki=16, ka=8, smem=14336, tile_rows=0, debug_flags=0,
                  lanes=32, banded=0, band_margin=16, hcap=0, band_cols_per_lane=16):
    n = ws.n_windows
    lens = np.diff(ws.seq_off.astype(np.int64))
    stride = int(max(64, 2 * lens.max() + 64))
    out = np.zeros((n, stride), dtype=np.uint8)
    cov = np.zeros((n, stride), dtype=np.uint16)
    out_len = np.zeros(n, dtype=np.uint32)
    pol = np.zeros(n, dtype=np.uint8)
    st = np.zeros(n, dtype=np.uint32)
    stats = np.zeros(8, dtype=np.uint64)
    limits = np.asarray([nmax, lmax, ki, ka, smem, tile_rows, debug_flags, lanes, banded, band_margin, hcap,
                         band_cols_per_lane], dtype=np.uint32)
    r = lib().rp_sim_poa(n, _ptr(ws.bases), _ptr(ws.quals), _ptr(ws.seq_off), _ptr(ws.seq_has_qual),
                         _ptr(ws.seq_begin), _ptr(ws.seq_end), _ptr(ws.win_first), _ptr(ws.win_type), m, x, g,
                         1 if trim else 0, limits.ctypes.data, out.ctypes.data, stride, out_len.ctypes.data,
                         pol.ctypes.data, st.ctypes.data, cov.ctypes.data, stats.ctypes.data)
    if r != 0:
        raise RuntimeError("rp_sim_poa failed: %d" % r)
    cons = [out[w, :out_len[w]].tobytes() for w in range(n)]
    covs = [cov[w, :out_len[w]].copy() for w in range(n)]
    return cons, pol.astype(bool), st, covs, stats


def runs_to_cigar(runs):
    return "".join("%d%s" % (int(r) >> 8, chr(int(r) & 0xff)) for r in runs)


def sim_align(pairs, max_len=None, store_words=53000, run_stride=None):
    """pairs: [(query bytes, target bytes), ...] -> ([(cigar, distance)], status array).  run_stride: the run capacity
    of every pair (default 2 * max_len + 8, more than any CIGAR needs)."""
    n = len(pairs)
    blob = b"".join(q + t for q, t in pairs)
    bases = np.frombuffer(blob, dtype=np.uint8).copy() if blob else np.zeros(1, np.uint8)
    q_off = np.zeros(n, np.uint32)
    q_len = np.zeros(n, np.uint32)
    t_off = np.zeros(n, np.uint32)
    t_len = np.zeros(n, np.uint32)
    o = 0
    for i, (q, t) in enumerate(pairs):
        q_off[i], q_len[i] = o, len(q)
        o += len(q)
        t_off[i], t_len[i] = o, len(t)
        o += len(t)
    if max_len is None:
        max_len = int(max([1] + [max(len(q), len(t)) for q, t in pairs]))
    stride = run_stride or 2 * max_len + 8
    runs = np.zeros((n, stride), np.uint32)
    n_runs = np.zeros(n, np.uint32)
    dist = np.zeros(n, np.int32)
    st = np.zeros(n, np.uint32)
    r = lib().rp_sim_aln(n, bases.ctypes.data, q_off.ctypes.data, q_len.ctypes.data, t_off.ctypes.data,
                         t_len.ctypes.data, max_len, store_words, runs.ctypes.data, stride, n_runs.ctypes.data,
                         dist.ctypes.data, st.ctypes.data)
    assert r == 0
    return [(runs_to_cigar(runs[i, :n_runs[i]]), int(dist[i])) for i in range(n)], st


def sim_align_bp(cases, window_length, store_words=53000):
    """cases: [(query, target, t_begin, q_start)] -> [(cigar, distance, (n,2) breaking points)], status"""
    n = len(cases)
    blob = b"".join(q + t for q, t, _, _ in cases)
    bases = np.frombuffer(blob, dtype=np.uint8).copy()
    q_off = np.zeros(n, np.uint32)
    q_len = np.zeros(n, np.uint32)
    t_off = np.zeros(n, np.uint32)
    t_len = np.zeros(n, np.uint32)
    t_begin = np.asarray([c[2] for c in cases], np.uint32)
    q_start = np.asarray([c[3] for c in cases], np.uint32)
    o = 0
    for i, (q, t, _, _) in enumerate(cases):
        q_off[i], q_len[i] = o, len(q)
        o += len(q)
        t_off[i], t_len[i] = o, len(t)
        o += len(t)
    max_len = int(max(max(len(q), len(t)) for q, t, _, _ in cases))
    stride = 2 * max_len + 8
    bstride = 2 * (max_len // window_length + 3)
    runs = np.zeros((n, stride), np.uint32)
    n_runs = np.zeros(n, np.uint32)
    dist = np.zeros(n, np.int32)
    st = np.zeros(n, np.uint32)
    bp = np.zeros((n, bstride, 2), np.uint32)
    n_bp = np.zeros(n, np.uint32)
    r = lib().rp_sim_aln_bp(n, bases.ctypes.data, q_off.ctypes.data, q_len.ctypes.data, t_off.ctypes.data,
                            t_len.ctypes.data, max_len, store_words, runs.ctypes.data, stride, n_runs.ctypes.data,
                            dist.ctypes.data, st.ctypes.data, window_length, t_begin.ctypes.data, q_start.ctypes.data,
                            bp.ctypes.data, bstride, n_bp.ctypes.data)
    assert r == 0
    return [(runs_to_cigar(runs[i, :n_runs[i]]), int(dist[i]), bp[i, :n_bp[i]].copy()) for i in range(n)], st

