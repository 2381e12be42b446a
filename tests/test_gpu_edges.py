"""The POA kernel on the device at its structural edges, window by window against the int32 oracle: lengths at the 16-column
lane blocks, the 32-position aln[] blocks and the 512-column chunks of a DP row; windows of every shape, status and soft
failure mixed in one shuffled batch (state carried between windows on a persistent worker); int8 score extremes; the int16
range limits on both sides; the default racon -b band layout with the band audit on.

The case generators are plain functions.  A small subset of them also runs through the CPU warp simulation of the same
device code (`test_sim_*` below), which needs no GPU."""
import os

import numpy as np
import pytest

from oracle import bindings as ob
from racon_b200 import windows
from tests import simlib, util

THREADS = os.cpu_count() or 4
GRID = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 257, 511, 512, 513, 1023, 1024, 1025, 1535, 1536]
SCORES = [(3, -5, 0), (0, -1, -1), (1, 0, -1), (2, 3, -1), (-1, -2, -3), (0, 0, 0), (127, -128, -1), (1, -128, -64),
          (4, -128, -2), (10, -1, -20)]
WIN_NEEDS_INT32, WIN_SEQ_TOO_LONG, WIN_ALPHABET_LIMIT = 4, 5, 7
INT16_FLOOR = -32768 + 1024    # spoa's int16 margin, and the limit of PoaWarp::matrix_in_range


# ---- case generators ---------------------------------------------------------------------------------------------------
def _rand(rng, n, alphabet=util.BASES):
    return bytes(alphabet[i] for i in rng.integers(len(alphabet), size=n))


def _subst(rng, s, p):
    """substitutions only: the length stays"""
    a = bytearray(s)
    for k in np.nonzero(rng.random(len(a)) < p)[0]:
        a[k] = util.BASES[(util.BASES.index(a[k]) + 1 + int(rng.integers(3))) % 4]
    return bytes(a)


def _layer_of_length(rng, bb, n):
    """a full-span layer of exactly n bases that follows the backbone: a slice of it, or it with a random insertion"""
    if n <= len(bb):
        o = int(rng.integers(0, len(bb) - n + 1))
        return _subst(rng, bb[o:o + n], 0.05)
    k = int(rng.integers(0, len(bb) + 1))
    return _subst(rng, bb[:k] + _rand(rng, n - len(bb)) + bb[k:], 0.05)


def grid_windows(seed=1, lengths=GRID):
    """Per length L: a window with an L-base backbone and layers of L bases, and one whose layers have the neighbouring
    grid lengths.  Depths 3 / 6 / 12, partial-span layers of the grid lengths, indel layers, qualities on every other
    window, both window types."""
    rng = np.random.default_rng(seed)
    wins, types = [], []
    for i, L in enumerate(lengths):
        nxt = lengths[i + 1] if i + 1 < len(lengths) and lengths[i + 1] <= 2 * L else L
        prv = lengths[i - 1] if i > 0 else L
        for v, lens in enumerate(((L,), (nxt, prv))):
            qual = (i + v) % 2 == 1
            depth = (3, 6, 12)[(i + v) % 3]
            bb = _rand(rng, L)
            win = [(bb, util.rand_qual(rng, L) if qual and v else None, 0, 0)]
            for d in range(depth):
                n = lens[d % len(lens)]
                if d % 4 == 3 and L >= 4:       # partial span: a grid-length piece of the backbone (at most L bases)
                    n = min(n, L - 1)
                    b = int(rng.integers(0, L - n + 1))
                    piece, b, e = _subst(rng, bb[b:b + n], 0.05), b, b + n - 1
                elif d % 4 == 2 and L >= 8:     # indels: the graph branches
                    piece, b, e = util.mutate(rng, bb, 0.12) or bb[:1], 0, L - 1
                else:
                    piece, b, e = _layer_of_length(rng, bb, n), 0, L - 1
                win.append((piece, util.rand_qual(rng, len(piece)) if qual else None, b, e))
            wins.append(win)
            types.append((i + v) % 2)
    return windows.from_lists(wins, types)


def other_windows(seed=2):
    """Every other kind of window, each with the status it must get (0: equal to the oracle) at window_length 500:
    < 3 sequences, 1-base backbones, skipped layers, 9 distinct characters, deep / long windows that need the escalation
    pass, and layers just over the first pass's (1023) and the escalation pass's (4092) length limits."""
    rng = np.random.default_rng(seed)
    bb = _rand(rng, 300)
    wins = [
        ([(bb, None, 0, 0)], 0),
        ([(bb, None, 0, 0), (util.mutate(rng, bb, 0.1), None, 0, 299)], 0),
        ([(b"A", None, 0, 0), (b"A", None, 0, 0), (b"C", None, 0, 0), (b"ACGT", None, 0, 0)], 0),
        ([(b"G", None, 0, 0)] + [(_rand(rng, 3), None, 0, 0) for _ in range(3)], 0),
        ([(bb, None, 0, 0), (b"", None, 0, 5), (bb[:10], None, 7, 7), (bb[40:90], None, 40, 89),
          (util.mutate(rng, bb, 0.1), None, 0, 299), (util.mutate(rng, bb, 0.1), None, 0, 299)], 0),
        ([(b"ACGTNRYKM" * 20, None, 0, 0)] + [(b"ACGTNRYKM" * 20, None, 0, 179)] * 3, WIN_ALPHABET_LIMIT),
    ]
    for k in range(2):  # > 3064 graph nodes: the escalation pass
        wins.append((util.make_window(rng, wlen=500, depth=150, err=0.15, partial_frac=0.2 * k), 0))
    for n, st in ((1024, 0), (1600, 0), (4093, WIN_SEQ_TOO_LONG)):
        w = util.make_window(rng, wlen=500, depth=6, err=0.08)
        w.insert(3, (_layer_of_length(rng, w[0][0], n), None, 0, len(w[0][0]) - 1))
        wins.append((w, st))
    return windows.from_lists([w for w, _ in wins], [1] * len(wins)), np.array([s for _, s in wins], np.uint32)


def mixed_batch(seed=3):
    """the length grid's windows (window_length 500) and every other kind, shuffled with a fixed seed: (windows, expected status)"""
    g = grid_windows()
    o, ost = other_windows()
    allw = [g.window(i) for i in range(g.n_windows)] + [o.window(i) for i in range(o.n_windows)]
    types = list(g.win_type) + list(o.win_type)
    want = np.concatenate([np.zeros(g.n_windows, np.uint32), ost])
    perm = np.random.default_rng(seed).permutation(len(allw))
    return windows.from_lists([allw[i] for i in perm], [int(types[i]) for i in perm]), want[perm]


def int16_limit_windows():
    """Windows whose first alignment, against the backbone chain, has column 0 down to blen*g and a read of len bases,
    so that column 0's minimum + len*g lands on INT16_FLOOR - 1, INT16_FLOOR and INT16_FLOOR + 1, for several gaps, depths
    and lengths (window_length 1000).  spoa's bound fails for all of them: the finished matrix is verified."""
    rng = np.random.default_rng(4)
    wins, gaps = [], []
    for target in (-INT16_FLOOR + 1, -INT16_FLOOR, -INT16_FLOOR - 1):
        found = 0
        for g in range(-64, -4):
            total = target // -g
            ln = min(2023, total * (2 + found) // 7)
            if target % -g or total - ln > 6000 or found == 3:
                continue
            bb = _rand(rng, total - ln)
            lay = [(bb[:ln], None, 0, len(bb) - 1)] + [(_layer_of_length(rng, bb, ln), None, 0, len(bb) - 1)
                                                       for _ in range(1 + found)]
            wins.append([(bb, None, 0, 0)] + lay)
            gaps.append(g)
            found += 1
    return wins, gaps


def positive_side_windows():
    """Large match, gap -1: a short read that copies a long stretch of a >= 2600-node backbone.  spoa's bound holds
    (|g| * (nodes - len) pays for match * len), yet the best cells reach match * len > 32767."""
    rng = np.random.default_rng(5)
    out = []
    for m, x, llen, blen, off in ((127, -128, 258, 2600, 0), (127, -128, 260, 2600, 0), (127, -128, 300, 2600, 1000),
                                  (100, -5, 330, 3000, 5), (40, -1, 822, 2400, 20), (20, -5, 1643, 3020, 10),
                                  (2, 3, 1000, 2600, 0)):
        bb = _rand(rng, blen)
        lay = [(bb[off:off + llen], None, 0, blen - 1), (_subst(rng, bb[off:off + llen], 0.02), None, 0, blen - 1),
               (bb[off:off + llen], None, 0, blen - 1)]
        out.append(((m, x, -1), windows.from_lists([[(bb, None, 0, 0)] + lay])))
    return out


def expected_range_status(ranges, m, x, g):
    """What PoaWarp must answer, from the oracle's int32 matrices of one window (oracle_matrix_ranges): RP_WIN_NEEDS_INT32
    at the first alignment whose cells could leave int16 (the largest step times the short side over 32767 - 1024, or spoa's
    bound failing and column 0's minimum + len * g below INT16_FLOOR), else 0."""
    top = max(m, x, 0)
    for ln, n, col0, _, _ in ranges:
        i, j = int(ln) + 8, int(n)
        worst = min(-(m * min(i, j) + g * abs(i - j)), g * (i + j))
        if g < -64 or top * min(i, j) > 32767 - 1024:
            return WIN_NEEDS_INT32
        if worst < INT16_FLOOR and col0 + ln * g < INT16_FLOOR:
            return WIN_NEEDS_INT32
    return 0


# ---- checks ------------------------------------------------------------------------------------------------------------
_oracle_cache = {}


def oracle(ws, key, scores=(3, -5, -4), trim=True):
    k = (key, scores, trim)
    if k not in _oracle_cache:
        _oracle_cache[k] = ob.oracle_consensus(ws, *scores, trim=trim, threads=THREADS, want_coverage=True)
    return _oracle_cache[k]


def check(ws, got, want, want_status=None, what=""):
    """got = (consensus, polished, status[, coverage]) of the device; want = the oracle's (consensus, polished, _, coverage).
    Status 0: consensus, polished flag and (polished windows) coverage equal the oracle's.  Any other status must be the
    expected one and come with an empty, unpolished consensus."""
    cons, pol, st = got[:3]
    want_status = np.zeros(ws.n_windows, np.uint32) if want_status is None else want_status
    bad_st = [w for w in range(ws.n_windows) if st[w] != want_status[w]]
    assert not bad_st, "%s: status differs on windows %s: got %s, expected %s" % (
        what, bad_st[:8], [int(st[w]) for w in bad_st[:8]], [int(want_status[w]) for w in bad_st[:8]])
    for w in range(ws.n_windows):
        if st[w]:
            assert cons[w] == b"" and not pol[w], "%s: window %d with status %d" % (what, w, st[w])
            continue
        assert cons[w] == want[0][w], "%s: consensus differs on window %d" % (what, w)
        assert pol[w] == want[1][w], "%s: polished flag differs on window %d" % (what, w)
        if len(got) > 3 and pol[w]:
            assert (got[3][w].astype(np.uint32) == want[3][w]).all(), "%s: coverage differs on window %d" % (what, w)


def sim(ws, scores=(3, -5, -4), trim=True, window_length=500, **kw):
    lim = dict(nmax=max(1024, 6 * window_length + 64), lmax=2 * window_length + 23)
    lim.update(kw)
    cons, pol, st, cov, stats = simlib.sim_consensus(ws, *scores, trim=trim, **lim)
    return (cons, pol, st, cov), stats


# ---- CPU twins: the same cases through the warp simulation (a subset: it runs one window at a time on the CPU) ------------
SIM_LENGTHS = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 257, 511, 512, 513]


@pytest.mark.parametrize("trim", [True, False])
def test_sim_length_grid(trim):
    ws = grid_windows(seed=11, lengths=SIM_LENGTHS)
    want = ob.oracle_consensus(ws, trim=trim, threads=THREADS, want_coverage=True)
    got, _ = sim(ws, trim=trim)
    check(ws, got, want, what="sim grid")
    got, stats = sim(ws, trim=trim, lanes=32, smem=9216, banded=1, band_cols_per_lane=8, debug_flags=2)
    check(ws, got, want, what="sim grid banded")
    assert stats[4] > 0 and stats[6] == 0, stats


@pytest.mark.parametrize("scores", SCORES)
def test_sim_score_extremes(scores):
    ws = grid_windows(seed=12, lengths=[1, 16, 17, 33, 64, 255, 257, 513])
    want = ob.oracle_consensus(ws, *scores, threads=THREADS, want_coverage=True)
    exp = np.array([expected_range_status(r, *scores) for r in ob.oracle_matrix_ranges(ws, *scores)], np.uint32)
    check(ws, sim(ws, scores)[0], want, exp, what="sim %s" % (scores,))


def test_sim_int16_limits():
    wins, gaps = int16_limit_windows()
    margins = set()
    for win, g in zip(wins, gaps):
        if len(win[0][0]) + len(win[1][0]) > 3600:   # the simulation's time
            continue
        ws = windows.from_lists([win])
        ranges = ob.oracle_matrix_ranges(ws, 3, -5, g)[0]
        margins.update(int(c0 + ln * g) for ln, _, c0, _, _ in ranges)
        exp = np.array([expected_range_status(ranges, 3, -5, g)], np.uint32)
        want = ob.oracle_consensus(ws, 3, -5, g, threads=1, want_coverage=True)
        check(ws, sim(ws, (3, -5, g), window_length=1000)[0], want, exp, what="sim gap %d" % g)
    assert {INT16_FLOOR - 1, INT16_FLOOR, INT16_FLOOR + 1} <= margins


def test_sim_int16_positive_side():
    for scores, ws in positive_side_windows():
        ranges = ob.oracle_matrix_ranges(ws, *scores)[0]
        exp = np.array([expected_range_status(ranges, *scores)], np.uint32)
        got, _ = sim(ws, scores, nmax=8192, lmax=4095)
        check(ws, got, ob.oracle_consensus(ws, *scores, want_coverage=True), exp, what="sim %s" % (scores,))
        assert got[2][0] or ranges[:, 4].max() <= 32767, "computed in int16, but the matrix reaches %d" % ranges[:, 4].max()


def test_sim_band_refusals_audited():
    """Layers with 110-base deletions / 120-base insertions in a 128-column band: refused band results are redone, the
    accepted ones equal the full matrix's (audit), the consensus equals the oracle's."""
    rng = np.random.default_rng(6)
    wins = []
    for _ in range(2):
        truth = _rand(rng, 500)
        bb = util.mutate(rng, truth, 0.1)[:500]
        win = [(bb, None, 0, 0)]
        for d in range(9):
            r = util.mutate(rng, truth, 0.1)
            r = r[:150] + r[260:] if d % 3 == 0 else r[:200] + _rand(rng, 120) + r[200:] if d % 3 == 1 else r
            win.append((r, None, 0, len(bb) - 1))
        wins.append(win)
    ws = windows.from_lists(wins)
    want = ob.oracle_consensus(ws, threads=THREADS, want_coverage=True)
    got, stats = sim(ws, window_length=1000, lanes=32, smem=9216, banded=1, band_cols_per_lane=4, debug_flags=2)
    check(ws, got, want, what="sim band 128")
    assert 0 < stats[5] < stats[4] and stats[6] == 0, stats


# ---- on the device -------------------------------------------------------------------------------------------------------
def _device(ws, scores=(3, -5, -4), trim=True, window_length=500, banded=False, band_stats=None, mem_bytes=0):
    from racon_b200 import api
    return api.consensus(ws, *scores, trim=trim, window_length=window_length, want_coverage=True, banded=banded,
                         band_stats=band_stats, mem_bytes=mem_bytes)


BAND_MODES = {"full": (False, None), "band_default": (True, None), "band_k4": (True, "4"), "band_k8": (True, "8")}


@pytest.mark.gpu
@pytest.mark.parametrize("trim", [True, False], ids=["trim", "no_trim"])
@pytest.mark.parametrize("mode", sorted(BAND_MODES))
@pytest.mark.parametrize("window_length", [500, 1000])
def test_gpu_length_grid(window_length, mode, trim, monkeypatch):
    banded, k = BAND_MODES[mode]
    if k:
        monkeypatch.setenv("RP_POA_BAND_K", k)
    monkeypatch.setenv("RP_BAND_AUDIT", "1")
    ws = grid_windows()
    stats = {}
    check(ws, _device(ws, trim=trim, window_length=window_length, banded=banded, band_stats=stats),
          oracle(ws, "grid", trim=trim), what="%s w=%d" % (mode, window_length))
    if banded and (k or window_length == 1000):
        assert stats["band_layout_in_use"] and stats["band_alignments"] > 0, stats
        assert stats["band_audit_mismatches"] == 0, stats


@pytest.mark.gpu
@pytest.mark.parametrize("banded", [False, True], ids=["full", "banded"])
@pytest.mark.parametrize("lanes", [8, 16])
@pytest.mark.parametrize("window_length", [500, 1000])
def test_gpu_length_grid_group_widths(window_length, lanes, banded, monkeypatch):
    monkeypatch.setenv("RP_POA_GROUP", str(lanes))
    monkeypatch.setenv("RP_BAND_AUDIT", "1")
    # an 8-lane group's shared memory (3.5 KB) holds the rank update of graphs up to ~1 780 nodes: the grid's 1023+
    # windows exceed that and are refused (RP_WIN_NODE_LIMIT), so 8 lanes run the grid up to 513 bases
    lengths = GRID if lanes == 16 else GRID[:16]
    ws = grid_windows(lengths=lengths)
    stats = {}
    check(ws, _device(ws, window_length=window_length, banded=banded, band_stats=stats),
          oracle(ws, "grid%d" % len(lengths)), what="%d lanes w=%d" % (lanes, window_length))
    if banded:
        assert stats["band_alignments"] > 0 and stats["band_audit_mismatches"] == 0, stats


@pytest.mark.gpu
def test_gpu_mixed_batch_is_order_and_company_independent():
    """All kinds of window in one shuffled batch: each equals the oracle or has its documented soft status, and the
    results are identical in reverse order, when each window runs alone, and when a small memory budget shrinks the
    per-window matrix scratch (hcap_min) so that large windows go through the escalation pass among the others."""
    from racon_b200 import api
    ws, want_st = mixed_batch()
    want = oracle(ws, "mixed")
    got = _device(ws)
    check(ws, got, want, want_st, what="shuffled")
    n = ws.n_windows
    rev = _device(ws.subset(np.arange(n)[::-1]))
    assert [rev[0][n - 1 - w] for w in range(n)] == got[0] and (rev[2][::-1] == got[2]).all()
    for w in range(n):
        alone = _device(ws.subset([w]))
        assert alone[0][0] == got[0][w] and alone[1][0] == got[1][w] and alone[2][0] == got[2][w], "window %d" % w
    b = api.PoaBatch(mem_bytes=4 << 30, window_length=500)
    try:
        assert b.add_window_set(ws) == n
        b.run()
        b.sync()
        out, lens, pol, st = b.fetch_all(2 * 4093 + 64)
        launches = b.info()["launches"]
    finally:
        b.close()
    assert launches >= 2, "no window went through the escalation pass"
    assert (st == got[2]).all() and [out[w, :lens[w]].tobytes() for w in range(n)] == got[0]


@pytest.mark.gpu
@pytest.mark.parametrize("scores", SCORES)
def test_gpu_score_extremes(scores):
    ws = grid_windows(lengths=GRID[:16])
    exp = np.array([expected_range_status(r, *scores) for r in ob.oracle_matrix_ranges(ws, *scores)], np.uint32)
    check(ws, _device(ws, scores), oracle(ws, "grid16", scores), exp, what=str(scores))
    mixed, want_st = mixed_batch()
    # not the deep windows (the oracle's matrix trace is serial), nor the one whose over-long layer would meet an earlier
    # int16 refusal first
    keep = [w for w in range(mixed.n_windows) if len(mixed.window(w)) < 60 and want_st[w] != WIN_SEQ_TOO_LONG]
    mixed = mixed.subset(keep)
    ranges = ob.oracle_matrix_ranges(mixed, *scores)
    exp = np.array([s or expected_range_status(r, *scores) for s, r in zip(want_st[keep], ranges)], np.uint32)
    check(mixed, _device(mixed, scores), oracle(mixed, "mixed_small", scores), exp, what="mixed %s" % (scores,))


@pytest.mark.gpu
def test_gpu_int16_limits():
    wins, gaps = int16_limit_windows()
    for win, g in zip(wins, gaps):
        ws = windows.from_lists([win])
        ranges = ob.oracle_matrix_ranges(ws, 3, -5, g)[0]
        exp = np.array([expected_range_status(ranges, 3, -5, g)], np.uint32)
        want = ob.oracle_consensus(ws, 3, -5, g, want_coverage=True)
        check(ws, _device(ws, (3, -5, g), window_length=1000), want, exp, what="gap %d" % g)
    for scores, ws in positive_side_windows():
        ranges = ob.oracle_matrix_ranges(ws, *scores)[0]
        exp = np.array([expected_range_status(ranges, *scores)], np.uint32)
        got = _device(ws, scores, window_length=1500)
        check(ws, got, ob.oracle_consensus(ws, *scores, want_coverage=True), exp, what=str(scores))
        assert got[2][0] or ranges[:, 4].max() <= 32767


def _synthetic_w1000(seed, err):
    return util.make_set(seed, 12, wlen=1000, depth=16, err=err, partial_frac=0.2, with_qual=True)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [None, "4"], ids=["band256", "band128"])
def test_gpu_default_band_layout_audited(k, monkeypatch):
    """racon -b with the band layout a w = 1000 object uses (32 lanes x 8 columns; RP_POA_BAND_K=4: x 4), band audit on: every
    accepted band alignment equals the full matrix's, and the consensus equals the reference's answers."""
    from tests import test_lambda as tl
    from racon_b200 import api
    if k:
        monkeypatch.setenv("RP_POA_BAND_K", k)
    monkeypatch.setenv("RP_BAND_AUDIT", "1")
    width = 128 if k else 256
    lam, lam_ref, _, _ = tl.load()
    w1000, w1000_ref, _ = tl.load_w1000()
    frag, frag_ref = tl.load_frag()
    cases = [(lam, lam_ref, (3, -5, -4)), (w1000, w1000_ref, (5, -4, -8)), (frag, frag_ref, (1, -1, -1))]
    for seed, err in ((7, 0.12), (8, 0.3)):
        ws = _synthetic_w1000(seed, err)
        cases.append((ws, ob.oracle_consensus(ws, threads=THREADS)[0], (3, -5, -4)))
    for ws, ref, scores in cases:
        stats = {}
        cons, pol, st = api.consensus(ws, *scores, window_length=1000, banded=True, band_stats=stats)
        assert (st == 0).all(), st
        bad = [w for w in range(ws.n_windows) if cons[w] != ref[w]]
        assert not bad, "windows differ: %s" % bad[:8]
        assert stats["band_layout_in_use"] and stats["band_width"] == width, stats
        assert stats["band_alignments"] > 0 and stats["band_audit_mismatches"] == 0, stats
