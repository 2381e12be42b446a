"""The POA kernel at the limits of the graph's shape, window by window against the int32 oracle.

- In-degree: a node's predecessors sit in its DP record (the first 7) and then in pred_ovf; the traceback scans up to 7
  of them serially, 8 to 32 one per lane, more than 32 in traceback_step_wide; the first pass keeps 16 in-edge slots
  per node and the escalation pass 96 (which switches the staged subgraph DFS off).  A "hub" node that many layers reach
  through different deletions / insertions just before it gets the in-degree; a seeded search over such windows, on
  the oracle's shape report, picks one window for every boundary.
- Aligned clusters: windows of exactly 8 characters where columns carry all 8 (al_cnt = 7 in the staged DFS's packed
  byte), with partial-span layers after them.
- Node count: graphs that cross, by one layer, the first pass's node budget (lim.nmax), the node count at which the
  order update's counters (add_alignment, Phase D) leave the group's shared memory for the slot's HBM copy, and the
  escalation pass's budget (lim_big.nmax).  Every node count up to lim_big.nmax must give status 0, in every layout.

The case generators are plain functions.  The CPU twins (`test_sim_*`) run small versions through the warp simulation."""
import os

import numpy as np
import pytest

from oracle import bindings as ob
from racon_b200 import windows
from tests import simlib, util
from tests.test_gpu_edges import _rand, check

THREADS = os.cpu_count() or 4
WIN_NODE_LIMIT, WIN_EDGE_LIMIT = 1, 2
INDEG_TARGETS = (3, 4, 7, 8, 9, 16, 17, 31, 32, 33)
SIM_INDEG_TARGETS = (7, 8, 16, 17, 24, 25, 32, 33)
CLUSTER_ALPHABET = b"ACGTNRYK"   # 8 codes: the window alphabet's limit


# ---- case generators ---------------------------------------------------------------------------------------------------
def hub_window(rng, n_layers, dmax, imax, blen=300, hub=250, partial=0.0, qual=False, tie=None, hub_sub=0.0):
    """A backbone with a unique hub character N at `hub`; every layer copies the backbone but deletes up to dmax bases
    just before the hub and inserts up to imax random ones there, so the hub collects in-edges from many tails.  With
    `partial`, that share of the layers covers only a stretch around the hub (begin > 1 % of the backbone), so some of
    the hub's predecessors fall outside the layer's subgraph.  `tie`: the bases before the hub are this repeat, so that
    deletions there tie and in-edge order decides the traceback.  `hub_sub`: that share of the layers has another base
    in the hub's place, so that the walk through the hub's row meets vertical candidates next to diagonal ones."""
    bb = bytearray(_rand(rng, blen))
    if tie:
        bb[hub - 24:hub] = (tie * 24)[:24]
    bb[hub] = ord("N")
    bb = bytes(bb)
    win = [(bb, None, 0, 0)]
    for _ in range(n_layers):
        d, i = int(rng.integers(0, dmax + 1)), int(rng.integers(0, imax + 1))
        b, e = 0, blen - 1
        if partial and rng.random() < partial:
            b = int(rng.integers(hub - min(hub - 4, 120), hub - 8))
            e = int(rng.integers(hub + 8, blen - 4))
            d = min(d, hub - b - 1)
        tail = bb[hub:e + 1]
        if hub_sub and rng.random() < hub_sub:
            tail = _rand(rng, 1) + tail[1:]
        lay = bb[b:hub - d] + _rand(rng, i) + tail
        win.append((lay, util.rand_qual(rng, len(lay)) if qual else None, b, e))
    return win


def indegree_ladder(seed, targets=INDEG_TARGETS, scores=(3, -5, -4), blen=300, hub=250, max_layers=400, **kw):
    """Seeded search over hub windows: one window whose final graph's largest in-degree (oracle) is exactly each target,
    and the window of the highest in-degree met.  Returns (window lists, in-degrees); asserts every target was hit."""
    rng = np.random.default_rng(seed)
    found, best = {}, (0, None)
    for _ in range(60):
        cands = []
        for k in range(32):
            n = int(np.exp(rng.uniform(np.log(2), np.log(60)))) if k % 2 else int(rng.integers(60, max_layers + 1))
            cands.append(hub_window(rng, n, int(rng.integers(1, hub - 10)), int(rng.integers(0, 9)), blen=blen, hub=hub,
                                    **kw))
        shapes = ob.oracle_graph_shape(windows.from_lists(cands), *scores, threads=THREADS)
        for c, (_, deg, _) in zip(cands, shapes):
            if deg in targets and deg not in found:
                found[deg] = c
            if deg > best[0]:
                best = (deg, c)
        if len(found) == len(targets) and best[0] > max(targets):
            break
    missing = sorted(set(targets) - set(found))
    assert not missing, "no window reached in-degree %s" % missing
    degs = sorted(found) + ([best[0]] if best[0] not in found else [])
    return [found[d] if d in found else best[1] for d in degs], degs


def cluster_windows(seed=21, n=4, blen=240):
    """Windows of exactly 8 characters: 7 full-span layers substitute, at every 6th column, each of the 7 characters the
    backbone does not have there (so those columns' aligned clusters are full: 8 nodes, 7 aligned each), more full-span
    layers pick any of the 8, and partial-span layers (aligned after them: layers are sorted by begin) walk the full
    clusters in the subgraph DFS."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        bb = _rand(rng, blen)
        cols = list(range(3, blen - 3, 6))
        win = [(bb, None, 0, 0)]
        for t in range(10):
            a = bytearray(bb)
            for c in cols:
                if t < 7:
                    k = CLUSTER_ALPHABET.index(bb[c])
                    a[c] = CLUSTER_ALPHABET[(k + 1 + t) % 8]
                else:
                    a[c] = CLUSTER_ALPHABET[int(rng.integers(8))]
            win.append((bytes(a), util.rand_qual(rng, blen) if t % 3 == 2 else None, 0, blen - 1))
        for _ in range(6):
            b = int(rng.integers(blen // 10, blen // 2))
            e = int(rng.integers(b + 20, blen - blen // 10))
            a = bytearray(bb[b:e + 1])
            for c in cols:
                if b <= c <= e:
                    a[c - b] = CLUSTER_ALPHABET[int(rng.integers(8))]
            win.append((bytes(a), None, b, e))
        out.append(win)
    return out


def node_ladder(seed, caps, window_length, reach=1):
    """For every cap c, windows whose graph crosses it by a single layer: a backbone of about c - 150 bases and
    partial-span copies of short stretches of it, each with a random insertion of 40-80 bases (the insertion's bases are
    the new nodes).  Per cap: the prefix of the layers that stays <= c, the one more layer that crosses c, and (reach=2)
    one more layer aligned to the graph of > c nodes.  Returns (window lists, final node counts)."""
    rng = np.random.default_rng(seed)
    wins = []
    for c in caps:
        blen = c - 150
        bb = _rand(rng, blen)
        lay = []
        for k in range(8):
            b = int(rng.integers(blen // 10, blen - blen // 10 - 200))
            piece = bb[b:b + 150]
            ins = _rand(rng, int(rng.integers(40, 81)))
            lay.append((piece[:75] + ins + piece[75:], None, b, b + 149))
        lay.sort(key=lambda s: s[2])   # the order layers are aligned in, so that a prefix is a prefix of that order
        full = [(bb, None, 0, 0)] + lay
        nodes = ob.oracle_graph_shape(windows.from_lists([full]), window_length=window_length)[0][0]
        k = int(np.searchsorted(nodes, c, side="right"))    # nodes[k - 1] <= c < nodes[k]
        assert 3 <= k < len(nodes) - reach, (c, nodes)
        for j in range(k, k + 1 + reach):
            wins.append(full[:j])
    shapes = ob.oracle_graph_shape(windows.from_lists(wins), window_length=window_length, threads=THREADS)
    return wins, [int(s[0][-1]) for s in shapes]


# ---- limits as the library configures them --------------------------------------------------------------------------
def node_caps(window_length, band_k=16, smem_per_sm=None):
    """(lim.nmax, lim_big.nmax, the node count above which Phase D's counters leave shared memory) for a 32-lane object
    with this many columns per lane of a row (16: full matrix), from rp_api.cu's configure()."""
    if smem_per_sm is None:
        import torch
        p = torch.cuda.get_device_properties(0)
        smem_per_sm, optin = p.shared_memory_per_multiprocessor, p.shared_memory_per_block_optin
    else:
        optin = smem_per_sm
    blocks_per_sm = 3 if band_k == 16 else 5
    per_block = min(smem_per_sm // blocks_per_sm - 1024, optin)
    per_group = (per_block // 4) & ~255
    nmax = min(65000, max(1024, 6 * window_length + 64))
    return nmax, min(65000, 8 * nmax), per_group // 2 - 4


# ---- checks ------------------------------------------------------------------------------------------------------------
def _oracle(ws, scores=(3, -5, -4)):
    return ob.oracle_consensus(ws, *scores, threads=THREADS, want_coverage=True)


def _sim(ws, scores=(3, -5, -4), window_length=500, **kw):
    lim = dict(nmax=max(1024, 6 * window_length + 64), lmax=2 * window_length + 23)
    lim.update(kw)
    cons, pol, st, cov, stats = simlib.sim_consensus(ws, *scores, **lim)
    return cons, pol, st, cov


def _device(ws, scores=(3, -5, -4), window_length=500, banded=False, band_stats=None):
    """(consensus, polished, status, coverage) of one batch object, and how many kernel launches it took"""
    from racon_b200 import api
    b = api.PoaBatch(match=scores[0], mismatch=scores[1], gap=scores[2], window_length=window_length, banded=banded)
    try:
        n = ws.n_windows
        assert b.add_window_set(ws) == n
        b.run()
        b.sync()
        lens_in = np.diff(ws.seq_off.astype(np.int64))
        out, lens, pol, st = b.fetch_all(int(2 * lens_in.max() + 64))
        covs = [b.fetch(i)[1] for i in range(n)]
        if band_stats is not None:
            band_stats.update(b.band_info())
        return ([out[w, :lens[w]].tobytes() for w in range(n)], pol, st, covs), b.info()["launches"]
    finally:
        b.close()


# ---- CPU twins -----------------------------------------------------------------------------------------------------------
_sim_cache = {}


def test_oracle_graph_shape_agrees_with_the_oracle_statistics():
    """The shape hook, window by window, against oracle_poa_stats's maxima (one window per call) and the window sizes:
    one node count per aligned layer plus the backbone, non-decreasing, starting at the backbone's length."""
    rng = np.random.default_rng(3)
    wins = [hub_window(rng, n, 40, 3, partial=0.3) for n in (2, 9, 40)] + cluster_windows(n=1, blen=60)
    wins.append([(b"ACGT", None, 0, 0), (b"ACGT", None, 0, 3)])   # < 3 sequences: no graph
    lib = ob.oracle_lib()
    stats = np.zeros(12, np.uint64)
    for win in wins:
        ws = windows.from_lists([win])
        lib.oracle_poa_stats(stats.ctypes.data)
        ob.oracle_consensus(ws)
        lib.oracle_poa_stats(stats.ctypes.data)
        nodes, indeg, aligned = ob.oracle_graph_shape(ws)[0]
        if len(win) < 3:
            assert len(nodes) == 0 and stats[7] == 0
            continue
        assert len(nodes) == len(win) and nodes[0] == len(win[0][0]) and (np.diff(nodes.astype(np.int64)) >= 0).all()
        assert (nodes[-1], indeg, aligned) == (stats[7], stats[8], stats[9])


def sim_ladder():
    """small hub windows (a 100-base backbone) for the simulation, at the in-degrees around 8, 16/17, 24/25, 32/33"""
    if "ladder" not in _sim_cache:
        wins, degs = indegree_ladder(31, SIM_INDEG_TARGETS, blen=100, hub=85, max_layers=260, partial=0.3,
                                     hub_sub=0.15)
        _sim_cache["ladder"] = (windows.from_lists(wins), np.array(degs))
    return _sim_cache["ladder"]


@pytest.mark.parametrize("debug_flags", [0, 1], ids=["staged", "hbm"])
@pytest.mark.parametrize("ki,lanes", [(16, 32), (24, 32), (96, 32), (96, 16)])
def test_sim_indegree_ladder(ki, lanes, debug_flags):
    """ki = 16 (the first pass): RP_WIN_EDGE_LIMIT exactly above in-degree 16; ki = 24: the same boundary at 24; ki = 96
    (the escalation pass, no staged DFS): every window computed, the ones above 32 (16) predecessors by the wide walk."""
    ws, degs = sim_ladder()
    want = _oracle(ws)
    exp = np.where(degs > ki, WIN_EDGE_LIMIT, 0).astype(np.uint32)
    check(ws, _sim(ws, ki=ki, lanes=lanes, debug_flags=debug_flags), want, exp, what="sim ki=%d" % ki)
    assert degs.max() > 32 and set(SIM_INDEG_TARGETS) <= set(degs.tolist())


def test_sim_full_clusters():
    wins = cluster_windows(n=2, blen=120)
    ws = windows.from_lists(wins)
    assert all(s[2] == 7 for s in ob.oracle_graph_shape(ws))
    want = _oracle(ws)
    for flags in (0, 1):
        check(ws, _sim(ws, debug_flags=flags), want, what="sim clusters debug_flags=%d" % flags)


def test_sim_node_count_past_the_shared_memory_counters():
    """A 32 x 8 band object's shared memory (11 264 B per group on the H100) holds the order update's counters for
    5 628 nodes: graphs around that count, within nmax, must be computed."""
    cap = 11264 // 2 - 4
    wins, nodes = node_ladder(41, [cap], window_length=1000, reach=2)
    ws = windows.from_lists(wins)
    assert nodes[0] <= cap < nodes[1] < nodes[2]
    want = _oracle(ws)
    check(ws, _sim(ws, window_length=1000, smem=11264, banded=1, band_cols_per_lane=8), want, what="sim band 32x8")
    check(ws, _sim(ws, window_length=1000, smem=11264), want, what="sim full, 11 KB")


def test_sim_node_budget_is_exact():
    """The node budget (lim.nmax in the first pass, lim_big.nmax in the escalation pass: the same check) refuses a window
    exactly when its graph grows past it, whichever layer does it."""
    nmax = 1600
    wins, nodes = node_ladder(43, [nmax], window_length=500, reach=2)
    ws = windows.from_lists(wins)
    assert nodes[0] <= nmax < nodes[1]
    exp = np.where(np.array(nodes) > nmax, WIN_NODE_LIMIT, 0).astype(np.uint32)
    check(ws, _sim(ws, nmax=nmax), _oracle(ws), exp, what="sim nmax %d" % nmax)


# ---- on the device -------------------------------------------------------------------------------------------------------
_gpu_cache = {}

LADDER_VARIANTS = {
    "plain": ((3, -5, -4), {}),
    "partial": ((3, -5, -4), {"partial": 0.4}),
    "qual": ((3, -5, -4), {"qual": True}),
    "scores_5_4_8": ((5, -4, -8), {}),
    "scores_1_1_1": ((1, -1, -1), {}),
    "tie_homopolymer": ((3, -5, -4), {"tie": b"A"}),
    "tie_repeat": ((3, -5, -4), {"tie": b"ACG", "partial": 0.2}),
}


def gpu_ladder(variant):
    if variant not in _gpu_cache:
        scores, kw = LADDER_VARIANTS[variant]
        seed = 100 + sorted(LADDER_VARIANTS).index(variant)
        wins, degs = indegree_ladder(seed, scores=scores, **kw)
        ws = windows.from_lists(wins)
        _gpu_cache[variant] = (ws, np.array(degs), _oracle(ws, scores))
    return _gpu_cache[variant]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", sorted(LADDER_VARIANTS))
def test_gpu_indegree_ladder(variant):
    """Every in-degree target, plus the highest the search met, equal to the oracle with status 0; the windows above 16
    in-edges go through the escalation pass (96 slots)."""
    scores = LADDER_VARIANTS[variant][0]
    ws, degs, want = gpu_ladder(variant)
    got, launches = _device(ws, scores)
    check(ws, got, want, what=variant)
    assert degs.max() > 33 and launches >= 2, (degs.tolist(), launches)


@pytest.mark.gpu
def test_gpu_indegree_ladder_alone_and_mixed():
    """The ladders' windows of all score-(3,-5,-4) variants in one shuffled batch, and the plain ladder's windows at and
    around the 8 / 17 / 33 boundaries alone: identical."""
    names = [v for v in sorted(LADDER_VARIANTS) if LADDER_VARIANTS[v][0] == (3, -5, -4)]
    sets = [gpu_ladder(v) for v in names]
    allw = [ws.window(i) for ws, _, _ in sets for i in range(ws.n_windows)]
    perm = np.random.default_rng(7).permutation(len(allw))
    mixed = windows.from_lists([allw[i] for i in perm])
    want = _oracle(mixed)
    got, launches = _device(mixed)
    check(mixed, got, want, what="shuffled")
    assert launches >= 2
    plain, degs, _ = gpu_ladder("plain")
    first = sum(ws.n_windows for ws, _, _ in sets[:names.index("plain")])   # the plain ladder's first window in allw
    for i in np.nonzero(np.isin(degs, (7, 8, 16, 17, 32, 33)) | (degs == degs.max()))[0]:
        w = perm.tolist().index(first + int(i))
        alone, _ = _device(plain.subset([int(i)]))
        assert alone[0][0] == got[0][w] and alone[2][0] == got[2][w], "in-degree %d" % degs[i]


@pytest.mark.gpu
@pytest.mark.parametrize("k", ["4", "8"])
def test_gpu_indegree_ladder_band_layout(k, monkeypatch):
    monkeypatch.setenv("RP_POA_BAND_K", k)
    monkeypatch.setenv("RP_BAND_AUDIT", "1")
    for variant in ("plain", "partial", "tie_repeat"):
        ws, _, want = gpu_ladder(variant)
        stats = {}
        got, _ = _device(ws, banded=True, band_stats=stats)
        check(ws, got, want, what="band k=%s %s" % (k, variant))
        assert stats["band_layout_in_use"] and stats["band_audit_mismatches"] == 0, stats


@pytest.mark.gpu
@pytest.mark.parametrize("banded", [False, True], ids=["full", "band_k8"])
def test_gpu_full_clusters(banded, monkeypatch):
    if banded:
        monkeypatch.setenv("RP_POA_BAND_K", "8")
    ws = windows.from_lists(cluster_windows())
    assert all(s[2] == 7 for s in ob.oracle_graph_shape(ws))
    check(ws, _device(ws, banded=banded)[0], _oracle(ws), what="clusters")


NODE_LAYOUTS = {"full": (False, None, 16), "band_k8": (True, None, 8), "band_k4": (True, "4", 4)}


@pytest.mark.gpu
@pytest.mark.parametrize("window_length,layout", [(500, "full"), (1000, "full"), (1000, "band_k8"), (1000, "band_k4")])
def test_gpu_node_count_ladder(window_length, layout, monkeypatch):
    """Graphs crossing, by one layer, lim.nmax and the Phase D shared-memory count of the full-matrix and of the 32 x 8 /
    32 x 4 bands' kernels: status 0 (the escalation pass takes what the first pass refuses), equal to the oracle in every
    layout (so banded results equal unbanded ones).  Where lim_big.nmax itself cuts off: test_sim_node_budget_is_exact
    (graphs of 24 512+ nodes take over a minute here)."""
    banded, k, band_k = NODE_LAYOUTS[layout]
    if k:
        monkeypatch.setenv("RP_POA_BAND_K", k)
    nmax, nmax_big, smem_full = node_caps(window_length)
    caps = sorted({nmax, smem_full, node_caps(window_length, 8)[2]})
    key = ("nodes", window_length)
    if key not in _gpu_cache:
        wins, nodes = node_ladder(51 + window_length, caps, window_length, reach=2)
        ws = windows.from_lists(wins)
        _gpu_cache[key] = (ws, np.array(nodes), _oracle(ws))
    ws, nodes, want = _gpu_cache[key]
    exp = np.where(nodes > nmax_big, WIN_NODE_LIMIT, 0).astype(np.uint32)
    got, launches = _device(ws, window_length=window_length, banded=banded)
    check(ws, got, want, exp, what="%s w=%d nodes %s" % (layout, window_length, nodes.tolist()))
    assert launches >= 2 and (exp == 0).all()
