"""GPU parity tests (run on an H100): the CUDA path, called through the C ABI, against the oracle,
the committed golden fixtures and the reference's known-answer checksums.  Integer/byte work => bit-exact."""
import json
import os

import numpy as np
import pytest

from oracle import bindings as ob
from racon_b200 import api, windows
from tests import util
from tests.test_oracle import KAT

pytestmark = pytest.mark.gpu

CASES = {
    "fullspan": dict(n=48, wlen=500, depth=32, err=0.12),
    "partial": dict(n=48, wlen=500, depth=30, err=0.10, partial_frac=0.5),
    "partial_qual": dict(n=48, wlen=500, depth=24, err=0.12, partial_frac=0.3, with_qual=True, backbone_qual=True),
    "ngs_short": dict(n=96, wlen=200, depth=40, err=0.01, partial_frac=0.9, with_qual=True, types=0),
    "acgtn": dict(n=32, wlen=300, depth=20, err=0.15, partial_frac=0.2, alphabet=b"ACGTN"),
    "shallow": dict(n=64, wlen=120, depth=3, err=0.2, partial_frac=0.3),
    "higherr": dict(n=32, wlen=300, depth=40, err=0.3),
    "long_layers": dict(n=8, wlen=700, depth=12, err=0.1, partial_frac=0.2),
}


def _mk(name, seed):
    kw = dict(CASES[name])
    n = kw.pop("n")
    t = kw.pop("types", None)
    ws = util.make_set(seed, n, **kw)
    if t is not None:
        ws.win_type[:] = t
    return ws


@pytest.fixture(autouse=True)
def _force_the_band_layout(request, monkeypatch):
    """A banded object only uses the band layout for windows of >= 768 bases (where it is the faster kernel).  The
    `banded` parametrisations below exist to test the band itself, so they ask for it explicitly (256 columns)."""
    if "banded" in getattr(request.node, "callspec", type("x", (), {"params": {}})).params and \
            request.node.callspec.params["banded"] and "RP_POA_BAND_K" not in os.environ:
        monkeypatch.setenv("RP_POA_BAND_K", "8")
    yield


def _compare(ws, scores=(3, -5, -4), trim=True, window_length=500, banded=False, band_stats=None):
    m, x, g = scores
    cons, pol, st, covs = api.consensus(ws, m, x, g, trim=trim, window_length=window_length, want_coverage=True,
                                        banded=banded, band_stats=band_stats)
    ora, opol, _, ocov = ob.oracle_consensus(ws, m, x, g, trim=trim, threads=os.cpu_count() or 4, want_coverage=True)
    assert (st == 0).all(), "device limit statuses: %s" % np.unique(st)
    bad = [w for w in range(ws.n_windows) if cons[w] != ora[w]]
    assert not bad, "consensus differs on windows %s" % bad[:8]
    assert (pol == opol).all()
    for w in range(ws.n_windows):
        if pol[w]:
            assert (covs[w].astype(np.uint32) == ocov[w]).all(), "coverage differs on window %d" % w


@pytest.mark.parametrize("banded", [False, True], ids=["full", "banded"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_gpu_equals_oracle(name, banded):
    """racon -b (banded=True) must return exactly what the full matrix returns: every alignment whose band result the
    device-side check refuses is redone with the full matrix on the device."""
    _compare(_mk(name, seed=101), window_length=1000 if name == "long_layers" else 500, banded=banded)


@pytest.mark.parametrize("banded", [False, True], ids=["full", "banded"])
@pytest.mark.parametrize("scores", [(5, -4, -8), (1, -1, -1)])
def test_gpu_equals_oracle_other_scores(scores, banded):
    _compare(_mk("partial_qual", seed=55), scores=scores, banded=banded)
    _compare(_mk("higherr", seed=56), scores=scores, banded=banded)


@pytest.mark.parametrize("banded", [False, True], ids=["full", "banded"])
@pytest.mark.parametrize("lanes", [8, 16, 32])
def test_gpu_every_group_width(lanes, banded, monkeypatch):
    """The kernel is compiled for 8, 16 and 32 lanes per window (RP_POA_GROUP); all of them, banded or not, are exact."""
    monkeypatch.setenv("RP_POA_GROUP", str(lanes))
    stats = {}
    _compare(_mk("partial", seed=33), banded=banded, band_stats=stats)
    _compare(_mk("fullspan", seed=34), banded=banded, band_stats=stats)
    if banded:
        assert stats["band_alignments"] > 0 and stats["band_width"] == (256 if lanes == 32 else 16 * lanes)


def test_gpu_band_refusals_are_redone_with_the_full_matrix(monkeypatch):
    """Layers with 110-base deletions / 120-base insertions leave a 128-column band: the device-side check must refuse
    those band results (counted), redo them with the full matrix, and the consensus must still equal the oracle's.  A
    margin wider than the band refuses everything."""
    rng = np.random.default_rng(5)
    wins = []
    for _ in range(24):
        truth = bytes(b"ACGT"[i] for i in rng.integers(4, size=500))
        bb = util.mutate(rng, truth, 0.1)[:500]
        win = [(bb, None, 0, 0)]
        for d in range(12):
            r = util.mutate(rng, truth, 0.1)
            if d % 3 == 0:
                r = r[:150] + r[260:]
            if d % 3 == 1:
                r = r[:200] + bytes(b"ACGT"[i] for i in rng.integers(4, size=120)) + r[200:]
            win.append((r, None, 0, len(bb) - 1))
        wins.append(win)
    ws = windows.from_lists(wins)
    monkeypatch.setenv("RP_POA_BAND_K", "4")     # 128-column band
    stats = {}
    _compare(ws, banded=True, band_stats=stats)
    assert 0 < stats["band_redone_full"] < stats["band_alignments"]
    monkeypatch.setenv("RP_BAND_MARGIN", "60")
    stats = {}
    _compare(_mk("fullspan", seed=35), banded=True, band_stats=stats)
    assert stats["band_redone_full"] == stats["band_alignments"] > 0


def test_gpu_no_trim_and_trivial_windows():
    _compare(_mk("partial", seed=9), trim=False)
    tiny = windows.from_lists([[(b"ACGTACGT", None, 0, 0), (b"ACGTTCGT", None, 0, 7)], [(b"AC", None, 0, 0)]])
    cons, pol, st = api.consensus(tiny)
    assert cons == [b"ACGTACGT", b"AC"] and not pol.any() and (st == 0).all()


@pytest.mark.parametrize("banded", [False, True], ids=["full", "banded"])
@pytest.mark.parametrize("err,n,expect", KAT)
def test_gpu_known_answer_checksums_of_the_reference(err, n, expect, banded):
    """FNV-1a-64 over the consensus of the SURVEY.md §8(d) synthetic windows, as produced by the reference."""
    ws, _ = windows.synth_windows(n, err=err)
    cons, pol, st = api.consensus(ws, banded=banded)
    assert (st == 0).all() and pol.all()
    assert "%016x" % windows.fnv1a64(cons) == expect


def test_gpu_matches_golden_fixtures():
    path = os.path.join(os.path.dirname(__file__), "golden", "poa_golden.json")
    gold = json.load(open(path))
    for case in gold["cases"]:
        ws = windows.from_lists([[(s[0].encode(), s[1].encode() if s[1] else None, s[2], s[3]) for s in win]
                                 for win in case["windows"]], case["types"])
        m, x, g = case["scores"]
        cons, pol, st = api.consensus(ws, m, x, g, trim=case["trim"])
        assert [c.decode() for c in cons] == case["consensus"], case["name"]
        assert [bool(p) for p in pol] == case["polished"], case["name"]


def test_gpu_host_mirror_classes():
    """createWindow / add_layer / BatchProcessor (the C++ mirror of the reference interface)."""
    ws = _mk("partial", seed=77)
    cons, pol = api.mirror_consensus(ws)
    ora, opol, _ = ob.oracle_consensus(ws, threads=8)
    assert cons == ora and (pol == opol).all()


def test_gpu_full_size_properties():
    """BASELINE config 2 size (10k windows): determinism, batch-composition independence, and a
    checksum-of-checksums against the oracle on a strided sample (the oracle is too slow for all 10k)."""
    n = 10000
    ws, _ = windows.synth_windows(n, err=0.12)
    cons, pol, st = api.consensus(ws)
    assert (st == 0).all() and pol.all()
    cons2, _, _ = api.consensus(ws)
    assert cons == cons2, "two runs of the same batch differ"
    idx = np.arange(0, n, 40)
    sub = ws.subset(idx)
    cons_sub, _, _ = api.consensus(sub)
    assert cons_sub == [cons[i] for i in idx], "result depends on batch composition"
    ora, _, _ = ob.oracle_consensus(sub, threads=os.cpu_count() or 4)
    assert windows.fnv1a64(cons_sub) == windows.fnv1a64(ora)
    lens = np.array([len(c) for c in cons])
    assert 480 < lens.mean() < 520


def test_gpu_escalation_of_deep_and_long_windows():
    """Windows that outgrow the default per-window limits (3064 nodes / 1023-base layers at w=500) are re-run on
    the GPU with larger limits — never on the CPU — and still match the oracle."""
    deep = util.make_set(5, 3, wlen=500, depth=150, err=0.15)          # > 3064 graph nodes
    long_layers = util.make_set(6, 3, wlen=500, depth=12, err=0.05)
    wins = [deep.window(i) for i in range(3)]
    # one layer much longer than the window (e.g. a large insertion): 1400 bases over a 500-base backbone
    rng = np.random.default_rng(1)
    w0 = long_layers.window(0)
    big = bytes(b"ACGT"[i] for i in rng.integers(4, size=1400))
    w0.append((big, None, 0, len(w0[0][0]) - 1))
    wins.append(w0)
    ws = windows.from_lists(wins)
    cons, pol, st = api.consensus(ws)
    ora, opol, _ = ob.oracle_consensus(ws, threads=os.cpu_count() or 4)
    assert (st == 0).all(), st
    assert cons == ora and (pol == opol).all()


def test_gpu_edge_cases_ragged_and_degenerate():
    bb = b"ACGTTGCAACGTAGCTAGCTAGGATCGATCGATCGTAGCTAGCTAGCATCGATCGTAGCATGCATGCAA"
    wins = [
        [(bb, None, 0, 0), (bb[:40], None, 0, 39), (b"", None, 0, 10), (bb[5:60], None, 5, 59), (b"ACG", None, 7, 7),
         (bb, None, 0, len(bb) - 1)],
        [(bb, None, 0, 0), (b"A", None, 0, 1), (b"T", None, 3, 4), (bb[10:50], b"5" * 40, 10, 49),
         (bb, None, 0, len(bb) - 1)],
        [(bb, None, 0, 0), (b"", None, 0, 5), (bb, None, 0, len(bb) - 1), (b"AC", None, 9, 9)],
        [(b"AC", None, 0, 0), (b"AC", None, 0, 1), (b"AG", None, 0, 1), (b"AC", None, 0, 1)],
        [(b"A", None, 0, 0)],
    ]
    ws = windows.from_lists(wins)
    cons, pol, st = api.consensus(ws)
    ora, opol, _ = ob.oracle_consensus(ws)
    assert cons == ora and (pol == opol).all() and (st == 0).all()
    bad = windows.from_lists([[(bb, None, 0, 0), (bb, None, 12, 5), (bb, None, 0, 60), (bb, None, 0, 60)]])
    with pytest.raises(api.RaconB200Error):
        api.consensus(bad)  # begin > end: RP_ERR_INVALID (the reference exit(1)s, window.cpp:53-58)


def test_gpu_batch_object_protocol():
    """add-until-full / run / fetch / reset, state errors, per-window status."""
    ws = _mk("shallow", seed=3)
    b = api.PoaBatch()
    with pytest.raises(api.RaconB200Error):
        b.launch()  # launch before upload
    took = b.add_window_set(ws)
    assert took == ws.n_windows == b.size()
    b.run()
    b.sync()
    c0, cov0, p0 = b.fetch(0)
    ora, opol, _ = ob.oracle_consensus(ws)
    assert c0 == ora[0] and p0 == bool(opol[0])
    with pytest.raises(api.RaconB200Error):
        b.add_window_set(ws)  # uploaded batch must be reset first
    b.reset()
    assert b.size() == 0
    assert b.add_window(ws.window(1)) == api.RP_OK
    b.run()
    assert b.fetch(0)[0] == ora[1]
    info = b.info()
    assert info["launches"] >= 2 and info["workers"] >= 32
    b.close()


def test_gpu_windows_beyond_spoa_int16_bound():
    """Scores for which spoa's worst-case bound selects its int32 engine (steep gap; or w=1000 with g=-8 at depth 40):
    computed in int16 with the finished matrix verified in range — results equal the oracle's (int32 throughout);
    a matrix that really leaves int16 is reported as RP_WIN_NEEDS_INT32."""
    from racon_b200 import api
    ws = util.make_set(21, 24, wlen=200, depth=16, err=0.12, partial_frac=0.3, with_qual=True)
    cons, pol, st = api.consensus(ws, match=3, mismatch=-5, gap=-60, window_length=200)
    ora, opol, _ = ob.oracle_consensus(ws, 3, -5, -60, window_length=200, threads=8)
    assert (st == 0).all() and cons == ora and (pol == opol).all()
    big = util.make_set(25, 6, wlen=1000, depth=40, err=0.12)
    cons, pol, st = api.consensus(big, match=5, mismatch=-4, gap=-8, window_length=1000)
    ora, opol, _ = ob.oracle_consensus(big, 5, -4, -8, window_length=1000, threads=8)
    assert (st == 0).all() and cons == ora and (pol == opol).all()
    bad = util.make_set(23, 4, wlen=600, depth=5, err=0.1)
    cons, pol, st = api.consensus(bad, match=3, mismatch=-5, gap=-64, window_length=600)
    assert (st == 4).all() and not pol.any()


def test_gpu_memory_budget_back_pressure():
    """createCUDABatch's avail_mem contract (cudabatch.cpp:23-72, cudapolisher.cpp:232-238): an object created with a small
    budget keeps its device allocations inside it, reports RP_BATCH_FULL when the next window would not fit (add-until-full
    -> run -> reset -> continue, cudabatch.cpp:126-132 / cudapolisher.cpp:254-276) and still produces the same consensus."""
    import torch
    n = 2000
    ws, _ = windows.synth_windows(n, err=0.12)
    free0 = torch.cuda.mem_get_info()[0]
    budget = 192 << 20
    b = api.PoaBatch(mem_bytes=budget, window_length=500)
    stride = 1200
    cons, batches, first = [], 0, 0
    peak_used = 0
    while first < n:
        b.reset()
        took = b.add_window_set(ws, first, n - first)
        assert took > 0
        if first + took < n:   # the batch is full: one more window must be refused, not crash
            assert b.add_window(ws.window(first + took)) == api.RP_BATCH_FULL
        b.run()
        b.sync()
        out, lens, pol, st = b.fetch_all(stride)
        assert (st == 0).all()
        cons += [out[i, :lens[i]].tobytes() for i in range(took)]
        peak_used = max(peak_used, free0 - torch.cuda.mem_get_info()[0])
        first += took
        batches += 1
    b.close()
    assert batches >= 3, "a 192 MB object swallowed %d windows in %d batches: the budget is not enforced" % (n, batches)
    assert peak_used <= budget * 1.25 + (64 << 20), "device memory in use %d MB for a %d MB budget" % (peak_used >> 20, budget >> 20)
    ref, _, _ = api.consensus(ws)
    assert cons == ref
    assert "%016x" % windows.fnv1a64(cons[:200]) == "50f18d884e3254d2"


def test_gpu_four_batch_objects_per_gpu_like_racon_c4():
    """racon -c 4: four batch objects on one GPU, each with 0.9 * free / 4 bytes (cudapolisher.cpp:226-240), alive at the
    same time, driven from four host threads."""
    import threading
    import torch
    ws, _ = windows.synth_windows(1200, err=0.12)
    free = torch.cuda.mem_get_info()[0]
    objs = [api.PoaBatch(mem_bytes=int(0.9 * free / 4), window_length=500) for _ in range(4)]
    res = [None] * 4

    def work(k):
        b = objs[k]
        lo, hi = 300 * k, 300 * (k + 1)
        assert b.add_window_set(ws, lo, hi - lo) == hi - lo
        b.run()
        b.sync()
        out, lens, pol, st = b.fetch_all(1200)
        res[k] = ([out[i, :lens[i]].tobytes() for i in range(hi - lo)], st)

    th = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    cons = sum((r[0] for r in res), [])
    assert all((r[1] == 0).all() for r in res)
    for b in objs:
        b.close()
    assert "%016x" % windows.fnv1a64(cons[:200]) == "50f18d884e3254d2"
    ref, _, _ = api.consensus(ws)
    assert cons == ref


def test_gpu_banded_policy_by_window_length():
    """racon -b is a request for speed with unchanged results: for 500-base windows the full matrix is the faster kernel,
    so a banded object does not use the band layout there (and says so); for 1000-base windows it does.  Same consensus
    either way."""
    assert "RP_POA_BAND_K" not in os.environ and "RP_POA_GROUP" not in os.environ
    ws = _mk("fullspan", seed=41)
    stats = {}
    _compare(ws, banded=True, band_stats=stats)
    assert stats["banded"] and not stats["band_layout_in_use"] and stats["band_alignments"] == 0
    big = util.make_set(42, 6, wlen=1000, depth=12, err=0.1, partial_frac=0.2)
    stats = {}
    _compare(big, window_length=1000, banded=True, band_stats=stats)
    assert stats["band_layout_in_use"] and stats["band_alignments"] > 0 and stats["band_width"] == 256
