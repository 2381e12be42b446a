"""What bench.py times, checked window by window and pair by pair: resident batches relaunched on two objects and two caller
streams with an event between them, the aligner launched warmup + steps times over one upload, and the device counters the
roofline's bytes come from (rp_poa_info [5]-[7]) against what the oracle counts on the same windows.

Every comparison covers all windows (or pairs): consensus, polished flag, status and coverage against the oracle, CIGAR,
edit distance, status and breaking points against edlib.  Tests whose name contains `stream` bind torch streams; the rest
also run over the simulated runtime (tools/sim_gpu_tests.sh ... -k "not stream"), where the families are sampled smaller."""
import argparse
import os

import numpy as np
import pytest

import bench
from oracle import bindings as ob
from racon_b200 import api, windows
from tests import test_gpu_edges as ge, util
from tests.test_zz_gpu_resident import _as_store

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 4
# a 500-base window takes seconds on the simulated runtime: there every family keeps its shape at a smaller size
SIMULATED = os.path.basename(os.path.dirname(api.lib_path())).startswith("simapi")
SCORES = (3, -5, -4)


def _size(gpu, sim):
    return sim if SIMULATED else gpu


@pytest.fixture(autouse=True)
def _room_for_the_escalation_pass(monkeypatch):
    """the simulated device reports 4 GB free, too little for the escalation pass's scratch (an H100 has room)"""
    if SIMULATED:
        monkeypatch.setenv("RP_SIM_FREE_MB", "16384")


# ---- helpers --------------------------------------------------------------------------------------------------------------
def oracle_run(ws, scores=SCORES, window_length=500):
    """The oracle's (consensus, polished, _, coverage) and its 12 counters (oracle_poa_stats) over exactly these windows."""
    c = np.zeros(12, np.uint64)
    ob.oracle_lib().oracle_poa_stats(c.ctypes.data)   # reading zeroes them
    want = ob.oracle_consensus(ws, *scores, window_length=window_length, threads=THREADS, want_coverage=True)
    ob.oracle_lib().oracle_poa_stats(c.ctypes.data)
    return want, [int(v) for v in c]


def new_batch(ws=None, scores=SCORES, window_length=500, banded=False, counters=True):
    b = api.PoaBatch(match=scores[0], mismatch=scores[1], gap=scores[2], window_length=window_length, banded=banded)
    if counters:
        b.enable_counters(True)
    if ws is not None:
        assert b.add_window_set(ws) == ws.n_windows
    return b


def results(b, ws):
    """(consensus, polished, status, coverage) of every window of the object's last run"""
    n = ws.n_windows
    out, lens, pol, st = b.fetch_all(int(2 * np.diff(ws.seq_off.astype(np.int64)).max() + 64))
    return [out[w, :lens[w]].tobytes() for w in range(n)], pol, st, [b.fetch(w)[1] for w in range(n)]


def same(a, b):
    return a[0] == b[0] and (a[1] == b[1]).all() and (a[2] == b[2]).all() and \
        all(np.array_equal(x, y) for x, y in zip(a[3], b[3]))


def counts(b):
    i = b.info()
    return [i["alignments"], i["dp_cells"], i["pred_cells"]]


def run_once(ws, **kw):
    b = new_batch(ws, **kw)
    try:
        b.run()
        b.sync()
        return results(b, ws), counts(b), b.info()["launches"], (b.band_info() if kw.get("banded") else None)
    finally:
        b.close()


# ---- a. the counters against the oracle ---------------------------------------------------------------------------------
def _partial(seed):
    return util.make_set(seed, _size(24, 4), wlen=_size(300, 120), depth=_size(12, 6), err=0.12, partial_frac=0.6)


FAMILIES = {
    "grid": lambda: (ge.grid_windows(lengths=ge.GRID[:_size(16, 9)]), SCORES, 500),
    "partial_span": lambda: (_partial(31), SCORES, 500),
    "qualities": lambda: (util.make_set(32, _size(24, 4), wlen=_size(300, 120), depth=_size(12, 6), err=0.12,
                                        partial_frac=0.2, with_qual=True, backbone_qual=True), SCORES, 500),
    "ngs": lambda: (util.make_set(33, _size(24, 3), [0] * _size(24, 3), wlen=_size(200, 100), depth=_size(24, 8), err=0.02,
                                  partial_frac=0.9, with_qual=True), SCORES, 200),
    "scores_0_0_0": lambda: (_partial(34), (0, 0, 0), 500),
    "scores_1_-1_-1": lambda: (_partial(35), (1, -1, -1), 500),
    "scores_5_-4_-8": lambda: (_partial(36), (5, -4, -8), 500),
}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_counters_equal_the_oracle(family):
    ws, scores, wl = FAMILIES[family]()
    want, oc = oracle_run(ws, scores, wl)
    got, c, launches, _ = run_once(ws, scores=scores, window_length=wl)
    ge.check(ws, got, want, what=family)
    assert launches == 1, "a window went through the escalation pass, which the counters leave out"
    assert c == oc[:3], "alignments / DP cells / predecessor cells %s, oracle %s" % (c, oc[:3])


def test_counters_on_a_bench_config2_sample():
    """The roofline's bytes per window (2 B x (DP cells + predecessor cells) / windows) on the first windows of bench config 2
    are the oracle's: 86.2 MB per window on the first 2 000 (the figure DESIGN.md quotes)."""
    ws, _ = bench.make_windows(2, argparse.Namespace(windows=0), 0, 1, sample=_size(2000, 3))
    want, oc = oracle_run(ws)
    got, c, launches, _ = run_once(ws)
    ge.check(ws, got, want, what="config 2")
    assert launches == 1 and c == oc[:3], (c, oc[:3])
    per_window = 2.0 * (c[1] + c[2]) / ws.n_windows
    assert per_window == 2.0 * (oc[1] + oc[2]) / ws.n_windows
    if ws.n_windows == 2000:
        assert round(per_window / 1e6, 1) == 86.2, per_window


def _zero_work_windows(rng, w=500):
    """Windows the first pass counts nothing for, each with its expected status: 1 and 2 sequences (never sent to the
    device), 9 distinct characters (never sent to the device), a backbone over the first pass's node budget (6w + 64) and a
    first layer over its length limit (2w + 23), both finished by the escalation pass, which is not counted."""
    bb = ge._rand(rng, 200)
    out = [([(bb, None, 0, 0)], 0),
           ([(bb, None, 0, 0), (util.mutate(rng, bb, 0.1), None, 0, 199)], 0),
           ([(b"ACGTNRYKM" * 20, None, 0, 0)] + [(b"ACGTNRYKM" * 20, None, 0, 179)] * 3, ge.WIN_ALPHABET_LIMIT)]
    long_bb = ge._rand(rng, 6 * w + 64 + 36)
    win = [(long_bb, None, 0, 0)]
    for b in (100, 1500, 3000):
        win.append((util.mutate(rng, long_bb[b:b + 90], 0.1), None, b, b + 89))
    out.append((win, 0))
    bb = ge._rand(rng, 300)
    first = bb[:150] + ge._rand(rng, 2 * w + 23 + 77 - 300) + bb[150:]    # begins at 0: aligned first
    win = [(bb, None, 0, 0), (first, None, 0, 299)]
    for _ in range(3):
        win.append((util.mutate(rng, bb[5:], 0.1), None, 5, 299))
    out.append((win, 0))
    return out


def test_counters_leave_out_windows_without_first_pass_work():
    rng = np.random.default_rng(41)
    base = util.make_set(42, _size(12, 3), wlen=_size(300, 100), depth=_size(10, 5), err=0.1, partial_frac=0.3)
    extra = _zero_work_windows(rng)
    allw = [base.window(i) for i in range(base.n_windows)] + [w for w, _ in extra]
    want_st = np.array([0] * base.n_windows + [s for _, s in extra], np.uint32)
    perm = np.random.default_rng(43).permutation(len(allw))
    ws = windows.from_lists([allw[i] for i in perm], [1] * len(allw))
    want_st = want_st[perm]
    want, _ = oracle_run(ws)
    _, oc = oracle_run(base)
    got, c, launches, _ = run_once(ws)
    ge.check(ws, got, want, want_st, what="mixed with zero-work windows")
    assert launches == 2, "the over-limit windows did not go through the escalation pass"
    assert c == oc[:3], "alignments / DP cells / predecessor cells %s, oracle over the other windows %s" % (c, oc[:3])


def test_counters_count_the_last_launch():
    """run twice, upload + N launches + download, reset + another batch, counters off then on: each reports the numbers of
    its own last launch, the oracle's for those windows."""
    ws = _partial(51)
    ws2 = util.make_set(52, _size(10, 3), wlen=_size(250, 90), depth=_size(9, 5), err=0.12, partial_frac=0.3)
    want, oc = oracle_run(ws)
    want2, oc2 = oracle_run(ws2)
    b = new_batch(ws, counters=False)
    try:
        b.run()
        b.sync()
        assert counts(b) == [0, 0, 0]
        first = results(b, ws)
        ge.check(ws, first, want, what="counters off")
        b.enable_counters(True)
        seen = []
        for _ in range(2):
            b.run()
            b.sync()
            seen.append(counts(b))
            assert same(results(b, ws), first)
        b.upload()
        for _ in range(3):
            b.launch()
        b.download()
        b.sync()
        seen.append(counts(b))
        assert same(results(b, ws), first)
        assert seen == [oc[:3]] * 3, "per launch %s, oracle %s" % (seen, oc[:3])
        b.reset()
        assert b.add_window_set(ws2) == ws2.n_windows
        b.run()
        b.sync()
        assert counts(b) == oc2[:3]
        ge.check(ws2, results(b, ws2), want2, what="after reset")
        b.enable_counters(False)
        b.run()
        b.sync()
        assert counts(b) == [0, 0, 0]
        b.enable_counters(True)
        b.run()
        b.sync()
        assert counts(b) == oc2[:3]
    finally:
        b.close()


def _band_width(k):
    return 32 * int(k)


@pytest.mark.parametrize("k", ["8", "4"], ids=["band_k8", "band_k4"])
def test_band_counters_on_layers_too_short_for_the_band(k, monkeypatch):
    """Every layer shorter than the band: nothing is tried in it, and the counters are the full matrix's."""
    monkeypatch.setenv("RP_POA_BAND_K", k)
    width = _band_width(k)
    ws = util.make_set(61, _size(16, 3), wlen=width * 3 // 4, depth=_size(10, 5), err=0.1, partial_frac=0.3)
    assert np.diff(ws.seq_off.astype(np.int64)).max() < width
    want, oc = oracle_run(ws)
    got, c, launches, bi = run_once(ws, banded=True)
    ge.check(ws, got, want, what="short layers, band %d" % width)
    assert bi["band_layout_in_use"] and bi["band_width"] == width and bi["band_alignments"] == 0, bi
    assert launches == 1 and c == oc[:3], (c, oc[:3])


@pytest.mark.parametrize("k", ["8", "4"], ids=["band_k8", "band_k4"])
def test_band_counters_when_every_alignment_stays_in_the_band(k, monkeypatch):
    """Every alignment accepted inside the band: each row of the DP counts the band's width of cells, and so does each
    predecessor row."""
    monkeypatch.setenv("RP_POA_BAND_K", k)
    width = _band_width(k)
    ws = util.make_set(62, _size(12, 2), wlen=500, depth=_size(10, 4), err=0.03)
    want, oc = oracle_run(ws)
    got, c, launches, bi = run_once(ws, banded=True)
    ge.check(ws, got, want, what="band %d" % width)
    assert bi["band_width"] == width and bi["band_alignments"] == oc[0] and bi["band_redone_full"] == 0, bi
    rows = sum(int((r[:, 1] + 1).sum()) for r in ob.oracle_matrix_ranges(ws))
    assert launches == 1 and c == [oc[0], width * rows, width * oc[11]], (c, oc)


@pytest.mark.parametrize("k", ["8", "4"], ids=["band_k8", "band_k4"])
def test_band_counters_when_alignments_are_redone(k, monkeypatch):
    """Layers with deletions and insertions as wide as the band: some band results are refused and redone with the full
    matrix.  Every alignment is still counted once, and no more cells than the full matrix's."""
    monkeypatch.setenv("RP_POA_BAND_K", k)
    width = _band_width(k)
    rng = np.random.default_rng(63)
    wins = []
    for _ in range(_size(4, 1)):
        truth = ge._rand(rng, 600)
        bb = util.mutate(rng, truth, 0.08)[:600]
        win = [(bb, None, 0, 0)]
        for d in range(_size(9, 4)):
            r = util.mutate(rng, truth, 0.08)
            if d % 3 == 0:
                r = r[:150] + r[150 + width:]
            elif d % 3 == 1:
                r = r[:200] + ge._rand(rng, width) + r[200:]
            win.append((r, None, 0, len(bb) - 1))
        wins.append(win)
    ws = windows.from_lists(wins)
    want, oc = oracle_run(ws, window_length=1000)
    got, c, launches, bi = run_once(ws, banded=True, window_length=1000)
    ge.check(ws, got, want, what="band %d, refusals" % width)
    assert bi["band_width"] == width and 0 < bi["band_redone_full"] <= bi["band_alignments"], bi
    assert launches == 1 and c[0] == oc[0] and c[1] <= oc[1] and c[2] <= oc[2], (c, oc[:3])


# ---- b. resident relaunches, shaped like bench.py ------------------------------------------------------------------------
def _relaunch_case(variant):
    """(windows, expected statuses, banded, by-reference store pieces or None)"""
    if variant == "mixed":
        if SIMULATED:   # the small kinds, and one window for the escalation pass
            ws, st = ge.other_windows()
            keep = [0, 1, 2, 3, 4, 5, 8]
            return ws.subset(keep), st[keep], False, None
        ws, st = ge.mixed_batch()
        return ws, st, False, None
    ws = util.make_set(71, _size(32, 3), wlen=_size(500, 300), depth=_size(16, 6), err=0.12, partial_frac=0.2,
                       with_qual=True)
    return ws, np.zeros(ws.n_windows, np.uint32), variant == "band", (_as_store(ws, 72) if variant == "by_reference" else None)


def _relaunch_parity(variant, streams, monkeypatch, launches=4):
    """Run A once; then, like bench.py, upload two objects, launch each once, and alternate `launches` launches between
    them (on two caller streams: the second waits for an event on the first, and the first for one on the second).  After
    download + sync both must equal A, and A the oracle."""
    if variant == "band":
        monkeypatch.setenv("RP_POA_BAND_K", "8")
    ws, want_st, banded, store_case = _relaunch_case(variant)
    want, _ = oracle_run(ws)
    torch = None
    if streams:
        torch = pytest.importorskip("torch")
        if not torch.cuda.is_available():
            pytest.skip("binding caller streams needs torch.cuda")
    store = api.ReadStore(store_case[0], store_case[1]) if store_case else None
    objs = []
    try:
        for _ in range(2):
            b = new_batch(None if store else ws, banded=banded, counters=False)
            if store:
                for w in range(ws.n_windows):
                    assert b.add_window_refs(store, store_case[2][w], window_type=int(ws.win_type[w])) == api.RP_OK
            objs.append(b)
        a, b2 = objs
        s1 = s2 = None
        if streams:
            s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
            a.set_stream(s1.cuda_stream)
            b2.set_stream(s2.cuda_stream)
        a.run()
        a.sync()
        first = results(a, ws)
        ge.check(ws, first, want, want_st, what=variant)
        band_first = a.band_info() if banded else None
        if banded:
            assert band_first["band_layout_in_use"] and band_first["band_alignments"] > 0, band_first
        a.upload()
        a.launch()
        b2.upload()
        b2.launch()
        if streams:
            ev0, evb = torch.cuda.Event(), torch.cuda.Event()
            ev0.record(s1)
            s2.wait_event(ev0)
        for k in range(launches):
            (a if k % 2 == 0 else b2).launch()
        if streams:
            evb.record(s2)
            s1.wait_event(evb)
        for b in objs:
            b.download()
        for b in objs:
            b.sync()
        for name, b in (("A relaunched", a), ("B", b2)):
            got = results(b, ws)
            assert same(got, first), "%s: %s differs from the first run" % (variant, name)
            if banded:
                bi = b.band_info()
                assert (bi["band_alignments"], bi["band_redone_full"]) == \
                    (band_first["band_alignments"], band_first["band_redone_full"]), (name, bi, band_first)
        if variant == "mixed":
            # first run + its escalation pass, the warm-up launch, its share of the alternation, the escalation pass again
            assert a.info()["launches"] == 2 + 1 + launches // 2 + 1, "the escalation pass did not run after the relaunch"
    finally:
        for b in objs:
            b.close()
        if store:
            store.close()
        if streams:
            torch.cuda.synchronize()


VARIANTS = ["full", "band", "by_reference", "mixed"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_relaunch_parity(variant, monkeypatch):
    _relaunch_parity(variant, False, monkeypatch)


@pytest.mark.parametrize("variant", VARIANTS)
def test_relaunch_parity_on_two_streams(variant, monkeypatch):
    _relaunch_parity(variant, True, monkeypatch)


# ---- c. the timed launches do all the work the value counts --------------------------------------------------------------
@pytest.mark.parametrize("config", [2, 3, 4])
def test_bench_config_windows_finish_in_the_first_pass(config):
    cfg = bench.CONFIGS[config]
    ws, _ = bench.make_windows(config, argparse.Namespace(windows=0), 0, 1, sample=_size(1000, 3))
    want, _ = oracle_run(ws, window_length=cfg["wl"])
    got, _, launches, _ = run_once(ws, window_length=cfg["wl"], banded=cfg["banded"])
    assert launches == 1 and (got[2] == 0).all(), "config %d: statuses %s" % (config, np.unique(got[2]))
    ge.check(ws, got, want, what="config %d" % config)


# ---- d. the aligner's timed path ---------------------------------------------------------------------------------------
MAX_LEN = 20000
RP_ALN_BAND_LIMIT, RP_ALN_ALPHABET_LIMIT, RP_ALN_TOO_LONG = 1, 2, 6
COMP = bytes.maketrans(b"ACGT", b"TGCA")


def _aln_cases(seed=81):
    """(query, target, expected status): 10-kb pairs at 12 % error, short pairs, and one pair for each soft status"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(_size(6, 1)):
        t = ge._rand(rng, int(rng.integers(9000, 11000)))
        out.append((util.mutate(rng, t, 0.12), t, 0))
    for n in rng.integers(1, 400, size=_size(40, 6)):
        t = ge._rand(rng, int(n))
        out.append((util.mutate(rng, t, 0.12) or t[:1], t, 0))
    if not SIMULATED:   # 16 385 rows of band: too slow for the simulated runtime
        out.append((b"A" * 16385, b"C" * 16385, RP_ALN_BAND_LIMIT))
    t = ge._rand(rng, 300)
    out.append((t[:100] + bytes(range(0x61, 0x61 + 17)) + t[100:], t, RP_ALN_ALPHABET_LIMIT))
    t = ge._rand(rng, MAX_LEN + 1)
    out.append((t[:500], t, RP_ALN_TOO_LONG))
    perm = np.random.default_rng(seed + 1).permutation(len(out))
    return [out[i] for i in perm]


def _expected(q, t):
    c, d = ob.ref_edlib_cigar(q, t) if ob.have_ref() else ob.oracle_myers_cigar(q, t)
    return c.encode(), d


def _aln_add(b, mode, cases, store, refs):
    for k, (q, t, _) in enumerate(cases):
        if mode == "by_reference":
            assert b.add_ref(store, *refs[k])
        else:
            assert b.add(q, t, t_begin=refs[k][5], q_start=refs[k][1])


def _aln_store(cases, seed):
    """every pair hidden in two stored 'reads'; the queries of ACGT pairs stored as reverse complements every other pair"""
    rng = np.random.default_rng(seed)
    reads, refs = [], []
    for k, (q, t, _) in enumerate(cases):
        pre_q, pre_t = ge._rand(rng, int(rng.integers(0, 50))), ge._rand(rng, int(rng.integers(0, 300)))
        stored = pre_q + q + ge._rand(rng, 20)
        rev = k % 2 == 1 and set(q) <= set(b"ACGT")
        if rev:
            stored = stored.translate(COMP)[::-1]
        reads += [pre_t + t + b"GATTACA", stored]
        refs.append((2 * k + 1, len(pre_q), len(q), int(rev), 2 * k, len(pre_t), len(t)))
    return reads, refs


def _breaking_points(b, mode, n):
    if mode == "pointer":     # no window length: none computed
        return [np.zeros((0, 2), np.uint32)] * n
    return [b.fetch_breaking_points(i) for i in range(n)]


def _aln_timed(mode, cases, store, refs, stream, warmup=3, steps=5):
    """time_aligner's shape: (caller stream,) upload, warmup + steps launches, download, sync"""
    b = api.AlnBatch(max_len=MAX_LEN)
    try:
        if stream is not None:
            b.set_stream(stream.cuda_stream)
        if mode != "pointer":
            b.set_window_length(500)
        _aln_add(b, mode, cases, store, refs)
        b.upload()
        for _ in range(warmup + steps):
            b.launch()
        b.download()
        b.sync()
        return [b.fetch(i) for i in range(len(cases))], _breaking_points(b, mode, len(cases)), b.info()["launches"]
    finally:
        b.close()


def _aln_single_run(mode, cases, store, refs):
    b = api.AlnBatch(max_len=MAX_LEN)
    try:
        if mode != "pointer":
            b.set_window_length(500)
        _aln_add(b, mode, cases, store, refs)
        b.run()
        b.sync()
        return [b.fetch(i) for i in range(len(cases))], _breaking_points(b, mode, len(cases))
    finally:
        b.close()


def _aligner_timed_path(mode, streams):
    torch = None
    if streams:
        torch = pytest.importorskip("torch")
        if not torch.cuda.is_available():
            pytest.skip("binding a caller stream needs torch.cuda")
    cases = _aln_cases()
    reads, refs = _aln_store(cases, 82)
    store = api.ReadStore(reads) if mode == "by_reference" else None
    try:
        stream = torch.cuda.current_stream() if streams else None
        got, bps, launches = _aln_timed(mode, cases, store, refs, stream)
        once, once_bps = _aln_single_run(mode, cases, store, refs)
    finally:
        if store:
            store.close()
    assert launches >= 8
    assert got == once, "the relaunched batch differs from a single run"
    assert all(np.array_equal(x, y) for x, y in zip(bps, once_bps))
    # edlib on every pair where the reference is built; its restatement on the short pairs and two long ones elsewhere
    n_long = 0
    for k, ((q, t, st_want), (cig, dist, st)) in enumerate(zip(cases, got)):
        assert st == st_want, (k, len(q), len(t), st)
        if st:
            assert cig == b"" and len(bps[k]) == 0, k
            continue
        if not ob.have_ref() and len(t) > 1000:
            n_long += 1
            if n_long > 2:
                continue
        assert (cig, dist) == _expected(q, t), (k, len(q), len(t), dist)
        if mode != "pointer":
            tb, qs = refs[k][5], refs[k][1]
            assert np.array_equal(bps[k], ob.oracle_breaking_points(cig, tb, tb + len(t), qs, 500)), k


ALN_MODES = ["pointer", "breaking_points", "by_reference"]


@pytest.mark.parametrize("mode", ALN_MODES)
def test_aligner_timed_path(mode):
    _aligner_timed_path(mode, False)


@pytest.mark.parametrize("mode", ALN_MODES)
def test_aligner_timed_path_on_a_caller_stream(mode):
    _aligner_timed_path(mode, True)
