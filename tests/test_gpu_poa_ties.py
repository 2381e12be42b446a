"""The POA kernel on tie-rich windows, window by window against the int32 oracle.  spoa's consensus is decided by its tie
rules as much as by its scores:

  1. traceback, diagonal step: predecessors are tried in in-edge order, the first that explains the cell wins;
  2. traceback, other steps: the vertical step over the predecessors before the horizontal one;
  3. sink choice: among equal best scores in the last column, the first sink in rank order;
  4. heaviest bundle, per node: equal edge weights go to the tail when scores[pred] <= scores[tail];
  5. heaviest bundle, best node: the strict maximum keeps the first best node in rank order.

Uniform random bases with phred 5-40 qualities reach these rules only by accident.  The generators below make windows
where they decide the output: homopolymer runs with run-length errors (the dominant error of nanopore reads), tandem
repeats whose layers gain or lose whole units, two-letter and one-letter sequence, and partial-span layers that begin and
end inside a repeat (the Subgraph path); with no qualities, one flat quality per window, every weight 0 ('!'), every
weight 93 ('~') or random qualities, each with and without backbone qualities.

Every window set proves that it reaches the rules: the oracle counts sink ties and branch completions on it, and for every
rule, the oracle with that one rule flipped (oracle_poa_set_tie_rules, tests only) changes the consensus of at least one
window.  A kernel that broke a tie another way would fail these windows.

The generators are plain functions.  Small windows also run through the CPU warp simulation of the same device code
(`test_sim_*`), which needs no GPU; the oracle's answers on one seed of each generator are pinned to those of the
unmodified reference in tests/golden/ref_answers.json (`test_oracle_pinned_*`)."""
import os

import numpy as np
import pytest

from oracle import bindings as ob
from racon_b200 import windows
from tests import test_gpu_edges as te
from tests import util

THREADS = os.cpu_count() or 4
SCORES = [(3, -5, -4), (5, -4, -8), (1, -1, -1), (0, 0, 0), (1, 0, -1), (2, 3, -1), (-1, -2, -3)]
QUAL_MODES = ["none", "flat", "zero", "max", "random"]
RULES = ob.TIE_RULES


# ---- sequence ------------------------------------------------------------------------------------------------------------
def _runs(s):
    """run-length encoding: [(base, length), ...]"""
    out = []
    for c in s:
        if out and out[-1][0] == c:
            out[-1][1] += 1
        else:
            out.append([c, 1])
    return out


def _run_length_errors(rng, s, p=0.3, subst=0.02):
    """each homopolymer run of s grows or shrinks by 1 or 2 bases with probability p (never below 1), then substitutions"""
    out = bytearray()
    for c, n in _runs(s):
        if rng.random() < p:
            n = max(1, n + int(rng.choice([-2, -1, 1, 2])))
        out += bytes([c]) * n
    return te._subst(rng, bytes(out), subst)


def homopolymer_truth(rng, n):
    """runs of 1-12 bases, each base other than the one before"""
    out = bytearray()
    prev = -1
    while len(out) < n:
        b = int(rng.integers(3))
        b = b + 1 if b >= prev >= 0 else b
        out += bytes([util.BASES[b]]) * int(rng.integers(1, 13))
        prev = b
    return bytes(out[:n])


def tandem_structure(rng, n):
    """[(spacer, unit, copies)] of about n bases: units of 1-6 bases repeated 2-12 times between random spacers of 0-8"""
    segs, total = [], 0
    while total < n:
        sp = te._rand(rng, int(rng.integers(0, 9)))
        unit = te._rand(rng, int(rng.integers(1, 7)))
        k = int(rng.integers(2, 13))
        segs.append((sp, unit, k))
        total += len(sp) + len(unit) * k
    return segs


def tandem_render(rng, segs, p=0.0):
    """the repeats with each copy number changed by 1 or 2 whole units with probability p (at least one copy stays)"""
    out = bytearray()
    for sp, unit, k in segs:
        if rng.random() < p:
            k = max(1, k + int(rng.choice([-2, -1, 1, 2])))
        out += sp + unit * k
    return bytes(out)


# ---- windows: [(bases, None, begin, end), ...]; qualities come later (with_quals) ---------------------------------------------
def _ragged(rng, s):
    """a layer's ends as a window cuts them: up to 3 bases lost or foreign bases gained at each end"""
    a, b = int(rng.integers(-3, 4)), int(rng.integers(-3, 4))
    s = s[max(0, -a):len(s) - max(0, -b)]
    return te._rand(rng, max(0, a)) + s + te._rand(rng, max(0, b))


def _window(rng, bb, layers):
    return [(bb, None, 0, 0)] + [(l, None, 0, len(bb) - 1) for l in (_ragged(rng, l) for l in layers) if l]


def homopolymer_window(rng, wlen, depth):
    truth = homopolymer_truth(rng, wlen)
    bb = _run_length_errors(rng, truth)[:wlen]
    return _window(rng, bb, [_run_length_errors(rng, truth) for _ in range(depth)])


def tandem_window(rng, wlen, depth):
    segs = tandem_structure(rng, wlen)
    bb = tandem_render(rng, segs, 0.3)[:wlen]
    return _window(rng, bb, [te._subst(rng, tandem_render(rng, segs, 0.3), 0.01) for _ in range(depth)])


def two_letter_window(rng, wlen, depth):
    ab = b"AT" if rng.random() < 0.5 else b"CG"
    truth = te._rand(rng, wlen, ab)
    bb = util.mutate(rng, truth, 0.08, ab)[:wlen] or truth[:1]
    return _window(rng, bb, [util.mutate(rng, truth, 0.08, ab) for _ in range(depth)])


def one_base_window(rng, wlen, depth):
    """a single repeated base; the layers differ in length only, so every alignment ties"""
    c = bytes([util.BASES[int(rng.integers(4))]])
    d = max(2, wlen // 20)
    return [(c * wlen, None, 0, 0)] + [(c * int(wlen + rng.integers(-d, d + 1)), None, 0, wlen - 1) for _ in range(depth)]


def _inside_run(bb, lo, hi, rng):
    """a position in [lo, hi) with the same base on both sides (inside a homopolymer run or a one-base repeat), or any"""
    cand = [k for k in range(max(1, lo), min(hi, len(bb) - 1)) if bb[k - 1] == bb[k] == bb[k + 1]]
    return int(rng.choice(cand)) if cand else int(rng.integers(lo, hi))


def partial_window(rng, wlen, depth):
    """homopolymer or tandem-repeat sequence; all but two layers are partial-span pieces of the backbone whose begin and
    end fall inside a run, so they are aligned to a subgraph"""
    truth = homopolymer_truth(rng, wlen) if rng.random() < 0.5 else tandem_render(rng, tandem_structure(rng, wlen))
    bb = _run_length_errors(rng, truth)[:wlen]
    win = _window(rng, bb, [_run_length_errors(rng, truth) for _ in range(2)])
    n = len(bb)
    for _ in range(depth - 2):
        b = _inside_run(bb, 0, n // 2, rng)
        e = _inside_run(bb, max(b + 8, n // 2), n - 1, rng)
        piece = _run_length_errors(rng, bb[b:e + 1])
        if piece:
            win.append((piece, None, b, e))
    return win


KINDS = {"homopolymer": homopolymer_window, "tandem": tandem_window, "two_letter": two_letter_window,
         "one_base": one_base_window, "partial": partial_window}


def _quals(rng, n, mode, flat):
    if mode == "flat":
        return bytes([33 + flat]) * n
    if mode == "zero":
        return b"!" * n
    if mode == "max":
        return b"~" * n
    return util.rand_qual(rng, n, 0, 60)


def with_quals(rng, win, mode, backbone):
    """qualities of one mode on the layers ("none": no qualities) and, with `backbone`, on the backbone too (random ones
    when the layers have none)"""
    flat = int(rng.integers(0, 94))
    out = []
    for k, (b, _, beg, end) in enumerate(win):
        if k == 0:
            q = _quals(rng, len(b), "random" if mode == "none" else mode, flat) if backbone else None
        else:
            q = None if mode == "none" else _quals(rng, len(b), mode, flat)
        out.append((b, q, beg, end))
    return out


def tie_set(kind, seed, wlen=500, depth=10, modes=QUAL_MODES):
    """windows of one kind for every quality mode (three flat-quality ones, one of each other mode), with and without
    backbone qualities, window types alternating (NGS, TGS): (window set, quality mode of each window)"""
    rng = np.random.default_rng(seed)
    wins, types, qm = [], [], []
    for mode in modes:
        for bq in (False, True):
            for _ in range(3 if mode == "flat" else 1):
                wins.append(with_quals(rng, KINDS[kind](rng, wlen, depth), mode, bq))
                types.append(1 - len(wins) % 2)
                qm.append(mode)
    return windows.from_lists(wins, types), qm


KIND_SEEDS = {k: 100 * (i + 1) for i, k in enumerate(sorted(KINDS))}


def kind_set(kind, wlen, depth=10):
    """one seeded set of a kind at a window length: (window set, quality mode of each window)"""
    return tie_set(kind, KIND_SEEDS[kind] + wlen, wlen=wlen, depth=depth)


def all_kinds(wlen, depth=10):
    """the sets of every kind at one window length, as one window set"""
    sets = [kind_set(k, wlen, depth)[0] for k in sorted(KINDS)]
    return windows.from_lists([s.window(w) for s in sets for w in range(s.n_windows)],
                              [int(t) for s in sets for t in s.win_type])


# ---- how a set reaches the rules ----------------------------------------------------------------------------------------------
# What a kind cannot reach, and why.  Every path through a one-letter graph spells the same letters and ends in its one
# sink, so only the length of the heaviest path shows, and only the best-node rule on zero-weight edges moves it: the other
# rules and the sink ties are checked to decide nothing there (should they start to, they belong to the reached ones).
UNREACHED = {"one_base": {"first_in_edge_diagonal", "vertical_before_horizontal", "first_tied_sink", "bundle_tie_le",
                          "sink_ties", "first_best_node/flat"}}


def oracle_stats(ws, scores=(3, -5, -4), trim=True):
    """the oracle's answer (consensus, polished, seconds, coverage) with spoa's rules, and its counters over that one run:
    (answer, sink ties, branch completions, subgraph alignments)"""
    lib = ob.oracle_lib()
    st = np.zeros(12, np.uint64)
    lib.oracle_poa_stats(st.ctypes.data)
    want = ob.oracle_consensus(ws, *scores, trim=trim, threads=THREADS, want_coverage=True)
    lib.oracle_poa_stats(st.ctypes.data)
    return want, int(st[3]), int(st[6]), int(st[5])


def reach(ws, qmodes, scores_list):
    """the oracle's answers per score set, and what the set reaches over all of them: {"sink_ties": n,
    "branch_completions": n, "subgraph": n, rule: [(scores, window) whose consensus changes with that rule flipped],
    "first_best_node/flat" and "/zero": the same on the flat-quality and the zero-weight windows}"""
    answers = {}
    got = {"sink_ties": 0, "branch_completions": 0, "subgraph": 0}
    got.update({name: [] for name in RULES})
    for scores in scores_list:
        want, t, c, s = oracle_stats(ws, scores)
        answers[scores] = want
        got["sink_ties"] += t
        got["branch_completions"] += c
        got["subgraph"] += s
        for name, bit in RULES.items():
            alt = ob.oracle_consensus_with_tie_rules(ws, bit, *scores, threads=THREADS)[0]
            got[name] += [(scores, w) for w in range(ws.n_windows) if alt[w] != want[0][w]]
    for mode in ("flat", "zero"):
        got["first_best_node/" + mode] = [(sc, w) for sc, w in got["first_best_node"] if qmodes[w] == mode]
    return answers, got


def assert_reaches_rules(kind, ws, qmodes, scores_list):
    """sink ties and branch completions happen (and subgraph alignments, for partial-span layers); flipping any one tie
    rule changes the consensus of some window under one of the score sets, and the best-node rule does so on the
    flat-quality and on the zero-weight windows too.  Returns the oracle's answers per score set."""
    answers, got = reach(ws, qmodes, scores_list)
    unreached = UNREACHED.get(kind, set())
    need = ["sink_ties", "branch_completions"] + list(RULES) + ["first_best_node/flat", "first_best_node/zero"]
    if kind == "partial":
        need.append("subgraph")
    missed = [k for k in need if k not in unreached and not got[k]]
    assert not missed, "%s windows do not reach %s: flipping a rule changes no consensus, or the counter stays 0" % (
        kind, missed)
    moved = [k for k in unreached if got[k]]
    assert not moved, "%s windows now reach %s, listed as unreachable for them" % (kind, moved)
    return answers


# ---- checks ---------------------------------------------------------------------------------------------------------------------
WLENS = (500, 1000)
_oracle_cache = {}


def oracle(wlen, scores=(3, -5, -4)):
    """the oracle's answer on all_kinds(wlen)"""
    k = (wlen, scores)
    if k not in _oracle_cache:
        _oracle_cache[k] = ob.oracle_consensus(all_kinds(wlen), *scores, threads=THREADS, want_coverage=True)
    return _oracle_cache[k]


@pytest.mark.parametrize("wlen", WLENS)
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_tie_sets_reach_every_rule(kind, wlen):
    """the device's window sets, on the oracle alone: each kind reaches the tie rules under the score sets it runs with"""
    ws, qm = kind_set(kind, wlen)
    assert_reaches_rules(kind, ws, qm, SCORES)


@pytest.mark.skipif(not ob.have_ref(), reason="oracle/_ref not built")
@pytest.mark.parametrize("wlen", WLENS)
def test_oracle_equals_reference_on_tie_sets(wlen):
    ws = all_kinds(wlen)
    for scores in SCORES:
        ref = ob.ref_consensus(ws, *scores, window_length=wlen, threads=THREADS)
        want = oracle(wlen, scores)
        bad = [w for w in range(ws.n_windows) if ref[0][w] != want[0][w] or ref[1][w] != want[1][w]]
        assert not bad, "oracle != reference at %s on windows %s" % (scores, bad[:8])


# ---- the oracle pinned to the reference's stored answers --------------------------------------------------------------------
def pinned_case(kind):
    """the set of one seed of each generator whose answers tests/golden/ref_answers.json holds, at every score set"""
    ws, _ = tie_set(kind, 7, wlen=300, depth=10)
    return lambda consensus, scores: consensus(ws, *scores, threads=THREADS)[:2]


def pinned_key(kind, scores):
    return "ties/%s/%d,%d,%d" % ((kind,) + scores)


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_oracle_pinned_on_tie_sets(kind):
    answers = util.ref_answers()["poa"]
    case = pinned_case(kind)
    for scores in SCORES:
        want = answers[pinned_key(kind, scores)]
        got = util.consensus_answer(*case(ob.oracle_consensus, scores))
        assert len(got) == len(want)
        bad = [w for w, (a, b) in enumerate(zip(got, want)) if a != b]
        assert not bad, "oracle != reference at %s on windows %s" % (scores, bad[:5])
        if ob.have_ref():
            assert util.consensus_answer(*case(ob.ref_consensus, scores)) == want


# ---- CPU twins: small windows through the warp simulation of the device code ------------------------------------------------
SIM_SCORES = [(3, -5, -4), (1, -1, -1), (0, 0, 0), (2, 3, -1)]
SIM_LAYOUTS = {   # layout: the score sets it runs with (the simulation takes its time)
    "full": ({}, SIM_SCORES),
    "band_32x4": (dict(lanes=32, smem=9216, banded=1, band_cols_per_lane=4, debug_flags=2), SIM_SCORES[::2]),
    "hbm_bundle": (dict(debug_flags=1), SIM_SCORES[1::2]),   # the heaviest bundle over int64 scores in HBM
}


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_sim_tie_windows(kind):
    """150-base windows, depth 8, every quality mode: equal to the oracle in the full matrix, the 128-column band (audited)
    and the HBM bundle; the set reaches the tie rules under the same score sets"""
    ws, qm = tie_set(kind, KIND_SEEDS[kind] + 7, wlen=150, depth=8)
    answers = assert_reaches_rules(kind, ws, qm, SIM_SCORES)
    for name, (kw, scores_list) in SIM_LAYOUTS.items():
        for scores in scores_list:
            got, stats = te.sim(ws, scores, **kw)
            te.check(ws, got, answers[scores], what="sim %s %s %s" % (kind, name, scores))
            if kw.get("banded"):
                assert stats[4] > 0 and stats[6] == 0, stats


def test_sim_tie_windows_band_256():
    """the 256-column band (32 lanes x 8 columns, audited) takes reads of 256 bases and more: 300-base windows of every
    kind"""
    ws = windows.from_lists([w for k in sorted(KINDS) for w in (lambda s: [s.window(i) for i in (0, 3, 4, 7)])(
        tie_set(k, KIND_SEEDS[k] + 9, wlen=300, depth=8)[0])])
    for scores in ((3, -5, -4), (0, 0, 0)):
        want = ob.oracle_consensus(ws, *scores, threads=THREADS, want_coverage=True)
        got, stats = te.sim(ws, scores, lanes=32, smem=9216, banded=1, band_cols_per_lane=8, debug_flags=2)
        te.check(ws, got, want, what="sim band 256 %s" % (scores,))
        assert stats[4] > 0 and stats[6] == 0, stats


# ---- on the device ------------------------------------------------------------------------------------------------------------
def _device(ws, scores=(3, -5, -4), window_length=500, banded=False, band_stats=None):
    from racon_b200 import api
    return api.consensus(ws, *scores, window_length=window_length, want_coverage=True, banded=banded,
                         band_stats=band_stats)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(te.BAND_MODES))
@pytest.mark.parametrize("wlen", WLENS)
def test_gpu_tie_windows(wlen, mode, monkeypatch):
    """every kind, quality mode and score set in the full matrix and the band layouts (audited)"""
    banded, k = te.BAND_MODES[mode]
    if k:
        monkeypatch.setenv("RP_POA_BAND_K", k)
    monkeypatch.setenv("RP_BAND_AUDIT", "1")
    ws = all_kinds(wlen)
    stats = {}
    for scores in SCORES:
        got = _device(ws, scores, window_length=wlen, banded=banded, band_stats=stats)
        te.check(ws, got, oracle(wlen, scores), what="%s w=%d %s" % (mode, wlen, scores))
    if banded and (k or wlen == 1000):
        assert stats["band_layout_in_use"] and stats["band_alignments"] > 0, stats
        assert stats["band_audit_mismatches"] == 0, stats


@pytest.mark.gpu
@pytest.mark.parametrize("banded", [False, True], ids=["full", "banded"])
@pytest.mark.parametrize("lanes", [8, 16])
def test_gpu_tie_windows_group_widths(lanes, banded, monkeypatch):
    """8- and 16-lane groups; 8 lanes only at window length 500 (their shared memory holds the rank update of graphs up
    to about 1 780 nodes)"""
    monkeypatch.setenv("RP_POA_GROUP", str(lanes))
    monkeypatch.setenv("RP_BAND_AUDIT", "1")
    for wlen in WLENS[:1] if lanes == 8 else WLENS:
        ws = all_kinds(wlen)
        for scores in SCORES:
            stats = {}
            got = _device(ws, scores, window_length=wlen, banded=banded, band_stats=stats)
            te.check(ws, got, oracle(wlen, scores), what="%d lanes w=%d %s" % (lanes, wlen, scores))
            if banded:
                assert stats["band_audit_mismatches"] == 0, stats


def _same(a, b, wa, wb):
    return a[0][wa] == b[0][wb] and a[1][wa] == b[1][wb] and a[2][wa] == b[2][wb] and (a[3][wa] == b[3][wb]).all()


@pytest.mark.gpu
def test_gpu_tie_windows_in_a_mixed_batch():
    """the tie windows shuffled into the structural-edge batch (test_gpu_edges.mixed_batch): each equals the oracle or has
    its documented status, and the results are the same in reverse order and when each window runs alone"""
    ties = all_kinds(500)
    mixed, mixed_st = te.mixed_batch()
    allw = [ties.window(w) for w in range(ties.n_windows)] + [mixed.window(w) for w in range(mixed.n_windows)]
    types = [int(t) for t in ties.win_type] + [int(t) for t in mixed.win_type]
    want_st = np.concatenate([np.zeros(ties.n_windows, np.uint32), mixed_st])
    perm = np.random.default_rng(13).permutation(len(allw))
    ws = windows.from_lists([allw[i] for i in perm], [types[i] for i in perm])
    want_st = want_st[perm]
    got = _device(ws)
    te.check(ws, got, ob.oracle_consensus(ws, threads=THREADS, want_coverage=True), want_st, what="tie windows mixed")
    n = ws.n_windows
    rev = _device(ws.subset(np.arange(n)[::-1]))
    bad = [w for w in range(n) if not _same(got, rev, w, n - 1 - w)]
    assert not bad, "reverse order differs on windows %s" % bad[:8]
    bad = [w for w in range(n) if not _same(got, _device(ws.subset([w])), w, 0)]
    assert not bad, "alone differs on windows %s" % bad[:8]


@pytest.mark.gpu
@pytest.mark.parametrize("wlen", WLENS)
def test_gpu_tie_windows_by_reference(wlen):
    """the same windows gathered on the device from a read store (layers hidden in longer reads, about half of them as
    reverse complements with reversed qualities): byte-equal to the pointer path and the oracle, with the device's weight
    computation seeing 0 ('!') and 93 ('~')"""
    from racon_b200 import api
    from tests import test_zz_gpu_resident as tr
    ws = all_kinds(wlen)
    lq = [q for w in range(ws.n_windows) for _, q, _, _ in ws.window(w)[1:] if q]
    assert any(set(q) == {33} for q in lq) and any(set(q) == {126} for q in lq)
    seqs, quals, pieces = tr._as_store(ws, seed=wlen)
    for scores in ((3, -5, -4), (1, -1, -1), (0, 0, 0), (2, 3, -1)):
        cons, pol, st, _, _ = tr._by_reference(ws, seqs, quals, pieces, scores=scores, window_length=wlen)
        ptr, ppol, pst = api.consensus(ws, *scores, window_length=wlen)
        want = oracle(wlen, scores)
        assert (st == 0).all() and (pst == 0).all(), (st, pst)
        bad = [w for w in range(ws.n_windows) if not cons[w] == ptr[w] == want[0][w]]
        assert not bad, "%s: by reference, by pointer and the oracle differ on windows %s" % (scores, bad[:8])
        assert (pol == ppol).all() and (pol == want[1]).all()
