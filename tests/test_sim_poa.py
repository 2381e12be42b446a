"""CPU-side parity of the DEVICE CODE (poa_core.cuh) run through the test-only 32-fibre warp simulation,
against the restated oracle: consensus bytes, polished flags and per-base coverage, window by window."""
import numpy as np
import pytest

from oracle import bindings as ob
from tests import simlib, util

CASES = {
    "fullspan_small": dict(n=6, wlen=120, depth=10, err=0.12),
    "partial": dict(n=6, wlen=150, depth=12, err=0.10, partial_frac=0.5),
    "partial_qual": dict(n=6, wlen=150, depth=10, err=0.12, partial_frac=0.4, with_qual=True, backbone_qual=True),
    "ngs": dict(n=8, wlen=100, depth=16, err=0.02, partial_frac=0.9, with_qual=True, types=0),
    "acgtn": dict(n=5, wlen=100, depth=10, err=0.2, partial_frac=0.2, alphabet=b"ACGTN"),
    "shallow": dict(n=10, wlen=60, depth=3, err=0.2, partial_frac=0.3),
    "higherr_ties": dict(n=8, wlen=80, depth=14, err=0.3),
    "multichunk": dict(n=1, wlen=560, depth=4, err=0.08),
    "threechunks": dict(n=1, wlen=1060, depth=3, err=0.05, partial_frac=0.3),
}


def _mk(name, seed):
    kw = dict(CASES[name])
    n = kw.pop("n")
    t = kw.pop("types", None)
    ws = util.make_set(seed, n, **kw)
    if t is not None:
        ws.win_type[:] = t
    return ws


def _check(ws, scores=(3, -5, -4), trim=True, **simkw):
    m, x, g = scores
    cons, pol, st, covs, stats = simlib.sim_consensus(ws, m, x, g, trim=trim, **simkw)
    ora, opol, _, ocov = ob.oracle_consensus(ws, m, x, g, trim=trim, threads=4, want_coverage=True)
    assert (st == 0).all(), st
    for w in range(ws.n_windows):
        assert cons[w] == ora[w], "window %d consensus differs" % w
        assert bool(pol[w]) == bool(opol[w])
        if pol[w]:
            assert (covs[w].astype(np.uint32) == ocov[w]).all(), "window %d coverage differs" % w
    return stats


@pytest.mark.parametrize("name", sorted(CASES))
def test_sim_equals_oracle(name):
    _check(_mk(name, seed=11))


@pytest.mark.parametrize("scores", [(5, -4, -8), (1, -1, -1), (2, -7, -3)])
def test_sim_scores(scores):
    _check(_mk("partial_qual", seed=5), scores=scores)
    _check(_mk("higherr_ties", seed=6), scores=scores)


def test_sim_tiny_ring_forces_far_predecessor_path():
    # 2 ring rows only: almost every predecessor that is not the previous row is fetched from the HBM copy
    ws = _mk("fullspan_small", seed=3)
    _check(ws, smem=4 * 1024 + 2 * 1024, tile_rows=8)  # profile chunk | 2 ring rows


def test_sim_tiny_traceback_tile_forces_out_of_tile_predecessors():
    # 3-rank tiles: most predecessor rows fall below the tile and are read from the HBM copy
    _check(_mk("fullspan_small", seed=8), tile_rows=3)
    _check(_mk("partial", seed=8), tile_rows=2)


def test_sim_hbm_fallback_of_the_order_dfs():
    # ka != 8 selects the HBM-resident variant of the spoa-order DFS
    _check(_mk("higherr_ties", seed=21), ka=7)
    _check(_mk("partial", seed=4), ka=9)
    _check(_mk("partial_qual", seed=4), debug_flags=1)


def test_sim_escalation_limits_configuration():
    # the limits of the GPU escalation pass (96 in-edge slots, large node budget) on ordinary windows
    _check(_mk("higherr_ties", seed=2), nmax=20000, lmax=4095, ki=96)
    _check(_mk("partial_qual", seed=2), nmax=20000, lmax=4095, ki=96)


def test_sim_branch_completion_is_exercised():
    # seeds chosen with the oracle's counters: the heaviest-bundle maximum is not a sink => BranchCompletion
    for seed in (48, 61, 78):
        _check(util.make_set(seed, 6, wlen=80, depth=14, err=0.3))
        _check(util.make_set(seed, 6, wlen=80, depth=14, err=0.3), debug_flags=1)  # HBM-resident variants


def test_sim_no_trim_and_trivial():
    _check(_mk("partial", seed=9), trim=False)
    from racon_b200 import windows
    tiny = windows.from_lists([[(b"ACGTACGT", None, 0, 0), (b"ACGTTCGT", None, 0, 7)], [(b"AC", None, 0, 0)]])
    cons, pol, st, _, _ = simlib.sim_consensus(tiny)
    assert cons == [b"ACGTACGT", b"AC"] and not pol.any()


def test_sim_sink_ties_are_exercised():
    stats = _check(_mk("higherr_ties", seed=21))
    assert stats[2] > 0, "no sink tie occurred; pick another seed so the tie-break path is covered"


def test_sim_limits_are_reported_not_crashed():
    ws = _mk("fullspan_small", seed=4)
    cons, pol, st, _, _ = simlib.sim_consensus(ws, nmax=150)
    assert (st == 1).all() and not pol.any()  # RP_WIN_NODE_LIMIT
    cons, pol, st, _, _ = simlib.sim_consensus(ws, ki=2)
    assert ((st == 2) | (st == 0)).all() and (st == 2).any()  # RP_WIN_EDGE_LIMIT


def test_sim_edge_cases_ragged_and_degenerate():
    """Empty / ragged inputs as the reference accepts them: skipped layers (len 0, begin == end), 1-base layers,
    a 1-base backbone, windows where everything but two layers is skipped (=> backbone copy, not polished)."""
    from racon_b200 import windows
    bb = b"ACGTTGCAACGTAGCTAGCTAGGATCGATCGATCGTAGCTAGCTAGCATCGATCGTAGCATGCATGCAA"
    wins = [
        # two real layers + skipped ones (zero length / begin == end)
        [(bb, None, 0, 0), (bb[:40], None, 0, 39), (b"", None, 0, 10), (bb[5:60], None, 5, 59), (b"ACG", None, 7, 7),
         (bb, None, 0, len(bb) - 1)],
        # 1-base layers and a quality-weighted one
        [(bb, None, 0, 0), (b"A", None, 0, 1), (b"T", None, 3, 4), (bb[10:50], b"5" * 40, 10, 49),
         (bb, None, 0, len(bb) - 1)],
        # everything skipped but one layer -> < 3 sequences
        [(bb, None, 0, 0), (b"", None, 0, 5), (bb, None, 0, len(bb) - 1), (b"AC", None, 9, 9)],
        # very short backbone
        [(b"AC", None, 0, 0), (b"AC", None, 0, 1), (b"AG", None, 0, 1), (b"AC", None, 0, 1)],
        [(b"A", None, 0, 0)],
    ]
    ws = windows.from_lists(wins)
    cons, pol, st, covs, _ = simlib.sim_consensus(ws)
    ora, opol, _, ocov = ob.oracle_consensus(ws, want_coverage=True)
    assert cons == ora and (pol == opol).all() and (st == 0).all()
    if ob.have_ref():
        ref, rpol, _ = ob.ref_consensus(ws)
        assert ref == cons and (rpol == pol).all()


def test_sim_rare_characters_inside_long_runs_of_bases_reach_the_alphabet():
    """The packer looks at 16 bases at a time and walks a block byte by byte only when it holds something other than
    ACGT: one lower-case / IUPAC character deep inside a layer (and in the unaligned tail of one) must still be in the
    window's alphabet — the consensus over it equals the oracle's, which compares characters directly."""
    from racon_b200 import windows
    rng = np.random.default_rng(11)
    bb = bytes(rng.choice(list(b"ACGT"), size=150).astype(np.uint8))
    lay = []
    for k, (pos, ch) in enumerate([(3, b"n"), (37, b"R"), (64, b"a"), (149, b"Y"), (100, b"R"), (17, b"n"), (64, b"a")]):
        t = bytearray(bb)
        t[pos:pos + 1] = ch
        lay.append((bytes(t), None, 0, len(bb) - 1))
    ws = windows.from_lists([[(bb, None, 0, 0)] + lay + [(bb, None, 0, len(bb) - 1)]])
    cons, pol, st, _, _ = simlib.sim_consensus(ws)
    ora, opol, _ = ob.oracle_consensus(ws)
    assert (st == 0).all() and cons == ora and (pol == opol).all()
    # nine distinct characters: beyond the device's 8-code alphabet -> reported, not computed wrongly
    t = bytearray(bb)
    t[20:25] = b"nRaYN"
    ws9 = windows.from_lists([[(bb, None, 0, 0), (bytes(t), None, 0, len(bb) - 1), (bb, None, 0, len(bb) - 1),
                               (bb, None, 0, len(bb) - 1)]])
    _, pol9, st9, _, _ = simlib.sim_consensus(ws9)
    assert (st9 != 0).all() and not pol9.any()


def test_sim_malformed_windows_are_rejected_not_crashed():
    """The reference exit(1)s on these (window.cpp:19-23,49-58); the ABI returns RP_ERR_INVALID instead."""
    from racon_b200 import windows
    bb = b"ACGTACGTACGTACGTACGT"
    for bad in ([(bb, None, 0, 0), (bb, None, 12, 5), (bb, None, 0, 19), (bb, None, 0, 19)],      # begin > end
                [(bb, None, 0, 0), (bb, None, 0, 25), (bb, None, 0, 19), (bb, None, 0, 19)]):     # end > backbone
        with pytest.raises(RuntimeError):
            simlib.sim_consensus(windows.from_lists([bad]))


def _spoa_would_use_int32(m, g, length, nodes):
    """spoa's engine choice (alignment_engine.cpp:101-110, simd impl :699-745)"""
    i, j = length + 8, nodes
    worst = min(-(m * min(i, j) + g * abs(i - j)), g * i + g * j)
    return worst < -32768 + 1024


def test_sim_windows_beyond_spoa_int16_bound_are_computed_exactly():
    """A steep gap penalty makes spoa's worst-case bound fail (it would switch to its int32 engine) although the real
    matrix stays far inside int16: such windows are computed in int16 and verified on the finished matrix — same
    result as the oracle (which is int32 throughout), no RP_WIN_NEEDS_INT32."""
    ws = util.make_set(21, 5, wlen=200, depth=16, err=0.12, partial_frac=0.3, with_qual=True)
    scores = (3, -5, -60)
    assert _spoa_would_use_int32(3, -60, 200, 500)
    _check(ws, scores=scores)
    ws2 = util.make_set(22, 3, wlen=250, depth=10, err=0.2)
    _check(ws2, scores=(5, -4, -40))
    if ob.have_ref():   # the unmodified spoa (its int32 engine here) agrees with both
        assert ob.ref_consensus(ws, 3, -5, -60)[0] == simlib.sim_consensus(ws, 3, -5, -60)[0]
        assert ob.ref_consensus(ws2, 5, -4, -40)[0] == simlib.sim_consensus(ws2, 5, -4, -40)[0]


def test_sim_windows_whose_matrix_leaves_int16_are_reported():
    """gap = -64 at 600 columns: column 0 alone reaches -38 000, so the range check must refuse the window."""
    ws = util.make_set(23, 2, wlen=600, depth=5, err=0.1)
    _, pol, st, _, _ = simlib.sim_consensus(ws, 3, -5, -64)
    assert (st == 4).all() and not pol.any()     # RP_WIN_NEEDS_INT32
    # and a gap beyond the packed-int16 design limit is refused up front
    _, pol, st, _, _ = simlib.sim_consensus(util.make_set(24, 2, wlen=100, depth=5, err=0.1), 3, -5, -100)
    assert (st == 4).all() and not pol.any()


# ---------------------------------------------------------------------------------------------------------------
# lane groups (8 / 16 lanes per window) and the banded DP of racon -b, same device code, same oracle
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lanes", [8, 16])
@pytest.mark.parametrize("name", ["fullspan_small", "partial_qual", "higherr_ties", "multichunk", "ngs"])
def test_sim_lane_groups_equal_oracle(name, lanes):
    _check(_mk(name, seed=11), lanes=lanes, smem=14336 * lanes // 32)


BAND_CASES = {
    "w300": dict(n=2, wlen=300, depth=12, err=0.12),
    "w500_partial_qual": dict(n=2, wlen=500, depth=16, err=0.12, partial_frac=0.4, with_qual=True),
    "w200_higherr": dict(n=3, wlen=200, depth=16, err=0.3),
    "w1000": dict(n=1, wlen=1000, depth=8, err=0.10, partial_frac=0.2),
}


@pytest.mark.parametrize("lanes", [8, 16])
@pytest.mark.parametrize("name", sorted(BAND_CASES))
def test_sim_banded_equals_oracle(name, lanes):
    kw = dict(BAND_CASES[name])
    ws = util.make_set(7, kw.pop("n"), **kw)
    stats = _check(ws, lanes=lanes, smem=14336 * lanes // 32, banded=1, nmax=8192, lmax=2047)
    if 16 * lanes < kw["wlen"] // 2:
        assert stats[4] > 0, "no alignment went through the band"


@pytest.mark.parametrize("scores", [(5, -4, -8), (1, -1, -1)])
def test_sim_banded_other_scores(scores):
    ws = util.make_set(8, 2, wlen=400, depth=12, err=0.15, partial_frac=0.3, with_qual=True)
    _check(ws, scores=scores, lanes=8, smem=3584, banded=1)


def test_sim_band_refusal_redoes_the_alignment_with_the_full_matrix():
    """(a) a margin wider than the band refuses every band result; (b) layers with a 110-base deletion or a 120-base
    insertion leave a 128-column band.  Both must fall back to the full matrix on the spot and stay exact."""
    ws = util.make_set(9, 2, wlen=400, depth=10, err=0.12, partial_frac=0.3)
    stats = _check(ws, lanes=8, smem=3584, banded=1, band_margin=56)
    assert stats[4] > 0 and stats[5] == stats[4]
    rng = np.random.default_rng(5)
    wins = []
    for _ in range(2):
        truth = bytes(b"ACGT"[i] for i in rng.integers(4, size=500))
        bb = util.mutate(rng, truth, 0.1)[:500]
        win = [(bb, None, 0, 0)]
        for d in range(9):
            r = util.mutate(rng, truth, 0.1)
            if d % 3 == 0:
                r = r[:150] + r[260:]
            if d % 3 == 1:
                r = r[:200] + bytes(b"ACGT"[i] for i in rng.integers(4, size=120)) + r[200:]
            win.append((r, None, 0, len(bb) - 1))
        wins.append(win)
    from racon_b200 import windows
    stats = _check(windows.from_lists(wins), lanes=8, smem=3584, banded=1, nmax=8192, lmax=2047)
    assert 0 < stats[5] < stats[4]


def test_sim_matrix_scratch_limit_is_reported():
    """A score matrix larger than the per-window scratch gets RP_WIN_MATRIX_LIMIT (the GPU escalation pass re-runs it)."""
    ws = _mk("fullspan_small", seed=4)
    _, pol, st, _, _ = simlib.sim_consensus(ws, hcap=20000)
    assert (st == 9).all() and not pol.any()


def test_sim_band_audit_finds_no_differing_alignment():
    """debug flag 2 recomputes every ACCEPTED band result with the full matrix inside the device code and counts the
    alignments that differ (stats[6]): none, also on the 30 %-error family whose graphs have > 8 in-edges per node."""
    ws = util.make_set(101, 32, wlen=300, depth=40, err=0.3).subset([0, 12])
    stats = _check(ws, lanes=8, smem=3584, banded=1, debug_flags=2)
    assert stats[4] > 0 and stats[6] == 0
    ws = util.make_set(12, 2, wlen=500, depth=20, err=0.12, partial_frac=0.3, with_qual=True)
    stats = _check(ws, lanes=8, smem=3584, banded=1, debug_flags=2)
    assert stats[4] > 0 and stats[6] == 0


@pytest.mark.parametrize("kb", [4, 8])
@pytest.mark.parametrize("name", sorted(BAND_CASES))
def test_sim_narrow_banded_rows_equal_oracle(name, kb):
    """racon -b default layout: 32 lanes x 4 (or 8) columns per lane — a 128- (256-) column band held in two (four) packed
    registers per lane; band audit on (every accepted band result recomputed with the full matrix: no difference)."""
    kw = dict(BAND_CASES[name])
    ws = util.make_set(7, kw.pop("n"), **kw)
    stats = _check(ws, lanes=32, smem=9216, banded=1, nmax=8192, lmax=2047, band_cols_per_lane=kb, debug_flags=2)
    assert stats[6] == 0
    if 32 * kb < kw["wlen"] // 2:
        assert stats[4] > 0, "no alignment went through the band"


def test_sim_narrow_band_refusal_and_other_scores():
    ws = util.make_set(9, 2, wlen=400, depth=10, err=0.12, partial_frac=0.3)
    stats = _check(ws, lanes=32, smem=9216, banded=1, band_margin=56, band_cols_per_lane=4)
    assert stats[4] > 0 and stats[5] == stats[4]
    ws = util.make_set(8, 2, wlen=400, depth=12, err=0.15, partial_frac=0.3, with_qual=True)
    for scores in ((5, -4, -8), (1, -1, -1)):
        _check(ws, scores=scores, lanes=32, smem=9216, banded=1, band_cols_per_lane=4, debug_flags=2)
    ws = util.make_set(101, 32, wlen=300, depth=40, err=0.3).subset([0, 12])
    stats = _check(ws, lanes=32, smem=9216, banded=1, band_cols_per_lane=4, debug_flags=2)
    assert stats[4] > 0 and stats[6] == 0


def test_sim_band_real_windows_whose_true_path_leaves_the_band():
    """Two windows of the lambda -f run (unit scores) found on the GPU by tools/find_band_divergence.py: a layer's true
    alignment runs 70-130 columns away from the band's centre line while an in-band path of almost the same score keeps
    every margin — the band result used to be accepted and the consensus differed from the reference's.  The acceptance
    check's alignment-quality rule (kBandJunkLimit) now refuses those band results; the on-device full-matrix redo makes the
    windows exact again."""
    import os
    from racon_b200 import windows
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lambda_frag_band_cases.npz"))
    ws = windows.WindowSet(bases=z["bases"], quals=z["quals"] if z["quals"].size else None, seq_off=z["seq_off"],
                           seq_has_qual=z["seq_has_qual"] if z["seq_has_qual"].size else None, seq_begin=z["seq_begin"],
                           seq_end=z["seq_end"], win_first=z["win_first"], win_type=z["win_type"])
    scores = tuple(int(v) for v in z["scores"])
    for kb in (8, 4):
        stats = _check(ws, scores=scores, lanes=32, smem=9216, banded=1, band_cols_per_lane=kb, debug_flags=2)
        assert stats[5] > 0 and stats[6] == 0, stats
