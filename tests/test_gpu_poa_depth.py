"""The POA kernel on deep windows (65 536 sequences and more), window by window against the int64 oracle.

The library keeps every layer of a window however deep (no depth cap, unlike cudapoa's 200), so the quantities that grow
with the number of sequences, not with the window length, must stay exact:
- sequences through a node (spoa's Node::Coverage), a 32-bit counter per node, and the per-column sum over a node and
  its aligned nodes, which decides racon's kTGS trim against (n_seq - 1) / 2.  The per-base coverage returned to the
  caller is uint16 (cudapoa's type) and saturates at 65 535, so it is compared as min(oracle, 65 535);
- the total edge weight, which picks int32 heaviest-bundle scores in shared memory (below 2^31 - 1) or int64 scores in
  HBM (from 2^31 - 1 on).

Every generator proves it reaches the edge it names, from its inputs: sequences through a node, column sums, total edge
weight.  Deep windows also run in mixed and small-budget batches and by reference from a read store, and a deep
amplicon goes through the racon_b200 command line against racon's bytes.  The case generators are plain functions.  One window also runs through the CPU warp simulation of the same
device code (`test_sim_depth_coverage_wrap`), and the oracle's answers on three ladder windows are pinned to those of the
unmodified reference in tests/golden/ref_answers.json (`test_oracle_pinned_depth`)."""
import os

import numpy as np
import pytest

from oracle import bindings as ob
from racon_b200 import windows
from tests import simlib, util

THREADS = os.cpu_count() or 4
U16 = 0xffff
TOP32 = 0x7fffffff                        # total edge weight from which the bundle scores go to int64 in HBM
LADDER = [65534, 65535, 65536, 65537, 131071, 131072, 131073]     # sequences per window, backbone included
QUALS = ["none", "flat", "random"]
PINNED = [65535, 65536, 131073]


# ---- what the window's inputs put into the graph -------------------------------------------------------------------------
def seq_weights(win):
    """per sequence, the weight it adds over its edges: sum over j >= 1 of w[j-1] + w[j], with w = quality - 33, 1 for a
    layer without qualities and 0 for a backbone without them (racon's dummy '!')"""
    out = []
    for s, (b, q, _, _) in enumerate(win):
        if len(b) < 2:
            out.append(0)
            continue
        if q is not None:
            w = np.frombuffer(q, np.uint8).astype(np.int64) - 33
        else:
            w = np.full(len(b), 0 if s == 0 else 1, np.int64)
        out.append(int(2 * w.sum() - w[0] - w[-1]))
    return out


def total_edge_weight(win):
    return sum(seq_weights(win))


def column_coverage(win):
    """sequences through each backbone column, for windows whose layers are exact copies of the backbone piece they
    span: every layer then runs through the backbone's own nodes"""
    bb = win[0][0]
    cov = np.ones(len(bb), np.int64)
    for b, _, s, e in win[1:]:
        assert b == bb[s:e + 1]
        cov[s:e + 1] += 1
    return cov


# ---- case generators -----------------------------------------------------------------------------------------------------
def _rand(rng, n):
    return bytes(util.BASES[i] for i in rng.integers(4, size=n))


def _layer_quals(rng, mode, n_layers, length):
    if mode == "none":
        return [None] * n_layers
    if mode == "flat":
        return [b"5" * length] * n_layers     # phred 20
    q = (rng.integers(0, 61, size=(n_layers, length)) + 33).astype(np.uint8)
    return [r.tobytes() for r in q]


def ladder_window(n_seq, quals="none", seed=1):
    """30 random bases between TTTTT and GGGGG as the backbone; n_seq - 1 layers that copy the 30 bases (a partial span,
    so each goes through the Subgraph path).  Every core node has n_seq sequences through it, the flanks 1: racon's
    trim keeps exactly the core."""
    core = _rand(np.random.default_rng(seed), 30)
    bb = b"TTTTT" + core + b"GGGGG"
    qs = _layer_quals(np.random.default_rng(seed + 100), quals, n_seq - 1, len(core))
    return [(bb, None, 0, 0)] + [(core, q, 5, 34) for q in qs]


def haplotype_window(per_hap=25000, n_hap=3):
    """n_hap haplotypes of 30 bases, each a run of its own letter (A, C, G), so that they differ at every column and
    align base for base as mismatches; per_hap partial-span layers each, the backbone haplotype A between TTTTT and
    TTTTT, with qualities (so that its flanks weigh more than nothing and stay in the untrimmed consensus).  A node
    holds one letter, so no node has more than per_hap + 1 sequences through it, less than both 65 536 and the trim
    threshold; only the sum over a column's aligned nodes reaches the threshold, and it passes 65 535.  (A 16-bit node
    counter does not wrap here, and a column sum clamped to 65 535 still clears the threshold of 37 500: this window
    checks the sum over aligned nodes, not the width; the ladder's 131 07x windows catch a saturated comparison.)"""
    haps = [bytes([c]) * 30 for c in b"ACG"[:n_hap]]
    bb = b"TTTTT" + haps[0] + b"TTTTT"
    win = [(bb, b"5" * len(bb), 0, 0)]
    for k in range(per_hap * n_hap):
        win.append((haps[k % n_hap], None, 5, 34))
    return win


def staggered_window(n_layers, seed=3):
    """Layers that copy the backbone from one of ten begins (5..14) to one of ten ends (25..34): coverage steps up by
    n_layers / 10 per column at the start and down at the end, and the trim threshold falls inside both staircases."""
    bb = b"TTTTT" + _rand(np.random.default_rng(seed), 30) + b"GGGGG"
    win = [(bb, None, 0, 0)]
    for k in range(n_layers):
        s, e = 5 + k % 10, 34 - (k // 10) % 10
        win.append((bb[s:e + 1], None, s, e))
    return win


def expected_trim(win):
    """the part of the backbone racon's trim keeps, from the column coverage of the inputs"""
    cov = column_coverage(win)
    thr = (len(win) - 1) // 2
    keep = np.nonzero(cov >= thr)[0]
    return win[0][0][keep[0]:keep[-1] + 1]


def weight_window(target, length=1000, seed=4):
    """Full-length layers with '~' qualities (weight 93 per base) from two haplotypes that differ at five SNPs, three
    layers of haplotype A to every two of B, the backbone A without qualities.  The last layer's qualities are lowered
    until the total edge weight is exactly `target`.  The heaviest-bundle score of the consensus path is then close to
    the total weight, so at 3 * 2^31 an int32 score would wrap several times along the path and end the consensus early;
    at 2^31 - 2 and 2^31 - 1 both score widths are exact, and the pair checks that each bundle path gives the oracle's
    answer at the switch."""
    rng = np.random.default_rng(seed)
    hap_a = _rand(rng, length)
    hb = bytearray(hap_a)
    for k in range(100, length, length // 5):
        hb[k] = util.BASES[(util.BASES.index(hb[k]) + 1) % 4]
    hap_b = bytes(hb)
    full = 2 * 93 * (length - 1)
    n = -(-target // full)
    units = n * full - target            # weight to take off the last layer
    q = np.full(length, 93, np.int64)
    q[-1] -= units % 2
    units //= 2
    for j in range(1, length - 1):       # an interior base counts twice
        d = min(units, q[j])
        q[j] -= d
        units -= d
    q[0] -= units                        # what is left (at most 93 units): both ends, once each
    q[-1] -= units
    last = (q + 33).astype(np.uint8).tobytes()
    win = [(hap_a, None, 0, 0)]
    for k in range(n):
        win.append((hap_b if k % 5 in (1, 3) else hap_a, last if k == n - 1 else b"~" * length, 0, length - 1))
    assert total_edge_weight(win) == target
    return win


WEIGHT_TARGETS = {"int32_top": TOP32 - 1, "int64_first": TOP32, "three_times": 3 * (1 << 31)}


# ---- end to end: a deep amplicon as files --------------------------------------------------------------------------------
AMPLICON_READS = 66000


def write_deep_amplicon(d, n_reads=AMPLICON_READS, seed=21):
    """A 1 499-base amplicon and its draft, which has one extra base at draft position 500, the first of the second
    500-base window; the extra base differs from both its neighbours, so the aligner cannot place the deletion anywhere
    else and that window's layers begin one base after its backbone.  n_reads reads (FASTA, more than 1 000 bases, so
    racon makes kTGS windows) copy the amplicon from one of the first ten bases to one of the last ten, each with one PAF
    line.  More than 65 536 sequences then run through every node of the middle window.  Writes reads.fasta,
    overlaps.paf and draft.fasta into d; returns their paths."""
    rng = np.random.default_rng(seed)
    truth = _rand(rng, 1499)
    extra = next(c for c in util.BASES if c not in (truth[499], truth[500]))
    draft = truth[:500] + bytes([extra]) + truth[500:]
    with open(os.path.join(d, "draft.fasta"), "wb") as f:
        f.write(b">amplicon\n" + draft + b"\n")
    starts = rng.integers(0, 10, size=n_reads)
    ends = len(truth) - rng.integers(0, 10, size=n_reads)
    reads, paf = [], []
    for k, (s, e) in enumerate(zip(starts.tolist(), ends.tolist())):
        reads.append(b">r%d\n%s\n" % (k, truth[s:e]))
        paf.append(b"r%d\t%d\t0\t%d\t+\tamplicon\t%d\t%d\t%d\t%d\t%d\t60\n" % (
            k, e - s, e - s, len(draft), s, e + 1, e - s, e + 1 - s))
    with open(os.path.join(d, "reads.fasta"), "wb") as f:
        f.write(b"".join(reads))
    with open(os.path.join(d, "overlaps.paf"), "wb") as f:
        f.write(b"".join(paf))
    return [os.path.join(d, n) for n in ("reads.fasta", "overlaps.paf", "draft.fasta")]


# ---- checks --------------------------------------------------------------------------------------------------------------
_cache = {}


def cached(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def oracle(ws, key, trim=True, window_length=500):
    return cached(("oracle", key, trim, window_length),
                  lambda: ob.oracle_consensus(ws, trim=trim, window_length=window_length, threads=THREADS,
                                              want_coverage=True))


def check(ws, got, want, what=""):
    """every window status 0, with the oracle's consensus and polished flag, and its coverage saturated at 65 535"""
    cons, pol, st, cov = got
    bad = [w for w in range(ws.n_windows) if st[w]]
    assert not bad, "%s: status %s on windows %s" % (what, [int(st[w]) for w in bad[:8]], bad[:8])
    for w in range(ws.n_windows):
        assert cons[w] == want[0][w], "%s: consensus differs on window %d (%d vs %d bases)" % (
            what, w, len(cons[w]), len(want[0][w]))
        assert pol[w] == want[1][w], "%s: polished flag differs on window %d" % (what, w)
        assert (np.asarray(cov[w], np.uint32) == np.minimum(want[3][w], U16)).all(), "%s: coverage differs on window %d" % (
            what, w)


def ladder_set(trim):
    """every ladder depth x quality mode, as kTGS windows and (with trim) as kNGS windows too"""
    wins, types, names = [], [], []
    for t in ((1, 0) if trim else (1,)):
        for n in LADDER:
            for q in QUALS:
                wins.append(ladder_window(n, q))
                types.append(t)
                names.append((n, q, t, wins[-1][0][0]))
    return names, windows.from_lists(wins, types)


def _ladder(trim):
    return cached(("ladder", trim), lambda: ladder_set(trim))


# ---- the edges the generators reach (no GPU) -----------------------------------------------------------------------------
def test_generators_reach_their_edges():
    for n in (65536, 131073):
        win = ladder_window(n)
        cov = column_coverage(win)
        assert cov.max() == n and cov[5:35].min() == n and cov[0] == 1
        assert expected_trim(win) == win[0][0][5:35]
    assert (131073 - 1) // 2 > U16          # the threshold itself passes 65 535
    hap = haplotype_window()
    thr = (len(hap) - 1) // 2
    letters = [set(b) for b, _, _, _ in hap[1:4]]           # the three haplotypes
    assert all(len(x) == 1 for x in letters) and len(set.union(*letters)) == 3
    assert not set.union(*letters) & set(hap[0][0][:5] + hap[0][0][-5:])     # nor the flanks' letter
    per_node = max(sum(1 for b, _, _, _ in hap[1:] if set(b) == x) for x in letters) + 1   # + the backbone
    assert per_node == 25001 and per_node < thr and per_node < U16 and len(hap) > U16
    for n in (70000, 140000):
        win = staggered_window(n)
        cov, thr = column_coverage(win), (len(win) - 1) // 2
        assert cov.max() > U16 and cov[5] < thr and cov[34] < thr
        assert 5 < win[0][0].index(expected_trim(win)) < 14
    for name, target in WEIGHT_TARGETS.items():
        win = weight_window(target)
        assert total_edge_weight(win) == target, name
    # the three quality modes do not change the coverage, only the edge weights
    w = ladder_window(65536, "random")
    assert 0 < total_edge_weight(w) < TOP32


def test_oracle_trims_the_ladder():
    """The oracle keeps exactly the core of every ladder window with trim, the whole backbone without, and counts every
    sequence through the core (coverage n_seq, above 65 535 from 65 536 on)."""
    for n in (65535, 65536, 131073):
        win = ladder_window(n)
        ws = windows.from_lists([win], [1])
        cons, pol, _, cov = ob.oracle_consensus(ws, threads=1, want_coverage=True)
        assert cons[0] == win[0][0][5:35] and pol[0] and cov[0].max() == n
        cons, _, _, cov = ob.oracle_consensus(ws, trim=False, threads=1, want_coverage=True)
        assert cons[0] == win[0][0] and cov[0].max() == n and cov[0][0] == 1


# ---- the oracle pinned to the reference's stored answers -----------------------------------------------------------------
def pinned_key(n):
    return "depth/ladder/%d" % n


def pinned_case(n):
    ws = windows.from_lists([ladder_window(n)], [1])
    return lambda consensus: consensus(ws)[:2]


def test_oracle_pinned_depth():
    answers = util.ref_answers()["poa"]
    for n in PINNED:
        want = answers[pinned_key(n)]
        assert util.consensus_answer(*pinned_case(n)(ob.oracle_consensus)) == want, n
        if ob.have_ref():
            assert util.consensus_answer(*pinned_case(n)(ob.ref_consensus)) == want, n


# ---- CPU twin: one window through the warp simulation ---------------------------------------------------------------------
def test_sim_depth_coverage_wrap():
    """65 536 sequences through the two core nodes of backbone TACG: a 16-bit node counter wraps to 0 there, no column
    reaches the trim threshold and the whole backbone comes back.  The shortest layers that still make the trim decide
    (2 bases), on an 8-lane group, keep the simulation to about half a minute."""
    ws = windows.from_lists([[(b"TACG", None, 0, 0)] + [(b"AC", None, 1, 2)] * 65535], [1])
    want = ob.oracle_consensus(ws, want_coverage=True)
    assert want[0][0] == b"AC" and want[3][0].max() == 65536
    cons, pol, st, cov, _ = simlib.sim_consensus(ws, nmax=64, lmax=8, lanes=8)
    check(ws, (cons, pol, st, cov), want, what="sim 65 536 sequences")


# ---- on the device -------------------------------------------------------------------------------------------------------
def _device(ws, trim=True, window_length=500, banded=False, band_stats=None, mem_bytes=0):
    from racon_b200 import api
    return api.consensus(ws, trim=trim, window_length=window_length, want_coverage=True, banded=banded,
                         band_stats=band_stats, mem_bytes=mem_bytes)


@pytest.mark.gpu
@pytest.mark.parametrize("trim", [True, False], ids=["trim", "no_trim"])
def test_gpu_coverage_ladder(trim):
    """65 534 .. 131 073 sequences, qualities none / flat / random; with trim as kTGS (the trim decides) and kNGS (never
    trimmed) windows, without trim as kTGS windows."""
    names, ws = _ladder(trim)
    want = oracle(ws, ("ladder", trim), trim=trim)
    for w, (n, q, t, bb) in enumerate(names):
        assert want[0][w] == (bb[5:35] if trim and t == 1 else bb), (n, q, t)
        assert int(want[3][w].max()) == n
    check(ws, _device(ws, trim=trim), want, what="ladder trim=%s" % trim)


@pytest.mark.gpu
def test_gpu_column_sums_decide_the_trim():
    """Three haplotypes that differ at every column, 25 000 layers each: the trim is decided by column sums of 75 001
    over aligned nodes of at most 25 001 sequences each.  Staggered partial spans (70 000 and 140 000 layers): coverage
    steps up and down along the consensus and the trim lands inside both staircases."""
    wins = [haplotype_window(), staggered_window(70000), staggered_window(140000)]
    ws = windows.from_lists(wins, [1] * len(wins))
    want = oracle(ws, "sums")
    assert len(want[0][0]) == 30 and (want[3][0] == len(wins[0])).all() and len(wins[0]) > U16
    for w in (1, 2):
        assert want[0][w] == expected_trim(wins[w])
        assert want[0][w] != wins[w][0][0][5:35]
    check(ws, _device(ws), want, what="column sums")


def _weight_set():
    names = sorted(WEIGHT_TARGETS)
    return names, windows.from_lists([weight_window(WEIGHT_TARGETS[k]) for k in names], [1] * len(names))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["full", "band256"])
def test_gpu_total_edge_weight_across_int32(mode, monkeypatch):
    """Total edge weight 2^31 - 2 (int32 bundle scores in shared memory), 2^31 - 1 (int64 in HBM) and 3 * 2^31, at
    window length 1000, in the full matrix and in the 256-column band with the band audit on."""
    names, ws = cached("weights", _weight_set)
    for w, k in enumerate(names):
        assert total_edge_weight(ws.window(w)) == WEIGHT_TARGETS[k]
    want = oracle(ws, "weights", window_length=1000)
    banded = mode != "full"
    if banded:
        monkeypatch.setenv("RP_POA_BAND_K", "8")
        monkeypatch.setenv("RP_BAND_AUDIT", "1")
    stats = {}
    check(ws, _device(ws, window_length=1000, banded=banded, band_stats=stats), want, what=mode)
    if banded:
        assert stats["band_width"] == 256 and stats["band_alignments"] > 0, stats
        assert stats["band_audit_mismatches"] == 0, stats


ORDINARY = 2000


@pytest.mark.gpu
def test_gpu_deep_window_in_a_mixed_batch():
    """A 65 536-sequence window shuffled into 2 000 ordinary windows and the structural-edge batch (windows of every shape
    and soft status), where the queue orders by cost: every window equals the oracle or has its expected status, in
    reverse order too; the structural windows and the deep one also alone."""
    from tests import test_gpu_edges as te
    mixed, mixed_st = te.mixed_batch()
    plain = util.make_set(31, ORDINARY, wlen=500, depth=8, err=0.12, partial_frac=0.2, with_qual=True)
    allw = [plain.window(i) for i in range(plain.n_windows)] + [mixed.window(i) for i in range(mixed.n_windows)] + \
        [ladder_window(65536, "random")]
    types = [int(t) for t in plain.win_type] + [int(t) for t in mixed.win_type] + [1]
    want_st = np.concatenate([np.zeros(plain.n_windows), mixed_st, [0]]).astype(np.uint32)
    structural = np.arange(plain.n_windows, len(allw))
    perm = np.random.default_rng(32).permutation(len(allw))
    ws = windows.from_lists([allw[i] for i in perm], [types[i] for i in perm])
    want_st = want_st[perm]
    at = int(np.nonzero(perm == len(allw) - 1)[0][0])
    want = ob.oracle_consensus(ws, threads=THREADS, want_coverage=True)
    assert want[3][at].max() == 65536
    got = _device(ws)
    te.check(ws, got[:3], want, want_st, what="mixed + deep")
    for w in np.nonzero(got[1])[0]:
        assert (np.asarray(got[3][w], np.uint32) == np.minimum(want[3][w], U16)).all(), "coverage of window %d" % w
    n = ws.n_windows
    rev = _device(ws.subset(np.arange(n)[::-1]))
    for w in range(n):
        r = n - 1 - w
        assert rev[0][r] == got[0][w] and rev[1][r] == got[1][w] and rev[2][r] == got[2][w], "reversed, window %d" % w
        assert np.array_equal(rev[3][r], got[3][w]), "reversed, coverage of window %d" % w
    for w in sorted(int(np.nonzero(perm == i)[0][0]) for i in structural):
        alone = _device(ws.subset([w]))
        assert alone[0][0] == got[0][w] and alone[1][0] == got[1][w] and alone[2][0] == got[2][w], "alone, window %d" % w
        assert np.array_equal(alone[3][0], got[3][w]), "alone, coverage of window %d" % w


def deep_long_window(n_layers=66000, core_len=300, seed=5):
    """n_layers partial-span copies of a 300-base core between TTTTT and GGGGG: about 20 MB of bases in one window,
    more than 65 536 sequences through every core node"""
    core = _rand(np.random.default_rng(seed), core_len)
    return [(b"TTTTT" + core + b"GGGGG", None, 0, 0)] + [(core, None, 5, 4 + core_len)] * n_layers


@pytest.mark.gpu
def test_gpu_deep_window_over_a_small_budget():
    """A 192 MB object takes about 12 MB of input bases per batch; a window of 19.8 MB is refused after another window
    (RP_BATCH_FULL), taken by an empty batch, and the window after it goes to the next batch.  Results equal those of a
    default-budget object and the oracle's."""
    from racon_b200 import api
    small = util.make_set(33, 2, wlen=500, depth=8, err=0.12)
    deep = deep_long_window()
    wins = [small.window(0), deep, small.window(1)]
    assert sum(len(b) for b, _, _, _ in deep) > 19_000_000
    ws = windows.from_lists(wins, [1, 1, 1])
    want = oracle(ws, "budget")
    assert want[3][1].max() == len(deep) and want[0][1] == deep[0][0][5:-5]
    b = api.PoaBatch(mem_bytes=192 << 20, window_length=500)

    def batch_of(w, refused=None):
        """window w into an empty batch (the window after it refused), run; (consensus, polished, status, coverage)"""
        b.reset()
        assert b.add_window(wins[w]) == api.RP_OK
        if refused is not None:
            assert b.add_window(wins[refused]) == api.RP_BATCH_FULL, "window %d was not refused" % refused
        b.run()
        b.sync()
        out, lens, pol, st = b.fetch_all(1100)
        return out[0, :lens[0]].tobytes(), bool(pol[0]), int(st[0]), np.asarray(b.fetch(0)[1]).copy()

    try:
        got = [batch_of(0, refused=1), batch_of(1, refused=2), batch_of(2)]
    finally:
        b.close()
    ref = _device(ws)
    for w in range(3):
        assert got[w][2] == 0 and ref[2][w] == 0, (w, got[w][2], ref[2][w])
        assert got[w][0] == ref[0][w] == want[0][w] and got[w][1] == ref[1][w] == want[1][w], w
        assert np.array_equal(got[w][3], ref[3][w]), w
        assert (np.asarray(ref[3][w], np.uint32) == np.minimum(want[3][w], U16)).all(), w


@pytest.mark.gpu
def test_gpu_deep_windows_by_reference():
    """Deep windows added by reference from a read store (layers hidden inside longer reads, about half of them stored
    reverse-complemented) give the bytes of the pointer path."""
    from tests import test_zz_gpu_resident as tr
    wins = [ladder_window(65536, "random"), ladder_window(131073), haplotype_window(), staggered_window(70000)]
    ws = windows.from_lists(wins, [1] * len(wins))
    seqs, quals, pieces = tr._as_store(ws, seed=34)
    assert 0.4 < np.mean([p[3] for pw in pieces for p in pw[1:]]) < 0.6
    cons, pol, st, _, _ = tr._by_reference(ws, seqs, quals, pieces)
    ptr = _device(ws)
    want = oracle(ws, "by_reference")
    assert (st == 0).all() and (ptr[2] == 0).all(), (st, ptr[2])
    assert cons == ptr[0] == want[0]
    assert (pol == ptr[1]).all() and (pol == want[1]).all()


@pytest.mark.gpu
def test_gpu_deep_amplicon_command_line(tmp_path):
    """racon_b200 on a deep amplicon (66 000 reads, tests/golden/cli_cases.json "deep_amplicon"): exit status 0 and the
    bytes racon's own command line prints.  The draft's extra base sits alone at the start of a window whose nodes have
    66 001 sequences through them; only a trim against the exact coverage removes it."""
    import hashlib
    import json
    from tests.test_cli import run_cli
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cli_cases.json")) as f:
        want = json.load(f)["deep_amplicon"]
    paths = write_deep_amplicon(str(tmp_path))
    assert [os.path.basename(p) for p in paths] == want["files"]
    status, out, err = run_cli(want["options"] + paths)
    assert status == 0, err
    lines = out.split(b"\n")
    assert [n[1:].decode() for n in lines[0:-1:2]] == want["names"]
    assert sum(len(x) for x in lines[1:-1:2]) == want["bases"]
    assert hashlib.md5(out).hexdigest() == want["md5"]
