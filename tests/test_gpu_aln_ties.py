"""The aligner (myers_core.cuh) where edlib's tie rules decide the CIGAR, and at its regime, band, alphabet and
run-capacity edges, against edlib (the unmodified reference where oracle/_ref is built, otherwise the oracle's
restatement).

edlib's alignment depends only on exact edit distances: its traceback priority below the 1 MiB rule, its smallest
split row above it.  That only shows on input with many co-optimal alignments: homopolymer-length errors, tandem
repeats, low-complexity runs.  Every pair here must either equal edlib in CIGAR and distance (status 0) or get exactly
the soft status that `predicted_status` (a restatement of the kernel's limits) gives it, with an empty CIGAR.  Every
generator asserts that it reached its edge; the short-query regime-switch pairs must also change their CIGAR when the
rule is moved across them, so that a wrong regime choice cannot go unseen.

The GPU tests are marked `gpu`; their CPU twins run the same device code through the warp simulation (tests/simlib.py)
at sizes it handles quickly."""
import ctypes as C
import functools
import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle import bindings as ob
from tests import simlib, util
from tests import test_myers_oracle as tm

MAX_LEN = 20000
RP_ALN_BAND_LIMIT, RP_ALN_ALPHABET_LIMIT, RP_ALN_RUN_LIMIT, RP_ALN_TOO_LONG = 1, 2, 5, 6
K_FIRST = 64 * 29          # the first threshold of the distance pass: the widest band of one 32-word round
ALN_SLOTS = 8              # band words per lane (kAlnSlots): bands of up to 256 words
MAX_SYMS = 16              # distinct bytes per pair (kAlnMaxSyms)
RULE = ob.EDLIB_RULE
COMP = bytes.maketrans(b"ACGT", b"TGCA")   # racon complements A, C, G, T and leaves every other byte as it is


# ------------------------------------------------------------------------------------------------------------------
# restatement of the kernel's limits
# ------------------------------------------------------------------------------------------------------------------

def band_span(n, m, k):
    """Band words of an (n x m) pass with threshold k (AlnWarp::band_span; k >= |n - m|)."""
    delta = n - m
    rows = (k + delta) // 2 + (k - delta) // 2 + 1
    return min((rows + 63) // 64 + 1, (n + 63) // 64)


def k_schedule(n, m, d):
    """The thresholds the distance pass runs with, up to the first that reaches distance d: K_FIRST, doubled each
    time, clipped at max(n, m), skipped while below |n - m|."""
    out, k = [], K_FIRST
    while True:
        if k >= abs(n - m):
            out.append(min(k, max(n, m)))
            if d <= out[-1]:
                return out
        k *= 2


def run_cap(n, m):
    """Runs the device keeps for a pair (rp_api.cu: aln_add_metadata)."""
    return (n + m) // 3 + 64


def n_runs(cigar):
    return len(re.findall(r"[MID]", cigar))


def predicted_status(q, t, cigar, d, max_len=MAX_LEN):
    """The status the kernel must give (q, t), whose edlib alignment is (cigar, d).  Only the distance pass can hit
    the band limit: a Hirschberg node or a leaf runs with k = its score <= d, so its band is never wider than that of
    the pass that found d, and a leaf's store (< 1 MiB / 20 B words) always fits."""
    n, m = len(q), len(t)
    if n > max_len or m > max_len:
        return RP_ALN_TOO_LONG
    if len(set(q) | set(t)) > MAX_SYMS:
        return RP_ALN_ALPHABET_LIMIT
    if n and m and any(band_span(n, m, k) > 32 * ALN_SLOTS for k in k_schedule(n, m, d)):
        return RP_ALN_BAND_LIMIT
    if n_runs(cigar) > run_cap(n, m):
        return RP_ALN_RUN_LIMIT
    return 0


@functools.lru_cache(maxsize=None)
def edlib(q, t):
    return ob.ref_edlib_cigar(q, t) if ob.have_ref() else ob.oracle_myers_cigar(q, t)


def expect_all(pairs):
    """edlib's answer on every pair, computed in parallel (the checkers release the GIL)."""
    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        return list(ex.map(lambda p: edlib(*p), pairs))


def check(pairs, got):
    """got: [(cigar bytes or str, distance, status)] of the device or the simulation for pairs."""
    assert len(got) == len(pairs)
    for (q, t), (cig, dist, st), (want_cig, want_d) in zip(pairs, got, expect_all(pairs)):
        cig = cig.decode() if isinstance(cig, bytes) else cig
        want_st = predicted_status(q, t, want_cig, want_d)
        assert st == want_st, (len(q), len(t), st, want_st)
        if st:
            assert cig == "" and dist == -1, (len(q), len(t), st)
        else:
            assert (cig, dist) == (want_cig, want_d), (len(q), len(t), dist, want_d)


def sim_run(pairs, **kw):
    got, st = simlib.sim_align(pairs, max_len=MAX_LEN, **kw)
    return [(c, d, int(s)) for (c, d), s in zip(got, st)]


def gpu_run(pairs):
    from racon_b200 import api
    return api.align(pairs, max_len=MAX_LEN)


# ------------------------------------------------------------------------------------------------------------------
# generators
# ------------------------------------------------------------------------------------------------------------------

def _runs(rng, n, alphabet=util.BASES):
    """n bases of homopolymer runs (mean length about 3)."""
    out, prev = bytearray(), -1
    while len(out) < n:
        c = int(rng.integers(len(alphabet)))
        if c != prev:
            out += bytes([alphabet[c]]) * int(rng.geometric(0.35))
            prev = c
    return bytes(out[:n])


def _stretch(rng, short, length):
    """`short` with every homopolymer run lengthened by a random factor, cut or padded to `length` bases."""
    f = length / len(short)
    out = bytearray()
    for mo in re.finditer(rb"(.)\1*", short):
        out += mo.group(1) * max(1, int(round(len(mo.group(0)) * f * rng.uniform(0.6, 1.4))))
    out = out[:length]
    pad = util.BASES[(util.BASES.index(out[-1]) + 1) % 4]
    return bytes(out) + bytes([pad]) * (length - len(out))


def _other_rule(ql, tl):
    """The rule that moves the (ql x tl) node to edlib's other regime and changes no smaller node."""
    data = ob.edlib_data_bytes(ql, tl)
    return data + 1 if data >= RULE else data


def discriminates(q, t, rule):
    return ob.oracle_myers_cigar(q, t)[0] != ob.oracle_myers_cigar(q, t, rule=rule)[0]


def _regime_pair(n, m, seed):
    """A homopolymer-run pair of n x m bases.  With the query the shorter, its CIGAR must change when the whole pair is
    moved to edlib's other regime.  With the query 12 times the longer (the 102-block solution) no pair was found that
    does: the optimal paths have next to no deletions, and where the path crosses the split column by an
    insertion or a diagonal step the up-first traceback and the smallest split row choose the same row.  Those pairs
    carry a deletion/substitution tie at the split column instead, and still must equal edlib."""
    for s in range(40):
        rng = np.random.default_rng(seed * 1000 + s)
        if n <= m:
            q = _runs(rng, n)
            t = _stretch(rng, q, m)
            if discriminates(q, t, _other_rule(n, m)):
                return q, t
        else:
            x = int(rng.integers(20, 60))
            pos = m // 2 - int(rng.integers(5, x - 5))
            t1, t2 = _runs(rng, pos), _runs(rng, m - pos - x)
            t = t1 + _runs(rng, x) + t2
            q = t1 + _runs(rng, x - int(rng.integers(3, 15))) + t2
            return _runs(rng, n - len(q)) + q, t
    raise AssertionError("no discriminating %d x %d pair" % (n, m))


def rule_equalities(max_len=MAX_LEN):
    """(query blocks, target length) where edlib's data 20 * blocks * m + 8 * m is exactly 1 MiB."""
    return [(b, RULE // (20 * b + 8)) for b in range(1, (max_len + 63) // 64 + 1)
            if RULE % (20 * b + 8) == 0 and RULE // (20 * b + 8) <= max_len]


REGIME_SHAPES = []
for _blocks, _m in ((6, 8192), (102, 512)):
    _lo, _hi = 64 * (_blocks - 1) + 1, 64 * _blocks
    REGIME_SHAPES += [(_lo, _m - 1), (_lo, _m), (_lo, _m + 1), (_hi, _m - 1), (_hi, _m), (_hi, _m + 1),
                      (_lo - 1, _m), (_hi + 1, _m)]


@functools.lru_cache(maxsize=None)
def regime_pairs():
    """Pairs around the two exact solutions of the rule: target lengths m - 1, m, m + 1 at the first and last query
    length of the block count, and the query lengths one block below and above."""
    assert rule_equalities() == [(6, 8192), (102, 512)]
    out = [_regime_pair(n, m, i) for i, (n, m) in enumerate(REGIME_SHAPES)]
    at_rule = [ob.edlib_data_bytes(len(q), len(t)) == RULE for q, t in out]
    assert sum(at_rule) == 4
    return out


@functools.lru_cache(maxsize=None)
def hirschberg_child_on_rule_pair():
    """A ~700-base query against a 16 384-base target whose first split gives a child of 6 query blocks x 8 192
    columns, exactly on the rule; moving the rule by one byte must change the CIGAR."""
    for seed in range(60):
        rng = np.random.default_rng(7000 + seed)
        q = _runs(rng, int(rng.integers(660, 760)))
        t = _stretch(rng, q, 16384)
        tree = ob.oracle_myers_tree(q, t)
        on_rule = [(a, b) for a, b, _, _ in tree[1:] if ob.edlib_data_bytes(a, b) == RULE]
        if on_rule and discriminates(q, t, RULE + 1):
            assert tree[0, 3] == 0 and all(b == 8192 and 321 <= a <= 384 for a, b in on_rule)
            return q, t
    raise AssertionError("no Hirschberg pair with a discriminating child on the rule")


def _children(tree, i):
    """The two leaves that are the children of split node i, or None."""
    if i + 2 >= len(tree) or not (tree[i + 1, 3] and tree[i + 2, 3]):
        return None
    a, b = tree[i + 1], tree[i + 2]
    return (a, b) if a[0] + b[0] == tree[i, 0] and a[1] + b[1] == tree[i, 1] else None


@functools.lru_cache(maxsize=None)
def word_band_pairs():
    """{(kind, words): pair}: a Hirschberg split whose forward and reverse passes have a band of exactly 16 words (one
    per half-warp) and of 17 (one after the other), and sibling leaves whose wider band is exactly 16 words (filled
    side by side) and 17 (one at a time)."""
    rng = np.random.default_rng(31)
    found = {}
    for i in range(40):   # top-level splits: 2.5-kb pairs around distance 900-1020
        t = tm._rand(rng, 2500)
        q = util.mutate(rng, t, 0.42 + 0.005 * i)
        tree = ob.oracle_myers_tree(q, t)
        for a, b, s, leaf in tree:
            if not leaf and band_span(a, b, s) in (16, 17):
                found.setdefault(("split", band_span(a, b, s)), (q, t))
        if ("split", 16) in found and ("split", 17) in found:
            break
    for i in range(60):   # sibling leaves of about 2 000 x 1 500 with scores near 1 000
        t = tm._rand(rng, 3000)
        q = util.mutate(rng, t, float(rng.uniform(0.25, 0.4)))
        q += tm._rand(rng, max(0, int(rng.integers(3600, 4300)) - len(q)))
        tree = ob.oracle_myers_tree(q, t)
        for k in range(len(tree)):
            kids = None if tree[k, 3] else _children(tree, k)
            if kids:
                w = max(band_span(*c[:3]) for c in kids)
                if w in (16, 17):
                    found.setdefault(("leaves", w), (q, t))
        if ("leaves", 16) in found and ("leaves", 17) in found:
            break
    assert sorted(found) == [("leaves", 16), ("leaves", 17), ("split", 16), ("split", 17)], sorted(found)
    return found


def distance_pass_pairs():
    """Distance 1 856 (the first threshold) and 1 857 (one doubling): a tie-rich target with that many bases deleted
    from its middle; and A^2100 x C^1550, a traceback-regime pair whose stored distance pass has a 33-word band."""
    rng = np.random.default_rng(41)
    t = _runs(rng, 4000)
    out = [(t[:1000] + t[1000 + d:], t) for d in (K_FIRST, K_FIRST + 1)]
    for (q, t), d in zip(out, (K_FIRST, K_FIRST + 1)):
        assert edlib(q, t)[1] == d
        assert k_schedule(len(q), len(t), d) == ([K_FIRST] if d == K_FIRST else [2 * K_FIRST])
    for q, t in ((b"A" * 2100, b"C" * 1550), (b"A" * 2100, b"CG" * 775)):
        assert ob.edlib_data_bytes(len(q), len(t)) < RULE
        assert [band_span(len(q), len(t), k) for k in k_schedule(len(q), len(t), 2100)] == [31, 33]
        out.append((q, t))
    return out


def band_limit_pairs():
    """The last distance the widest band (256 words) reaches, and one more: A^16384 x C^16384 (distance 16 384: the
    band clips to the query's 256 words) and A^16385 x C^16385 (k reaches 16 385 and needs 257 words); for a
    16 400-base query, distance 14 848 (the last doubling that fits) and 14 849."""
    out = [(b"A" * 16384, b"C" * 16384), (b"A" * 16385, b"C" * 16385)]
    for p in (16400 - 14848, 16400 - 14849):
        out.append((b"A" * 16400, b"A" * p + b"C" * (16400 - p)))
    return out, [0, RP_ALN_BAND_LIMIT, 0, RP_ALN_BAND_LIMIT]


def _alternating_indels(rng, length):
    """A random target and every other base of it as the query (edlib's CIGAR has about 0.5 runs per base of the
    pair, the cap one third)."""
    t = tm._rand(rng, length)
    return t[int(rng.integers(2))::2], t


@functools.lru_cache(maxsize=None)
def run_cap_pairs(length):
    """Pairs of `length` bases and a tail whose edlib CIGAR has exactly run_cap and run_cap + 1 runs: alternating
    indels dense enough to exceed the cap, then a tail matched on both sequences that raises the cap one step at a
    time."""
    out = []
    for excess in (0, 1):
        for seed in range(20):
            rng = np.random.default_rng(100 * length + 10 * excess + seed)
            q, t = _alternating_indels(rng, length)
            runs = n_runs(edlib(q, t)[0])
            tail = b""
            while run_cap(len(q) + len(tail), len(t) + len(tail)) < runs - excess:
                tail += tm._rand(rng, 1)
            cig = edlib(q + tail, t + tail)[0]
            if n_runs(cig) == run_cap(len(q) + len(tail), len(t) + len(tail)) + excess:
                out.append((q + tail, t + tail))
                break
        else:
            raise AssertionError("no pair with run_cap + %d runs at %d bases" % (excess, length))
    return out


ALPHABET_16 = [0x00, 0x1f, 0x20, 0x41, 0x43, 0x61, 0x63, 0x7f, 0x80, 0x9c, 0xa0, 0xc5, 0xd1, 0xe0, 0xf7, 0xff]


def alphabet_pairs():
    """Pairs with exactly 16 and 17 distinct bytes: bytes from all eight 32-value ranges of the kernel's alphabet
    bitmap (>= 0x80 included), upper and lower case of the same base, a byte that occurs in the query only and one in
    the target only; the 17th byte in each range in turn.  A Hirschberg-regime pair has all 16."""
    rng = np.random.default_rng(51)
    sym = bytes(ALPHABET_16)
    assert len({c >> 5 for c in sym}) == 8
    out = []
    for n in (300, 1500, 3000):
        shared = sym[1:15]
        t = _runs(rng, n, shared)
        q = util.mutate(rng, t, 0.15, shared)
        q, t = q + sym[0:1] + q[:20], t + sym[15:16] + t[-20:]    # 0x00 in the query only, 0xff in the target only
        out.append(((q, t), 0))
    q, t = out[0][0]
    extra = [0x02, 0x3a, 0x44, 0x62, 0x90, 0xa5, 0xd3, 0xfe]
    assert sorted({c >> 5 for c in extra}) == list(range(8)) and not set(extra) & set(sym)
    for k, c in enumerate(extra):
        out.append(((q + bytes([c]), t) if k % 2 else (q, bytes([c]) + t), RP_ALN_ALPHABET_LIMIT))
    for (q, t), st in out:
        assert len(set(q) | set(t)) == (16 if st == 0 else 17)
    return out


def tie_set(lengths):
    return [(q, t) for n in lengths for _, q, t in tm.tie_rich_pairs(2000 + n, n)]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the generators reach their edges, and the simulation of the device code
# ------------------------------------------------------------------------------------------------------------------

def test_restatement_of_the_limits():
    assert k_schedule(100, 100, 5) == [100]
    assert k_schedule(5000, 100, 4950) == [5000]                 # 1856 and 3712 < |n - m| are skipped
    assert k_schedule(20000, 20000, 10000) == [1856, 3712, 7424, 14848]
    assert band_span(2048, 2048, K_FIRST) == 31 and band_span(16384, 16384, 16384) == 256
    assert band_span(16385, 16385, 16385) == 257
    assert run_cap(1000, 1000) == 730
    assert predicted_status(b"A" * 3, b"AB" * 9, "", 0, max_len=17) == RP_ALN_TOO_LONG


def test_sim_tie_rich_set():
    pairs = tie_set((100, 700))
    perm = np.random.default_rng(3).permutation(len(pairs))
    shuffled = [pairs[i] for i in perm]
    got = sim_run(shuffled)
    assert sim_run(shuffled[::-1])[::-1] == got, "results depend on the order of the batch"
    check(shuffled, got)
    pairs = tie_set((2500,))
    check(pairs, sim_run(pairs))


def test_sim_regime_switch_at_exact_equality():
    """The 102-block shapes, the 6-block shapes at the first query length of the block, and the Hirschberg child on
    the rule (the other 8 192-column pairs only run on the device)."""
    pairs = [(q, t) for q, t in regime_pairs() if len(t) < 1024 or len(q) == 321] + [hirschberg_child_on_rule_pair()]
    assert len(pairs) == 12
    check(pairs, sim_run(pairs))


def test_sim_band_edges():
    lib = simlib.lib()
    lib.rp_sim_leaf_pairs.restype = C.c_ulong
    words = word_band_pairs()
    for key in sorted(words):
        before = lib.rp_sim_leaf_pairs()
        check([words[key]], sim_run([words[key]]))
        if key == ("leaves", 16):
            assert lib.rp_sim_leaf_pairs() > before      # the 16-word siblings shared the warp
    pairs = distance_pass_pairs()
    check(pairs, sim_run(pairs))


def test_sim_band_limit():
    pairs, want = band_limit_pairs()
    got = sim_run(pairs[1:2])
    assert [g[2] for g in got] == want[1:2]
    check(pairs[1:2], got)


@pytest.mark.parametrize("length", [900, 2400])
def test_sim_run_capacity(length):
    pairs = run_cap_pairs(length)
    for (q, t), excess in zip(pairs, (0, 1)):
        got = sim_run([(q, t)], run_stride=run_cap(len(q), len(t)))
        assert got[0][2] == (RP_ALN_RUN_LIMIT if excess else 0)
        check([(q, t)], got)
    q, t = pairs[0]
    (cig, d, bp), = simlib.sim_align_bp([(q, t, 777, 31)], 500)[0]
    assert (cig, d) == edlib(q, t)
    assert np.array_equal(bp, ob.oracle_breaking_points(cig, 777, 777 + len(t), 31, 500))


def test_sim_alphabet_edges():
    cases = alphabet_pairs()
    got = sim_run([p for p, _ in cases])
    assert [g[2] for g in got] == [st for _, st in cases]
    check([p for p, _ in cases], got)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_tie_rich_set_shuffled_and_reversed():
    pairs = tie_set((100, 700, 3000, 12000))
    perm = np.random.default_rng(4).permutation(len(pairs))
    shuffled = [pairs[i] for i in perm]
    got = gpu_run(shuffled)
    assert gpu_run(shuffled[::-1])[::-1] == got, "results depend on the order of the batch"
    check(shuffled, got)


@pytest.mark.gpu
def test_regime_switch_at_exact_equality():
    pairs = regime_pairs() + [hirschberg_child_on_rule_pair()]
    check(pairs, gpu_run(pairs))


@pytest.mark.gpu
def test_band_edges():
    words = word_band_pairs()
    pairs = [words[k] for k in sorted(words)] + distance_pass_pairs()
    limit, want = band_limit_pairs()
    got = gpu_run(pairs + limit)
    assert [g[2] for g in got[len(pairs):]] == want
    assert got[len(pairs)][1] == 16384
    check(pairs + limit, got)


@pytest.mark.gpu
def test_run_capacity():
    from racon_b200 import api
    pairs = run_cap_pairs(900) + run_cap_pairs(2400)
    b = api.AlnBatch(max_len=MAX_LEN)
    try:
        b.set_window_length(500)
        for q, t in pairs:
            assert b.add(q, t, t_begin=777, q_start=31)
        b.run()
        b.sync()
        got = [b.fetch(i) for i in range(len(pairs))]
        assert [g[2] for g in got] == [0, RP_ALN_RUN_LIMIT] * 2
        check(pairs, got)
        for i in (0, 2):
            q, t = pairs[i]
            want = ob.oracle_breaking_points(got[i][0], 777, 777 + len(t), 31, 500)
            assert np.array_equal(b.fetch_breaking_points(i), want), i
    finally:
        b.close()


@pytest.mark.gpu
def test_alphabet_edges():
    cases = alphabet_pairs()
    got = gpu_run([p for p, _ in cases])
    assert [g[2] for g in got] == [st for _, st in cases]
    check([p for p, _ in cases], got)


@pytest.mark.gpu
def test_by_reference_tie_rich_and_iupac_equal_by_pointer():
    """Tie-rich and IUPAC-bearing pairs named as slices of a device-resident store, every other query stored as its
    reverse complement (racon's: A, C, G, T only), equal the same pairs added by pointer, breaking points included."""
    from racon_b200 import api
    rng = np.random.default_rng(61)
    cases = tie_set((100, 700, 3000))
    iupac = b"ACGTNRYKMSWBacgtn"[:16]
    for n in (400, 2600):
        t = _runs(rng, n, iupac)
        cases.append((util.mutate(rng, t, 0.12, iupac) or b"N", t))
    reads, refs = [], []
    for k, (q, t) in enumerate(cases):
        pre_q, pre_t = tm._rand(rng, int(rng.integers(0, 50))), tm._rand(rng, int(rng.integers(0, 300)))
        stored_q = pre_q + q + tm._rand(rng, 20)
        if k % 2:
            stored_q = stored_q.translate(COMP)[::-1]
        reads += [pre_t + t + b"GATTACA", stored_q]
        refs.append((2 * k + 1, len(pre_q), len(q), k % 2, 2 * k, len(pre_t), len(t)))
    store = api.ReadStore(reads)
    a, b = api.AlnBatch(max_len=MAX_LEN), api.AlnBatch(max_len=MAX_LEN)
    try:
        for batch in (a, b):
            batch.set_window_length(500)
        for (q, t), r in zip(cases, refs):
            assert a.add_ref(store, *r)
            assert b.add(q, t, t_begin=r[5], q_start=r[1])
        for batch in (a, b):
            batch.run()
            batch.sync()
        for i in range(len(cases)):
            assert a.fetch(i) == b.fetch(i), i
            assert np.array_equal(a.fetch_breaking_points(i), b.fetch_breaking_points(i)), i
        check(cases, [a.fetch(i) for i in range(len(cases))])
    finally:
        a.close()
        b.close()
        store.close()


@pytest.mark.gpu
def test_lambda_fragment_correction_cigars():
    """The 7 780 all-vs-all overlaps of the -f configuration: every CIGAR equals edlib's (every 50th the
    restatement's where the unmodified edlib is not built), and none reaches a soft status."""
    from racon_b200 import api
    from tests.lambda_overlaps import LambdaOverlaps
    lam = LambdaOverlaps("lambda_frag_overlaps.npz")
    pairs = [lam.spans(k)[:2] for k in range(lam.n_overlaps())]
    got = api.align(pairs)
    assert all(st == 0 for _, _, st in got)
    idx = range(len(pairs)) if ob.have_ref() else range(0, len(pairs), 50)
    want = expect_all([pairs[k] for k in idx])
    for k, (cig, d) in zip(idx, want):
        assert got[k][:2] == (cig.encode(), d), k
