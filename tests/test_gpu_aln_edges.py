"""The aligner on the device at its structural edges, against edlib (the unmodified reference where oracle/_ref is built,
otherwise the oracle's restatement): lengths at the 64-row words, 2048 rows (32 lanes x 64), both sides of edlib's switch
from its traceback to Hirschberg, max_len and max_len + 1, skewed and unrelated pairs (many rounds of band doubling), all
in one shuffled batch and in reverse order; the 10-kb / 12 % shape of bench config 5 with breaking points; every pair by
reference (rp_aln_add_overlap_ref), with reverse-complemented queries, equal to the pair by pointer."""
import numpy as np
import pytest

from oracle import bindings as ob
from tests import util

pytestmark = pytest.mark.gpu

MAX_LEN = 20000
RP_ALN_TOO_LONG = 6
COMP = bytes.maketrans(b"ACGT", b"TGCA")


def _rand(rng, n):
    return bytes(util.BASES[i] for i in rng.integers(4, size=n))


def _expected(q, t):
    c, d = ob.ref_edlib_cigar(q, t) if ob.have_ref() else ob.oracle_myers_cigar(q, t)
    return c.encode(), d


def edge_pairs(seed=1):
    """(query, target) pairs at the length edges, each with the status it must get under max_len = MAX_LEN"""
    rng = np.random.default_rng(seed)
    out = []
    for n in (63, 64, 65, 127, 128, 2047, 2048, 2049, 4095, 4096, 4097, 16383, 16384):
        for err in (0.01, 0.12, 0.3):
            t = _rand(rng, n)
            q = util.mutate(rng, t, err) or t[:1]
            out.append(((q, t), 0))
        t = _rand(rng, n)                   # query of exactly n bases too (substitutions only)
        out.append(((bytes(b if rng.random() > 0.1 else util.BASES[(util.BASES.index(b) + 1) % 4] for b in t), t), 0))
    for lq, lt in ((150, 8000), (8000, 150), (1, 3000), (3000, 1)):    # skewed
        t = _rand(rng, lt)
        o = int(rng.integers(0, max(1, lt - lq)))
        q = util.mutate(rng, t[o:o + lq], 0.1) if lq < lt else _rand(rng, lq)
        out.append(((q or b"A", t), 0))
    for n in (500, 3000, 9000):             # unrelated: the band doubles up to the whole matrix
        out.append(((_rand(rng, n), _rand(rng, n + 37)), 0))
    t = _rand(rng, MAX_LEN + 1)
    out.append(((util.mutate(rng, t[:MAX_LEN], 0.05)[:MAX_LEN - 3], t[:MAX_LEN]), 0))
    out.append(((t[:MAX_LEN], t[:MAX_LEN]), 0))
    out.append(((t[:500], t), RP_ALN_TOO_LONG))
    out.append(((t, t[:500]), RP_ALN_TOO_LONG))
    return out


def frag_pairs(seed, n):
    """bench config 5's shape: 8-12 kb reads, 12 % error"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        t = _rand(rng, int(rng.integers(8000, 12000)))
        out.append((util.mutate(rng, t, 0.12), t))
    return out


def test_aln_length_edges_mixed_shuffled_and_reversed():
    from racon_b200 import api
    cases = edge_pairs()
    perm = np.random.default_rng(2).permutation(len(cases))
    pairs = [cases[i][0] for i in perm]
    want_st = [cases[i][1] for i in perm]
    got = api.align(pairs, max_len=MAX_LEN)
    rev = api.align(pairs[::-1], max_len=MAX_LEN)
    assert rev[::-1] == got, "results depend on the order of the batch"
    for (q, t), st_want, (cig, dist, st) in zip(pairs, want_st, got):
        assert st == st_want, (len(q), len(t), st)
        if st:
            assert cig == b""
            continue
        assert (cig, dist) == _expected(q, t), (len(q), len(t), dist)


def test_aln_config5_shape_against_edlib_with_breaking_points():
    from racon_b200 import api
    pairs = frag_pairs(3, 48 if ob.have_ref() else 4)
    b = api.AlnBatch()
    try:
        b.set_window_length(500)
        begins = [int(k * 977) for k in range(len(pairs))]
        starts = [int(k * 13) for k in range(len(pairs))]
        for (q, t), tb, qs in zip(pairs, begins, starts):
            assert b.add(q, t, t_begin=tb, q_start=qs)
        b.run()
        b.sync()
        for i, ((q, t), tb, qs) in enumerate(zip(pairs, begins, starts)):
            cig, dist, st = b.fetch(i)
            assert st == 0 and (cig, dist) == _expected(q, t), i
            assert np.array_equal(b.fetch_breaking_points(i), ob.oracle_breaking_points(cig, tb, tb + len(t), qs, 500)), i
    finally:
        b.close()


def test_aln_by_reference_with_reverse_complement_equals_by_pointer():
    from racon_b200 import api
    rng = np.random.default_rng(4)
    cases = [c for c, st in edge_pairs(5) if st == 0 and len(c[0]) <= 4097 and len(c[1]) <= 4097]
    cases += frag_pairs(6, 6)
    reads, refs = [], []
    for k, (q, t) in enumerate(cases):
        pre_q, pre_t = _rand(rng, int(rng.integers(0, 50))), _rand(rng, int(rng.integers(0, 300)))
        stored_q = pre_q + q + _rand(rng, 20)
        if k % 2:
            stored_q = stored_q.translate(COMP)[::-1]
        reads += [pre_t + t + b"GATTACA", stored_q]
        refs.append((2 * k + 1, len(pre_q), len(q), k % 2, 2 * k, len(pre_t), len(t)))
    store = api.ReadStore(reads)
    a, b = api.AlnBatch(), api.AlnBatch()
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
            assert a.fetch(i) == b.fetch(i) and a.fetch(i)[2] == 0, i
            assert np.array_equal(a.fetch_breaking_points(i), b.fetch_breaking_points(i)), i
    finally:
        a.close()
        b.close()
        store.close()
