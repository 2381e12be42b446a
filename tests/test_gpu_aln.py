"""Batched pre-alignment on the GPU through the C ABI (rp_aln_*): CIGAR strings byte-identical to what
Overlap::align_overlaps (src/overlap.cpp:205-224) gets from edlib — checked against the oracle restatement and,
where oracle/_ref is built, the unmodified edlib itself."""
import numpy as np
import pytest

from oracle import bindings as ob
from tests import util

pytestmark = pytest.mark.gpu


def _pair(rng, n, err, skew=0.0):
    t = bytes(util.BASES[i] for i in rng.integers(4, size=n))
    q = util.mutate(rng, t, err)
    if skew:
        k = int(len(q) * skew)
        q = q[k // 2:len(q) - k // 2]
    return q or b"A", t


def _expected(q, t):
    c, d = (ob.ref_edlib_cigar(q, t) if ob.have_ref() else ob.oracle_myers_cigar(q, t))[:2]
    return (c.encode() if isinstance(c, str) else c), d


def _check(pairs, **kw):
    from racon_b200 import api
    got = api.align(pairs, **kw)
    assert len(got) == len(pairs)
    for (q, t), (cig, dist, st) in zip(pairs, got):
        assert st == 0, (len(q), len(t), st)
        exp = _expected(q, t)
        assert (cig, dist) == exp, (len(q), len(t), dist, exp[1])


def test_aln_degenerate_and_small():
    pairs = [(b"A", b"A"), (b"A", b"C"), (b"ACGT", b"A"), (b"A", b"ACGT"), (b"AAAA", b"TTTT"), (b"ACGTACGT", b"ACGT"),
             (b"ACGTTGCA" * 9, b"ACGTTGCA" * 9), (b"ACGT" * 40, b"ACGT" * 5), (b"", b"ACG"), (b"ACG", b"")]
    from racon_b200 import api
    got = api.align(pairs)
    for (q, t), (cig, dist, st) in zip(pairs, got):
        assert st == 0
        if not q or not t:   # edlib.cpp:1136-1143: all D / all I
            assert cig == (b"%d%s" % (len(q) + len(t), b"D" if not q else b"I"))
            assert dist == len(q) + len(t)
        else:
            assert (cig, dist) == _expected(q, t)


def test_aln_traceback_regime_mixed_lengths():
    rng = np.random.default_rng(11)
    pairs = []
    for n in (30, 63, 64, 65, 127, 128, 129, 200, 500, 700, 1000, 1500, 2000):
        for err in (0.02, 0.12, 0.3):
            pairs.append(_pair(rng, n, err, skew=float(rng.choice([0.0, 0.2]))))
    _check(pairs)


def test_aln_hirschberg_regime():
    rng = np.random.default_rng(12)
    pairs = [_pair(rng, n, err, skew=float(rng.choice([0.0, 0.1])))
             for n, err in [(2500, 0.12), (3500, 0.05), (3000, 0.3), (6000, 0.15), (9000, 0.1), (12000, 0.12)]]
    _check(pairs)


def test_aln_many_pairs_queue_and_order():
    rng = np.random.default_rng(13)
    pairs = [_pair(rng, int(rng.integers(50, 900)), float(rng.uniform(0.0, 0.25))) for _ in range(400)]
    _check(pairs)


def test_aln_soft_failures():
    from racon_b200 import api
    rng = np.random.default_rng(14)
    ok = _pair(rng, 300, 0.1)
    many_syms = (bytes(range(65, 65 + 20)) * 10, bytes(range(65, 65 + 20)) * 10)
    too_long = (b"A" * 3000, b"A" * 3000)
    iupac = (b"ACGTNRYKMSWB" * 30 + b"ACGT" * 50, b"ACGTNRYKMSW" * 30 + b"ACGA" * 55)   # 12 symbols: fine
    got = api.align([ok, many_syms, too_long, ok, iupac], max_len=2048)
    assert got[0][2] == 0 and got[3][2] == 0 and got[0] == got[3]
    assert got[0][0] == _expected(*ok)[0]
    assert got[4][2] == 0 and (got[4][0], got[4][1]) == _expected(*iupac)
    assert got[1][2] == 2 and got[1][0] == b""      # RP_ALN_ALPHABET_LIMIT (> 16 distinct characters)
    assert got[2][2] == 6 and got[2][0] == b""      # RP_ALN_TOO_LONG
    # unrelated sequences: the band doubles until k = 14 848 reaches the distance (about 10 k), within 256 words;
    # the status is the one the restatement of the kernel's limits predicts
    from tests.test_gpu_aln_ties import predicted_status
    a = bytes(util.BASES[i] for i in rng.integers(4, size=20000))
    b = bytes(util.BASES[i] for i in rng.integers(4, size=20000))
    (cig, dist, st), = api.align([(a, b)])
    want_cig, want_d = _expected(a, b)
    assert st == predicted_status(a, b, want_cig.decode(), want_d) == 0
    assert (cig, dist) == (want_cig, want_d)


def test_aln_batch_reuse_and_state_errors():
    from racon_b200 import api
    rng = np.random.default_rng(15)
    b = api.AlnBatch()
    with pytest.raises(api.RaconB200Error):
        b.launch()
    p1, p2 = _pair(rng, 400, 0.1), _pair(rng, 800, 0.2)
    for pr in (p1, p2):
        b.reset()
        assert b.add(*pr)
        b.run()
        b.sync()
        assert b.fetch(0)[0] == _expected(*pr)[0]
    with pytest.raises(api.RaconB200Error):
        b.fetch(5)
    b.reset()
    b.run()
    b.sync()
    assert b.size() == 0
    b.close()


def test_aln_host_mirror_batch_aligner():
    """racon_b200::BatchAligner (mirror of CUDABatchAligner) driven in small batches, as cudapolisher.cpp:100-213."""
    from racon_b200 import api
    rng = np.random.default_rng(16)
    pairs = [_pair(rng, int(rng.integers(100, 3000)), float(rng.uniform(0.02, 0.2))) for _ in range(60)]
    got = api.mirror_align(pairs, max_alignments=7)
    for (q, t), c in zip(pairs, got):
        assert c == _expected(q, t)[0]


def _cigar_cost(cigar, q, t):
    """(query bases, target bases, edit operations) implied by a CIGAR on the two sequences"""
    import re
    qa = np.frombuffer(q, np.uint8)
    ta = np.frombuffer(t, np.uint8)
    i = j = cost = 0
    for cnt, op in re.findall(rb"(\d+)([MID])", cigar):
        c = int(cnt)
        if op == b"M":
            cost += int((qa[i:i + c] != ta[j:j + c]).sum())
            i += c
            j += c
        elif op == b"I":
            cost += c
            i += c
        else:
            cost += c
            j += c
    return i, j, cost


def test_aln_full_size_properties():
    """BASELINE config 5's shape (10-kb reads, 12 % error), checked through properties that need no oracle: every
    CIGAR consumes exactly both sequences, its own cost equals the reported edit distance, and the distance is
    symmetric (query and target swapped in a second batch)."""
    from racon_b200 import api
    rng = np.random.default_rng(17)
    pairs = []
    for _ in range(1500):
        n = int(rng.integers(8000, 12000))
        t = bytes(util.BASES[i] for i in rng.integers(4, size=n))
        pairs.append((util.mutate(rng, t, 0.12), t))
    fwd = api.align(pairs)
    rev = api.align([(t, q) for q, t in pairs])
    for (q, t), (cig, dist, st), (_, rdist, rst) in zip(pairs, fwd, rev):
        assert st == 0 and rst == 0
        assert _cigar_cost(cig, q, t) == (len(q), len(t), dist)
        assert dist == rdist
