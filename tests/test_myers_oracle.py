"""Pins oracle/myers_oracle.cpp (the plain-DP restatement of what racon asks of edlib, SURVEY.md §8 a10) against
the UNMODIFIED edlib: identical CIGAR strings and edit distances on random pairs in both of edlib's regimes
(stored-matrix traceback below 1 MiB of alignment data, Hirschberg above), on random pairs and on tie-rich pairs —
homopolymer-length errors, tandem repeats, low-complexity runs — where many alignments share the optimal distance and
only edlib's tie rules decide which one it returns.  edlib's answers are stored in tests/golden/ref_answers.json
(tests/golden/make_ref_answers.py); where oracle/_ref is built they are checked against edlib itself as well."""
import numpy as np
import pytest

from oracle import bindings as ob
from tests import util

TRACEBACK = [(1, 0.5, 20), (7, 0.3, 60), (64, 0.2, 60), (65, 0.1, 40), (300, 0.15, 40), (1500, 0.12, 12), (1900, 0.25, 8)]
HIRSCHBERG = [(2500, 0.12, 6), (4000, 0.05, 4), (6000, 0.15, 3), (3000, 0.35, 4)]
DEGENERATE = [(b"A", b"A"), (b"A", b"C"), (b"ACGT", b"A"), (b"A", b"ACGT"), (b"AAAA", b"TTTT"),
              (b"ACGTACGT", b"ACGT"), (b"ACGT" * 700, b"ACGT" * 100), (b"A" * 3000, b"A" * 2990 + b"C" * 500)]


TANDEM_UNITS = (1, 2, 3, 7, 16, 63, 64, 65)
TIES_TRACEBACK = (100, 400, 1200)       # every pair below edlib's 1 MiB rule
TIES_HIRSCHBERG = (2500, 5000)          # every pair above it


def _rand(rng, n, alphabet=util.BASES):
    return bytes(alphabet[i] for i in rng.integers(len(alphabet), size=n))


def homopolymer_pair(rng, n, err):
    """A target of homopolymer runs (mean length 3) and a query with the same runs, each run's length off by one or two
    with probability err and a rare substitution: ONT's dominant error mode."""
    runs, total, prev = [], 0, -1
    while total < n:
        c = int(rng.integers(4))
        if c == prev:
            continue
        length = int(rng.geometric(0.35))
        runs.append((c, length))
        total += length
        prev = c
    t = b"".join(bytes([util.BASES[c]]) * length for c, length in runs)
    q = bytearray()
    for c, length in runs:
        if rng.random() < err:
            length = max(0, length + int(rng.choice([-2, -1, 1, 2])))
        q += bytes([util.BASES[c]]) * length
    for i in rng.integers(len(q), size=max(1, len(q) // 200)):
        q[i] = util.BASES[(util.BASES.index(q[i]) + 1) % 4]
    return bytes(q), t


def tandem_pair(rng, unit_len, n):
    """A tandem repeat of a unit_len-base unit between two random flanks (about n bases in all); the query has 1-3
    copies more or fewer, one copy with a point error and lightly mutated flanks."""
    unit = _rand(rng, unit_len)
    flank = max(1, n // 6)
    copies = max(3, (n - 2 * flank) // unit_len)
    left, right = _rand(rng, flank), _rand(rng, flank)
    t = left + unit * copies + right
    change = int(rng.choice([-3, -2, -1, 1, 2, 3]))
    body = bytearray(unit * (copies + change))
    i = int(rng.integers(len(body)))
    body[i] = util.BASES[(util.BASES.index(body[i]) + 1) % 4]
    q = util.mutate(rng, left, 0.02) + bytes(body) + util.mutate(rng, right, 0.02)
    return q, t


def tie_rich_pairs(seed, n):
    """The tie-rich families at about n bases a side: [(family, query, target)]."""
    rng = np.random.default_rng(seed)
    out = [("homopolymer/%g" % err,) + homopolymer_pair(rng, n, err) for err in (0.05, 0.2)]
    out += [("tandem/%d" % u,) + tandem_pair(rng, u, n) for u in TANDEM_UNITS]
    d = int(rng.integers(1, max(2, n // 8)))
    out.append(("A^n/A^m", b"A" * n, b"A" * (n - d)))
    out.append(("A^n/C^m", b"A" * (n - d), b"C" * n))
    t = _rand(rng, n, b"AC")
    out.append(("two-letter", util.mutate(rng, t, 0.1, b"AC") or b"A", t))
    t = _rand(rng, n, b"GT")
    out.append(("two-letter", util.mutate(rng, t[n // 10:], 0.25, b"GT") or b"G", t))
    out.append(("AC/CA", b"AC" * (n // 2), b"CA" * (n // 2)))
    return out


def tie_pairs(n):
    return [(q, t) for _, q, t in tie_rich_pairs(1000 + n, n)]


def _pair(rng, n, err, skew=0.0):
    t = bytes(util.BASES[i] for i in rng.integers(4, size=n))
    q = util.mutate(rng, t, err)
    if skew:  # drop a prefix/suffix of the query so the lengths differ markedly
        k = int(len(q) * skew)
        q = q[k // 2:len(q) - k // 2]
    return q, t


def traceback_pairs(n, err, count):
    rng = np.random.default_rng(n)
    pairs = [_pair(rng, n, err, skew=rng.choice([0.0, 0.0, 0.2])) for _ in range(count)]
    return [(q, t) for q, t in pairs if q]


def hirschberg_pairs(n, err, count):
    rng = np.random.default_rng(n + 1)
    return [_pair(rng, n, err, skew=rng.choice([0.0, 0.1, 0.3])) for _ in range(count)]


def _check(key, pairs):
    want = util.ref_answers()["edlib"][key]
    assert [util.cigar_answer(ob.oracle_myers_cigar(q, t)) for q, t in pairs] == want
    if ob.have_ref():
        assert [util.cigar_answer(ob.ref_edlib_cigar(q, t)) for q, t in pairs] == want


@pytest.mark.parametrize("n,err,count", TRACEBACK)
def test_traceback_regime(n, err, count):
    _check("traceback/%d" % n, traceback_pairs(n, err, count))


@pytest.mark.parametrize("n,err,count", HIRSCHBERG)
def test_hirschberg_regime(n, err, count):
    _check("hirschberg/%d" % n, hirschberg_pairs(n, err, count))


def test_degenerate_pairs():
    _check("degenerate", DEGENERATE)


@pytest.mark.parametrize("n", TIES_TRACEBACK + TIES_HIRSCHBERG)
def test_tie_rich_pairs(n):
    pairs = tie_pairs(n)
    below = [ob.edlib_data_bytes(len(q), len(t)) < ob.EDLIB_RULE for q, t in pairs]
    assert all(below) if n in TIES_TRACEBACK else not any(below)
    _check("ties/%d" % n, pairs)


def test_rule_and_tree_hooks():
    """The oracle's rule parameter and node tree: edlib's rule by default; a lower rule splits the pair into a deeper
    tree whose leaves tile the target, a rule above a pair's data traces the whole pair back."""
    q, t = tie_pairs(1200)[2]
    data = ob.edlib_data_bytes(len(q), len(t))
    assert ob.oracle_myers_cigar(q, t) == ob.oracle_myers_cigar(q, t, rule=ob.EDLIB_RULE)
    tree = ob.oracle_myers_tree(q, t)
    assert tree.tolist() == [[len(q), len(t), ob.oracle_myers_cigar(q, t)[1], 1]]
    assert ob.oracle_myers_tree(q, t, rule=data).tolist()[0][3] == 0
    assert ob.oracle_myers_tree(q, t, rule=data + 1).tolist()[0][3] == 1
    rule = data // 16
    deep = ob.oracle_myers_tree(q, t, rule=rule)
    below = np.asarray([ob.edlib_data_bytes(a, b) < rule for a, b in deep[:, :2]])
    assert (below == (deep[:, 3] == 1)).all() and len(deep) == 15   # 7 splits, 8 leaves
    assert deep[deep[:, 3] == 1, 1].sum() == len(t)     # the leaves tile the target
    assert ob.oracle_myers_cigar(q, t, rule=rule)[1] == tree[0, 2]
