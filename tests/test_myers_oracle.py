"""Pins oracle/myers_oracle.cpp (the plain-DP restatement of what racon asks of edlib, SURVEY.md §8 a10) against
the UNMODIFIED edlib: identical CIGAR strings and edit distances on random pairs in both of edlib's regimes
(stored-matrix traceback below 1 MiB of alignment data, Hirschberg above).  edlib's answers are stored in
tests/golden/ref_answers.json (tests/golden/make_ref_answers.py); where oracle/_ref is built they are checked against
edlib itself as well."""
import numpy as np
import pytest

from oracle import bindings as ob
from tests import util

TRACEBACK = [(1, 0.5, 20), (7, 0.3, 60), (64, 0.2, 60), (65, 0.1, 40), (300, 0.15, 40), (1500, 0.12, 12), (1900, 0.25, 8)]
HIRSCHBERG = [(2500, 0.12, 6), (4000, 0.05, 4), (6000, 0.15, 3), (3000, 0.35, 4)]
DEGENERATE = [(b"A", b"A"), (b"A", b"C"), (b"ACGT", b"A"), (b"A", b"ACGT"), (b"AAAA", b"TTTT"),
              (b"ACGTACGT", b"ACGT"), (b"ACGT" * 700, b"ACGT" * 100), (b"A" * 3000, b"A" * 2990 + b"C" * 500)]


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
