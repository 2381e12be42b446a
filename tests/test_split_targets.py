"""Split targets without a device: the planner of the host layer (racon_b200::plan_read_groups with a window length,
api.plan_read_groups(..., t_begin=, t_end=, window_length=)) cuts a target whose own read store exceeds the budget into
maximal parts of consecutive windows and leaves every other target to the planner without splitting; the command line
takes --split-targets; a split run over the simulated runtime gives the one-group bytes (tests/test_gpu_split_targets.py
runs everything on the GPU)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from racon_b200 import api
from tests.test_cli import CONTIG, NO_DEVICE, ROOT, run_cli, sample


def _random_input(rng, fragment):
    """(n_targets, lengths, has_quality, q_id, t_id, t_begin, t_end), window_length.  Contigs: a few targets of 1 to
    hundreds of windows and reads after them, some with two overlaps; fragment (racon -f): the reads are the targets."""
    w = int(rng.choice([50, 200, 500]))
    quality = rng.random() < 0.5
    if fragment:
        n_targets = int(rng.integers(2, 60))
        lengths = rng.integers(1, 40 * w, n_targets)
        n_ov = int(rng.integers(0, 300))
        q_id = rng.integers(0, n_targets, n_ov)
        t_id = rng.integers(0, n_targets, n_ov)
    else:
        n_targets = int(rng.integers(1, 6))
        n_reads = int(rng.integers(0, 400))
        lengths = np.concatenate([rng.integers(1, int(rng.choice([2, 20, 300])) * w + 1, n_targets),
                                  rng.integers(50, 3000, n_reads)])
        q_id = np.repeat(np.arange(n_targets, n_targets + n_reads), rng.integers(1, 3, n_reads))
        t_id = rng.integers(0, n_targets, len(q_id))
    span = np.minimum(lengths[q_id], lengths[t_id])
    size = np.maximum(1, (span * rng.random(len(q_id))).astype(np.int64))
    t_begin = (rng.random(len(q_id)) * (lengths[t_id] - size + 1)).astype(np.int64)
    t_end = t_begin + size
    has_q = rng.random(len(lengths)) < (0.5 if quality else 0.0)
    return (n_targets, lengths, has_q, q_id, t_id, t_begin, t_end), w


def _n_windows(inp, w, t):
    return (int(inp[1][t]) + w - 1) // w


def _touching(inp, w, t, a, b):
    """file-order indices of the overlaps onto target t whose span touches a window in [a, b)"""
    _, _, _, _, t_id, t_begin, t_end = inp
    return np.flatnonzero((t_id == t) & (t_begin // w < b) & ((t_end - 1) // w >= a))


def _store(inp, targets, overlaps):
    _, lengths, has_q, q_id = inp[:4]
    ids = np.unique(np.concatenate([np.asarray(targets, np.int64), q_id[overlaps].astype(np.int64)]))
    return api.read_store_bytes(lengths[ids], has_q[ids])


def _own(inp, t):
    return _store(inp, [t], np.flatnonzero(inp[4] == t))


def _window_needs(inp, w):
    """(target, window, bytes) of every window: the target and the reads touching that window"""
    return [(t, k, _store(inp, [t], _touching(inp, w, t, k, k + 1)))
            for t in range(inp[0]) for k in range(_n_windows(inp, w, t))]


def _plan(inp, w, budget):
    return api.plan_read_groups(*inp[:5], budget, t_begin=inp[5], t_end=inp[6], window_length=w)


def _check_split_plan(inp, w, budget):
    n_targets, lengths, has_q, q_id, t_id, _, _ = inp
    first, nbytes, ofirst, order, fwin, ewin, aligned_in = _plan(inp, w, budget)
    n_groups = len(nbytes)
    assert first[-1] == n_targets and len(fwin) == len(ewin) == n_groups and len(aligned_in) == len(q_id)
    seen = np.zeros(len(q_id), np.int64)
    g, next_target = 0, 0
    while g < n_groups:
        assert int(first[g]) == next_target
        if ewin[g] == 0:   # a group of whole targets: fits, and keeps its targets' overlaps in file order
            a, b = int(first[g]), int(first[g + 1])
            assert b > a
            ov = order[ofirst[g]:ofirst[g + 1]].astype(np.int64)
            assert ov.tolist() == np.flatnonzero((t_id >= a) & (t_id < b)).tolist()
            assert nbytes[g] == _store(inp, range(a, b), ov) <= budget
            assert all(_own(inp, t) <= budget for t in range(a, b))
            assert np.all(aligned_in[ov] == g)
            seen[ov] += 1
            if b < n_targets and _own(inp, b) <= budget:   # closed only by a target that would not fit
                assert _store(inp, range(a, b + 1), np.flatnonzero((t_id >= a) & (t_id <= b))) > budget
            g, next_target = g + 1, b
            continue
        # a split target: its own store is over the budget; parts are contiguous, cover its windows once, fit, are
        # maximal, hold exactly the overlaps touching them in file order, and align each overlap in its first part
        t = next_target
        assert _own(inp, t) > budget
        n_w = _n_windows(inp, w, t)
        a = 0
        while a < n_w:
            b = int(ewin[g])
            assert int(fwin[g]) == a and a < b <= n_w
            assert int(first[g]) == t and int(first[g + 1]) == (t if b < n_w else t + 1)
            ov = order[ofirst[g]:ofirst[g + 1]].astype(np.int64)
            assert ov.tolist() == _touching(inp, w, t, a, b).tolist()
            assert nbytes[g] == _store(inp, [t], ov) <= budget
            if b < n_w:
                assert _store(inp, [t], _touching(inp, w, t, a, b + 1)) > budget
            assert np.all(aligned_in[ov[seen[ov] == 0]] == g) and np.all(aligned_in[ov] <= g)
            seen[ov] += 1
            a = b
            g += 1
        next_target = t + 1
    assert next_target == n_targets
    assert np.all(seen >= 1)
    for k in range(len(q_id)):   # aligned exactly once: in the first group that holds it
        holders = [h for h in range(n_groups) if k in order[ofirst[h]:ofirst[h + 1]]]
        assert aligned_in[k] == holders[0]
    return first, nbytes, fwin, ewin


@pytest.mark.parametrize("fragment", [False, True], ids=["contigs", "fragments"])
@pytest.mark.parametrize("seed", range(10))
def test_split_parts_are_contiguous_within_budget_and_maximal(seed, fragment):
    rng = np.random.default_rng(100 + seed)
    inp, w = _random_input(rng, fragment)
    needs = _window_needs(inp, w)
    largest = max(n for _, _, n in needs)
    owns = [_own(inp, t) for t in range(inp[0])]
    whole = api.read_store_bytes(inp[1], inp[2])
    budgets = {largest, (largest + max(owns)) // 2, max(owns), whole, whole * 2}
    budgets |= {o - 1 for o in owns if o - 1 >= largest}   # each target just over
    for budget in sorted(budgets):
        first, nbytes, fwin, ewin = _check_split_plan(inp, w, budget)
        if budget >= max(owns):   # nothing over: exactly the groups of the planner without splitting
            plain = api.plan_read_groups(*inp[:5], budget)
            split = _plan(inp, w, budget)
            for want, got in zip(plain, split[:4]):
                assert want.tolist() == got.tolist()
            assert not np.any(split[5])
    # one byte below the largest single-window need: the first window (in target order) that needs it is named
    t, k, n = next(x for x in needs if x[2] == largest)
    with pytest.raises(api.RaconB200Error, match="window %d of target #%d needs a read store of %d bytes, over the budget "
                       "of %d bytes per device" % (k, t, n, n - 1)):
        _plan(inp, w, largest - 1)


def test_an_overlap_across_parts_is_in_each_and_aligned_in_the_first():
    """One 1 000-base target in ten windows of 100.  Read 1 (40 bases) spans windows 2-6; reads 2-5 (30 bases) sit in
    windows 0, 3, 5 and 9."""
    lengths = np.array([1000, 40, 30, 30, 30, 30], np.uint32)
    inp = (1, lengths, np.zeros(6, np.uint8), np.array([1, 2, 3, 4, 5]), np.zeros(5, np.int64),
           np.array([250, 0, 300, 550, 900]), np.array([650, 90, 390, 600, 1000]))
    target = 1000 + 16
    runs = {target + 40 + 30 + 30: ([(0, 5), (5, 10)], [[0, 1, 2], [0, 3, 4]], [0, 0, 0, 1, 1]),
            target + 40 + 30: ([(0, 3), (3, 5), (5, 9), (9, 10)], [[0, 1], [0, 2], [0, 3], [4]], [0, 0, 1, 2, 3])}
    for budget, (windows, overlaps, aligned) in runs.items():
        first, nbytes, ofirst, order, fwin, ewin, aligned_in = _plan(inp, 100, budget)
        assert first.tolist() == [0] * len(windows) + [1]
        assert list(zip(fwin.tolist(), ewin.tolist())) == windows
        assert [order[ofirst[g]:ofirst[g + 1]].tolist() for g in range(len(windows))] == overlaps
        assert aligned_in.tolist() == aligned
        assert nbytes.tolist() == [_store(inp, [0], np.array(ov)) for ov in overlaps]
    with pytest.raises(api.RaconB200Error, match="window 3 of target #0 needs a read store of 1086 bytes, over the "
                       "budget of 1085 bytes"):
        _plan(inp, 100, 1085)
    # without a window length the planner does not split
    with pytest.raises(api.RaconB200Error, match="target #0 needs a read store of 1176 bytes"):
        api.plan_read_groups(*inp[:5], 1175)


def test_a_split_target_closes_the_open_group_and_the_next_target_opens_one():
    """targets 0 and 2 would fit in one group, target 1 (1 916 bytes) does not fit: [0], the parts of 1, [2]"""
    lengths = np.array([100, 1000, 100, 300, 300, 300], np.uint32)
    inp = (3, lengths, np.zeros(6, np.uint8), np.array([3, 4, 5]), np.array([1, 1, 1]),
           np.array([0, 400, 800]), np.array([300, 700, 1000]))
    first, nbytes, ofirst, order, fwin, ewin, aligned_in = _plan(inp, 100, 1700)
    assert first.tolist() == [0, 1, 1, 2, 3]
    assert list(zip(fwin.tolist(), ewin.tolist())) == [(0, 0), (0, 8), (8, 10), (0, 0)]
    assert nbytes.tolist() == [116, 1000 + 300 + 300 + 16, 1000 + 300 + 16, 116]
    assert [order[ofirst[g]:ofirst[g + 1]].tolist() for g in range(4)] == [[], [0, 1], [2], []]
    assert api.plan_read_groups(*inp[:5], 10 ** 6)[0].tolist() == [0, 3]


# ---- the command line ---------------------------------------------------------------------------------------------------
def test_help_lists_split_targets():
    status, out, _ = run_cli(["-h"])
    assert status == 0 and b"--split-targets" in out


def test_split_targets_gets_as_far_as_the_device():
    status, out, err = run_cli(["--split-targets"] + sample(*CONTIG), env=dict(NO_DEVICE, RP_READ_STORE_BYTES="1000"))
    assert status == 1 and out == b"" and "no CUDA device" in err, err


def test_split_targets_needs_resident_reads(tmp_path):
    with pytest.raises(ValueError, match="resident_reads"):
        api.polish_files(*sample(*CONTIG), str(tmp_path / "o.fasta"), resident_reads=False, split_targets=True)


# ---- a split run over the simulated runtime -----------------------------------------------------------------------------
def test_split_run_over_the_simulated_runtime():
    """tests/test_gpu_split_targets.py's small split case on the C ABI over the simulated runtime: every part budget gives
    the bytes of the one-group run"""
    from racon_b200 import build
    lib = build.build_simapi()
    env = dict(os.environ, RACON_B200_LIB=lib)
    r = subprocess.run([sys.executable, "-m", "pytest", "tests/test_gpu_split_targets.py::test_small_split_case",
                        "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    tail = "\n".join(r.stdout.splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "1 passed" in tail, tail
