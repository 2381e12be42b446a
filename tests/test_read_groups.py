"""The target-group planner of the host layer (racon_b200::plan_read_groups, api.plan_read_groups) without a device: over
seeded random inputs the groups are contiguous, cover every target once, fit the budget and are maximal; a target over the
budget is an error; a read is counted once per group that uses it; every group's overlaps keep their file order.  The
command line refuses a malformed RP_READ_STORE_BYTES before it looks for a device.  The automatic budget runs over the
simulated runtime here (tests/test_gpu_read_groups.py runs everything on the GPU)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from racon_b200 import api
from tests.test_cli import CONTIG, NO_DEVICE, ROOT, run_cli, sample


def _random_input(rng, fragment):
    """n_targets, lengths, has_quality, q_id, t_id.  fragment: the reads are the targets (racon -f), several overlaps per
    read; otherwise reads follow the targets, most with one overlap and some with two (a read across contig ends)."""
    n_targets = int(rng.integers(1, 40))
    n_reads = 0 if fragment else int(rng.integers(0, 300))
    n_seq = n_targets + n_reads
    lengths = rng.integers(0, 5000, n_seq)
    has_q = rng.random(n_seq) < (0.5 if rng.random() < 0.5 else 0.0)
    if fragment:
        n_ov = int(rng.integers(0, 200))
        q_id = rng.integers(0, n_targets, n_ov)
        t_id = rng.integers(0, n_targets, n_ov)
    else:
        q_id = np.repeat(np.arange(n_targets, n_seq), rng.integers(1, 3, n_reads))
        t_id = rng.integers(0, n_targets, len(q_id))
    return n_targets, lengths, has_q, q_id, t_id


def _store(plan_input, first, end, overlaps):
    """bytes of the store of targets [first, end) and the reads of `overlaps`"""
    n_targets, lengths, has_q, q_id, t_id = plan_input
    ids = np.unique(np.concatenate([np.arange(first, end), q_id[overlaps]]).astype(np.int64))
    return api.read_store_bytes(lengths[ids], has_q[ids])


def _check_plan(plan_input, budget):
    n_targets, lengths, has_q, q_id, t_id = plan_input
    first, nbytes, ofirst, order = api.plan_read_groups(*plan_input, budget)
    assert first[0] == 0 and first[-1] == n_targets and np.all(np.diff(first.astype(np.int64)) > 0)
    assert sorted(order.tolist()) == list(range(len(q_id)))
    for g in range(len(nbytes)):
        a, b = int(first[g]), int(first[g + 1])
        ov = order[ofirst[g]:ofirst[g + 1]].astype(np.int64)
        assert np.all(np.diff(ov) > 0), "a group's overlaps leave file order"
        assert np.all((t_id[ov] >= a) & (t_id[ov] < b))
        assert nbytes[g] == _store(plan_input, a, b, ov) <= budget
        if g + 1 < len(nbytes):   # maximal: the next target would not fit
            nxt = np.flatnonzero((t_id >= a) & (t_id < b + 1))
            assert _store(plan_input, a, b + 1, nxt) > budget
    return first, nbytes


@pytest.mark.parametrize("fragment", [False, True], ids=["contigs", "fragments"])
@pytest.mark.parametrize("seed", range(12))
def test_groups_are_contiguous_within_budget_and_maximal(seed, fragment):
    rng = np.random.default_rng(seed)
    inp = _random_input(rng, fragment)
    n_targets = inp[0]
    singles = [_store(inp, t, t + 1, np.flatnonzero(inp[4] == t)) for t in range(n_targets)]
    whole = api.read_store_bytes(inp[1], inp[2])
    for budget in (max(singles), (max(singles) + whole) // 2, whole, whole * 3):
        first, _ = _check_plan(inp, budget)
        if budget >= whole:
            assert len(first) == 2
    with pytest.raises(api.RaconB200Error, match="target #%d needs a read store of %d bytes, over the budget of %d"
                       % (int(np.argmax(singles)), max(singles), max(singles) - 1)):
        api.plan_read_groups(*inp, max(singles) - 1)


def test_contig_reads_are_counted_once_and_shared_reads_once_per_group():
    """Contigs: a read with one overlap is in one group.  Fragments: a read that two groups use is in both stores."""
    lengths = np.array([100, 100, 100, 50, 60], np.uint32)   # three targets, two reads
    has_q = np.zeros(5, np.uint8)
    # read 3 onto targets 0 and 2, read 4 onto target 1
    inp = (3, lengths, has_q, np.array([3, 4, 3]), np.array([0, 1, 2]))
    first, nbytes, _, _ = api.plan_read_groups(*inp, 10 ** 9)
    assert first.tolist() == [0, 3] and nbytes.tolist() == [100 * 3 + 50 + 60 + 16]
    first, nbytes, _, _ = api.plan_read_groups(*inp, 100 + 60 + 16)
    assert first.tolist() == [0, 1, 2, 3] and nbytes.tolist() == [166, 176, 166]
    # -f: the targets are the reads; target 1 overlaps onto targets 0 and 2
    frag = (3, lengths[:3], has_q[:3], np.array([1, 1]), np.array([0, 2]))
    first, nbytes, _, _ = api.plan_read_groups(*frag, 216)
    assert first.tolist() == [0, 2, 3] and nbytes.tolist() == [216, 216]   # target 1 is in both stores
    first, nbytes, _, _ = api.plan_read_groups(*frag, 316)
    assert first.tolist() == [0, 3] and nbytes.tolist() == [316]


def test_qualities_double_the_store():
    lengths = np.array([100, 40], np.uint32)
    first, nbytes, _, _ = api.plan_read_groups(1, lengths, np.array([0, 1]), np.array([1]), np.array([0]), 10 ** 6)
    assert nbytes.tolist() == [2 * (140 + 16)]
    first, nbytes, _, _ = api.plan_read_groups(1, np.array([100, 0]), np.array([0, 1]), np.array([1]), np.array([0]),
                                               10 ** 6)
    assert nbytes.tolist() == [116]   # an empty sequence brings no qualities


def test_no_target_no_group():
    first, nbytes, ofirst, order = api.plan_read_groups(0, np.zeros(0), np.zeros(0), np.zeros(0), np.zeros(0), 0)
    assert first.tolist() == [0] and len(nbytes) == 0


# ---- the command line's RP_READ_STORE_BYTES ----------------------------------------------------------------------------
@pytest.mark.parametrize("value", ["-1", "1e9", "12MB", " 100", "0x10", "99999999999999999999999", "abc"])
def test_malformed_read_store_budget_exits_1_before_any_device(value):
    status, out, err = run_cli(sample(*CONTIG), env=dict(NO_DEVICE, RP_READ_STORE_BYTES=value))
    assert status == 1 and out == b""
    assert "RP_READ_STORE_BYTES must be a decimal byte count" in err and "no CUDA device" not in err, err


@pytest.mark.parametrize("value", ["", "0", "1000000"])
def test_well_formed_read_store_budget_gets_as_far_as_the_device(value):
    status, out, err = run_cli(sample(*CONTIG), env=dict(NO_DEVICE, RP_READ_STORE_BYTES=value))
    assert status == 1 and out == b"" and "no CUDA device" in err, err


def test_help_names_the_read_store_budget():
    status, out, _ = run_cli(["-h"])
    assert status == 0 and b"RP_READ_STORE_BYTES" in out


# ---- the automatic budget over the simulated runtime --------------------------------------------------------------------
def test_automatic_budget_over_the_simulated_runtime():
    """tests/test_gpu_read_groups.py's automatic-budget test and store-size test on the C ABI over the simulated runtime,
    with 48 MB of free device memory: a 24 MB budget, under which the shrunk multi-contig case runs in several groups."""
    from racon_b200 import build
    from tests import test_gpu_read_groups as groups
    lib = build.build_simapi()
    tests = ["tests/test_gpu_read_groups.py::test_automatic_budget_gives_the_one_group_file",
             "tests/test_gpu_read_groups.py::test_read_store_bytes_follow_the_documented_rule"]
    env = dict(os.environ, RACON_B200_LIB=lib, RP_SIM_FREE_MB="48")
    r = subprocess.run([sys.executable, "-m", "pytest"] + tests + ["-m", "gpu", "-x", "-q", "-p", "no:cacheprovider"],
                       cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    tail = "\n".join(r.stdout.splitlines()[-15:])
    assert r.returncode == 0, tail
    assert "2 passed" in tail, tail
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        paths = groups.write_small_multi_contig(d)
        inp = api.InputFiles(*paths)
        try:
            plan = (inp.n_targets, np.diff(inp.seq_off.astype(np.int64)), inp.seq_has_qual, inp.overlaps[:, 0],
                    inp.overlaps[:, 1])
            assert len(api.plan_read_groups(*plan, (48 << 20) // 2)[1]) >= 2
        finally:
            inp.close()
