"""Split targets on the device (racon_b200::Polisher::polish_groups with split_targets, racon_b200 --split-targets): a
target whose reads do not fit the read store budget is polished in parts of consecutive windows, and the output is racon's
one-pass output, byte for byte.  The sample-file cases of tests/golden/cli_cases.json run under the largest single-window
need (the lambda contig in many parts) and under the smallest budget that gives two parts; where every target fits, the
option changes neither the groups nor the bytes; a generated long contig between two short ones (write_long_contig;
racon's own command line answered it in tests/golden/split_targets_cases.json, made by
tests/golden/make_split_targets_cases.py) runs in one, two and the most parts, on
more lanes and on two lanes of one GPU; a refused overlap across a part boundary is reported once, under its whole-run
index.  The planner itself is tested without a device in tests/test_split_targets.py."""
import hashlib
import json
import os

import numpy as np
import pytest

from racon_b200 import api
from tests.test_cli import ROOT, run_cli, sample
from tests.test_gpu_read_groups import (BASES, FIXTURE, _budgets, _check, _golden, _mutate, _plan_input,
                                        _single_target_need)

pytestmark = pytest.mark.gpu


def _split_golden(case):
    """racon's answer for a generated case (read when a test needs it: the generator below makes the file)"""
    with open(os.path.join(ROOT, "tests", "golden", "split_targets_cases.json")) as f:
        return json.load(f)[case]


# ---- the plan of an input ---------------------------------------------------------------------------------------------
def _window_length(opts):
    return int(opts[opts.index("-w") + 1]) if "-w" in opts else 500


def _split_input(paths, opts):
    """(n_targets, lengths, has_quality, q_id, t_id, t_begin, t_end) of the input after racon's filter"""
    frag = "-f" in opts
    e = float(opts[opts.index("-e") + 1]) if "-e" in opts else 0.3
    inp = api.InputFiles(*paths, fragment_correction=frag, error_threshold=e)
    try:
        return (inp.n_targets, np.diff(inp.seq_off.astype(np.int64)), inp.seq_has_qual.copy(),
                inp.overlaps[:, 0].copy(), inp.overlaps[:, 1].copy(), inp.overlaps[:, 6].copy(),
                inp.overlaps[:, 7].copy())
    finally:
        inp.close()


def _split_plan(inp, w, budget):
    return api.plan_read_groups(*inp[:5], budget, t_begin=inp[5], t_end=inp[6], window_length=w)


def _largest_window_need(inp, w):
    """the largest store one window needs: its target and the reads whose span touches it"""
    n_targets, lengths, has_q, q_id, t_id, t_begin, t_end = inp
    need = 0
    for t in range(n_targets):
        on = t_id == t
        for k in range((int(lengths[t]) + w - 1) // w):
            ids = np.unique(np.append(q_id[on & (t_begin // w <= k) & ((t_end - 1) // w >= k)], t))
            need = max(need, api.read_store_bytes(lengths[ids], has_q[ids]))
    return need


def _parts(inp, w, budget):
    return int(np.count_nonzero(_split_plan(inp, w, budget)[5]))


def _two_part_budget(inp, w):
    """the smallest budget under which the plan has at most two parts (it has exactly two there)"""
    lo, hi = _largest_window_need(inp, w), api.read_store_bytes(inp[1], inp[2])
    while lo < hi:
        mid = (lo + hi) // 2
        if _parts(inp, w, mid) <= 2:
            hi = mid
        else:
            lo = mid + 1
    assert _parts(inp, w, lo) == 2
    return lo


def _kwargs(opts):
    """api.polish_files' keywords for racon's options"""
    kw, i = {}, 0
    names = {"-w": ("window_length", int), "-q": ("quality_threshold", float), "-e": ("error_threshold", float),
             "-m": ("match", int), "-x": ("mismatch", int), "-g": ("gap", int)}
    while i < len(opts):
        o = opts[i]
        if o in names:
            kw[names[o][0]] = names[o][1](opts[i + 1])
            i += 2
            continue
        kw.update({"-u": {"drop_unpolished": False}, "-f": {"fragment_correction": True},
                   "--no-trimming": {"trim": False}}[o])
        i += 1
    return kw


def _polish(paths, opts, out, **kw):
    n, fo, fw = api.polish_files(*paths, str(out), **_kwargs(opts), **kw)
    return (n, fo, fw), open(out, "rb").read(), api.last_grouped_run()


# ---- the sample cases ----------------------------------------------------------------------------------------------------
CONTIG_CASES = sorted(k for k in FIXTURE if "generator" not in FIXTURE[k] and "-f" not in FIXTURE[k]["options"])
FRAGMENT_CASES = sorted(k for k in FIXTURE if "generator" not in FIXTURE[k] and "-f" in FIXTURE[k]["options"])


@pytest.mark.parametrize("case", CONTIG_CASES)
def test_sample_cases_in_parts_give_racons_output(case, tmp_path):
    """--split-targets under the largest single-window need and the smallest two-part budget: racon's bytes; each part's
    store is the size the planner predicts"""
    want = FIXTURE[case]
    paths = sample(*want["files"])
    opts = want["options"]
    inp = _split_input(paths, opts)
    w = _window_length(opts)
    for budget in (_largest_window_need(inp, w), _two_part_budget(inp, w)):
        plan = _split_plan(inp, w, budget)
        assert np.count_nonzero(plan[5]) >= 2
        _check(want, *run_cli(["--split-targets"] + opts + paths, env={"RP_READ_STORE_BYTES": str(budget)}))
        (n, fo, fw), data, run = _polish(paths, opts, tmp_path / "o.fasta", read_store_bytes=budget,
                                         split_targets=True)
        assert (n, fo, fw) == (want["count"], 0, 0)
        assert hashlib.md5(data).hexdigest() == want["md5"]
        assert run["group_bytes"] == [int(b) for b in plan[1]]


@pytest.mark.parametrize("case", FRAGMENT_CASES)
def test_fragment_cases_get_the_same_groups_with_the_option(case, tmp_path):
    """-f: every target fits the smallest budget of tests/test_gpu_read_groups.py, so the option changes nothing"""
    want = FIXTURE[case]
    paths = sample(*want["files"])
    opts = want["options"]
    budget = _single_target_need(_plan_input(paths, opts))
    runs = [_polish(paths, opts, tmp_path / "o.fasta", read_store_bytes=budget, split_targets=s) for s in (False, True)]
    assert runs[0][1] == runs[1][1] and hashlib.md5(runs[1][1]).hexdigest() == want["md5"]
    assert runs[0][2] == runs[1][2] and len(runs[1][2]["group_bytes"]) >= 3


def test_multi_contig_gets_the_same_groups_with_the_option(tmp_path):
    from tests.test_gpu_read_groups import write_multi_contig
    paths = write_multi_contig(str(tmp_path))
    want = _golden("multi_contig")
    for budget in _budgets(_plan_input(paths, want["options"])):
        runs = [_polish(paths, want["options"], tmp_path / "o.fasta", read_store_bytes=budget, split_targets=s)
                for s in (False, True)]
        assert runs[0][1] == runs[1][1] and hashlib.md5(runs[1][1]).hexdigest() == want["md5"]
        assert runs[0][2] == runs[1][2]


# ---- the generated long contig ---------------------------------------------------------------------------------------------
def write_long_contig(d, long_len=60000, short_len=3000, coverage=20, read_len=4000, seed=23):
    """A genome of three consecutive contigs, a long one between two short ones (drafts: the genome with 3 %
    substitutions); FASTQ reads with 10 % error on both strands sampled within the contigs, one PAF line each.  Writes
    reads.fastq, overlaps.paf and contigs.fasta into d; returns their paths."""
    rng = np.random.default_rng(seed)
    lengths = [short_len, long_len, short_len]
    start = np.concatenate([[0], np.cumsum(lengths)])
    genome = rng.integers(0, 4, int(start[-1])).astype(np.uint8)
    with open(os.path.join(d, "contigs.fasta"), "wb") as f:
        for c in range(3):
            truth = genome[start[c]:start[c + 1]]
            draft = np.where(rng.random(len(truth)) < 0.03, (truth + rng.integers(1, 4, len(truth))) % 4, truth)
            f.write(b">contig%d\n" % c + BASES[draft].tobytes() + b"\n")
    reads, paf = [], []
    n_reads = int(coverage * start[-1] / read_len)
    for r in range(n_reads):
        c = int(rng.choice(3, p=np.array(lengths) / start[-1]))
        length = min(int(rng.integers(read_len // 2, read_len * 3 // 2)), lengths[c])
        t0 = int(rng.integers(0, lengths[c] - length + 1))
        codes, _ = _mutate(rng, genome[start[c] + t0:start[c] + t0 + length], 0.04, 0.03, 0.03)
        L = len(codes)
        rev = bool(rng.random() < 0.5)
        seq = BASES[3 - codes[::-1]] if rev else BASES[codes]
        qual = (rng.integers(8, 40, L) + 33).astype(np.uint8)
        reads.append(b"@read%d\n" % r + seq.tobytes() + b"\n+\n" + qual.tobytes() + b"\n")
        paf.append(b"read%d\t%d\t0\t%d\t%s\tcontig%d\t%d\t%d\t%d\t%d\t%d\t60\n" % (
            r, L, L, b"-" if rev else b"+", c, lengths[c], t0, t0 + length, min(L, length), max(L, length)))
    with open(os.path.join(d, "reads.fastq"), "wb") as f:
        f.write(b"".join(reads))
    with open(os.path.join(d, "overlaps.paf"), "wb") as f:
        f.write(b"".join(paf))
    return [os.path.join(d, n) for n in ("reads.fastq", "overlaps.paf", "contigs.fasta")]


@pytest.fixture(scope="module")
def long_contig(tmp_path_factory):
    want = _split_golden("long_contig")
    paths = write_long_contig(str(tmp_path_factory.mktemp("long_contig")))
    assert [os.path.basename(p) for p in paths] == want["files"]
    inp = _split_input(paths, want["options"])
    most = _largest_window_need(inp, 500)
    budgets = {"one": int(max(_single_target_need(inp[:5]), 1)), "two": _two_part_budget(inp, 500), "most": most}
    assert _parts(inp, 500, budgets["one"]) == 0 and _parts(inp, 500, budgets["most"]) > 10
    # the edges the case is for: reads over three or more parts
    _, _, ofirst, order, _, ewin, _ = _split_plan(inp, 500, most)
    parts = np.flatnonzero(ewin)   # the long contig's, one after the other
    assert np.bincount(order[ofirst[parts[0]]:ofirst[parts[-1] + 1]].astype(np.int64)).max() >= 3
    return paths, inp, budgets


def test_long_contig_in_one_two_and_the_most_parts(long_contig, tmp_path):
    paths, inp, budgets = long_contig
    want = _split_golden("long_contig")
    aligned = {}
    for name, budget in budgets.items():
        _check(want, *run_cli(["--split-targets"] + paths, env={"RP_READ_STORE_BYTES": str(budget)}))
        (n, fo, fw), data, run = _polish(paths, [], tmp_path / "o.fasta", read_store_bytes=budget, split_targets=True)
        assert (n, fo, fw) == (want["count"], 0, 0) and hashlib.md5(data).hexdigest() == want["md5"]
        plan = _split_plan(inp, 500, budget)
        assert run["group_bytes"] == [int(b) for b in plan[1]]
        assert len(run["group_windows"]) == len(plan[1]) and run["group_windows"][0][0] == 0
        assert all(run["group_windows"][g][1] == run["group_windows"][g + 1][0] for g in range(len(plan[1]) - 1))
        aligned[name] = sum(run["group_aligned"])
    one_group = _polish(paths, [], tmp_path / "o.fasta", read_store_bytes=api.read_store_bytes(inp[1], inp[2]))[2]
    assert len(one_group["group_aligned"]) == 1
    assert set(aligned.values()) == {one_group["group_aligned"][0]} and one_group["group_aligned"][0] == len(inp[3])


def test_long_contig_on_two_lanes(long_contig, tmp_path):
    paths, inp, budgets = long_contig
    want = _split_golden("long_contig")
    _check(want, *run_cli(["-c", "2", "--split-targets"] + paths, env={"RP_READ_STORE_BYTES": str(budgets["most"])}))
    for budget in (budgets["two"], budgets["most"]):
        (n, fo, fw), data, run = _polish(paths, [], tmp_path / "o.fasta", device=[0, 0], read_store_bytes=budget,
                                         split_targets=True)
        assert (n, fo, fw) == (want["count"], 0, 0) and hashlib.md5(data).hexdigest() == want["md5"]
        assert run["group_bytes"] == [int(b) for b in _split_plan(inp, 500, budget)[1]]


def test_long_contig_over_the_budget(long_contig, tmp_path):
    """without the option a splitting budget is still the old error; with it, one byte below the largest window need is
    the new one — both before any output"""
    paths, inp, budgets = long_contig
    status, out, err = run_cli(paths, env={"RP_READ_STORE_BYTES": str(budgets["two"])})
    own = _single_target_need(inp[:5])
    assert status == 1 and out == b""
    assert "target contig1 needs a read store of %d bytes, over the budget of %d bytes per device" % (
        own, budgets["two"]) in err, err
    assert "--split-targets" in err
    most = budgets["most"]
    status, out, err = run_cli(["--split-targets"] + paths, env={"RP_READ_STORE_BYTES": str(most - 1)})
    assert status == 1 and out == b""
    assert "of target contig1 needs a read store of %d bytes, over the budget of %d bytes per device" % (
        most, most - 1) in err, err
    with pytest.raises(api.RaconB200Error, match="window [0-9]+ of target contig1 needs"):
        api.polish_files(*paths, str(tmp_path / "o.fasta"), read_store_bytes=most - 1, split_targets=True)
    assert not os.path.exists(tmp_path / "o.fasta")


# ---- a refused overlap across a part boundary -------------------------------------------------------------------------------
def _write_refused_long_read(d):
    """One 3 kb contig; three exact copies of each of its thirds as reads, and a read over [500, 2500) with 17 distinct
    letters — one more than the aligner takes — last in the files."""
    rng = np.random.default_rng(29)
    contig = bytes(b"ACGT"[i] for i in rng.integers(4, size=3000))
    odd = bytearray(contig[500:2500])
    for k, c in enumerate(b"BDEFHIJKLMNOP"):
        odd[50 + 140 * k] = c
    reads = [(b"r%d_%d" % (p, i), 1000 * p, contig[1000 * p:1000 * (p + 1)]) for p in range(3) for i in range(3)]
    reads.append((b"odd", 500, bytes(odd)))
    with open(os.path.join(d, "t.fasta"), "wb") as f:
        f.write(b">contig0\n%s\n" % contig)
    with open(os.path.join(d, "r.fasta"), "wb") as f:
        f.write(b"".join(b">" + n + b"\n" + s + b"\n" for n, _, s in reads))
    with open(os.path.join(d, "o.paf"), "wb") as f:
        f.write(b"".join(b"%s\t%d\t0\t%d\t+\tcontig0\t3000\t%d\t%d\t%d\t%d\t60\n" % (n, len(s), len(s), t0, t0 + len(s),
                                                                                     len(s), len(s))
                         for n, t0, s in reads))
    return [os.path.join(d, n) for n in ("r.fasta", "o.paf", "t.fasta")]


def test_refused_overlap_across_parts_is_reported_once(tmp_path):
    paths = _write_refused_long_read(str(tmp_path))
    inp = _split_input(paths, [])
    odd = len(inp[3]) - 1
    most = _largest_window_need(inp, 500)
    plan = _split_plan(inp, 500, most)
    holders = [g for g in range(len(plan[1])) if odd in plan[3][plan[2][g]:plan[2][g + 1]]]
    assert len(holders) >= 2 and plan[6][odd] == holders[0]
    runs = {}
    for name, budget, split in (("one", 0, False), ("parts", most, True)):
        out = tmp_path / (name + ".fasta")
        n, fo, fw = api.polish_files(*paths, str(out), read_store_bytes=budget, split_targets=split)
        runs[name] = (open(out, "rb").read(), api.last_grouped_run(), (n, fo, fw))
    assert len(runs["parts"][1]["group_bytes"]) == len(plan[1])
    assert runs["one"][0] == runs["parts"][0]
    assert runs["one"][2] == runs["parts"][2] and runs["parts"][2][1] == 1
    assert runs["one"][1]["failed_overlaps"] == runs["parts"][1]["failed_overlaps"] == [odd]
    assert runs["one"][1]["failed_windows"] == runs["parts"][1]["failed_windows"]
    status, out, err = run_cli(["--split-targets"] + paths, env={"RP_READ_STORE_BYTES": str(most)})
    assert status == 2 and "refused 1 overlap(s)" in err, err
    assert out == runs["one"][0]


# ---- a small case (also run over the simulated runtime by tests/test_split_targets.py) ------------------------------------
def write_small_split_case(d, seed=31, length=800, n_reads=16):
    """One 800-base contig (windows of 100) with 3 % substitutions, and 16 FASTQ reads of 100 to 250 bases from both
    strands with 5 % error: small enough for the simulated runtime."""
    rng = np.random.default_rng(seed)
    truth = rng.integers(0, 4, length).astype(np.uint8)
    draft = np.where(rng.random(length) < 0.03, (truth + rng.integers(1, 4, length)) % 4, truth)
    with open(os.path.join(d, "t.fasta"), "wb") as f:
        f.write(b">contig0\n" + BASES[draft].tobytes() + b"\n")
    reads, paf = [], []
    for r in range(n_reads):
        span = int(rng.integers(100, 251))
        t0 = int(rng.integers(0, length - span + 1))
        codes, _ = _mutate(rng, truth[t0:t0 + span], 0.02, 0.015, 0.015)
        L = len(codes)
        rev = r % 2 == 1
        seq = BASES[3 - codes[::-1]] if rev else BASES[codes]
        reads.append(b"@r%d\n" % r + seq.tobytes() + b"\n+\n" + (rng.integers(15, 40, L) + 33).astype(np.uint8).tobytes()
                     + b"\n")
        paf.append(b"r%d\t%d\t0\t%d\t%s\tcontig0\t%d\t%d\t%d\t%d\t%d\t60\n" % (
            r, L, L, b"-" if rev else b"+", length, t0, t0 + span, min(L, span), max(L, span)))
    with open(os.path.join(d, "r.fastq"), "wb") as f:
        f.write(b"".join(reads))
    with open(os.path.join(d, "o.paf"), "wb") as f:
        f.write(b"".join(paf))
    return [os.path.join(d, n) for n in ("r.fastq", "o.paf", "t.fasta")]


def test_small_split_case(tmp_path):
    """windows of 100: the parts under the largest window need and the two-part budget give the one-group file, the
    same refusals and, summed, the one-group run's aligned overlaps"""
    paths = write_small_split_case(str(tmp_path))
    inp = _split_input(paths, [])
    budgets = [_largest_window_need(inp, 100), _two_part_budget(inp, 100)]
    assert _parts(inp, 100, budgets[0]) >= 3
    runs = []
    for budget, split in [(api.read_store_bytes(inp[1], inp[2]), False)] + [(b, True) for b in budgets]:
        runs.append(_polish(paths, ["-w", "100"], tmp_path / "o.fasta", read_store_bytes=budget, split_targets=split))
    for result, data, run in runs[1:]:
        assert data == runs[0][1] and result == runs[0][0]
        assert run["failed_overlaps"] == runs[0][2]["failed_overlaps"]
        assert run["failed_windows"] == runs[0][2]["failed_windows"]
        assert sum(run["group_aligned"]) == runs[0][2]["group_aligned"][0] == len(inp[3])
    assert runs[0][0][0] == 1 and len(runs[0][1]) > 500
