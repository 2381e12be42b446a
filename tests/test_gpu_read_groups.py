"""Polishing in target groups (racon_b200::Polisher::polish_groups) on the device: under any read store budget the output
is the one-pass output, byte for byte.  The sample-file cases of tests/golden/cli_cases.json run under the smallest budget
that still holds every target; a generated multi-contig case (write_multi_contig; racon's own command line answered it in
tests/golden/read_groups_cases.json, made by tests/golden/make_read_groups_cases.py) runs in one group, two groups and one target per group, on more lanes and through api.polish_files; refused overlaps keep
their whole-run indices; the automatic budget (half of the smallest free device memory) gives the same file.  The planner
itself is tested without a device in tests/test_read_groups.py."""
import hashlib
import json
import os

import numpy as np
import pytest

from racon_b200 import api
from tests.test_cli import ROOT, run_cli, sample

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "cli_cases.json")) as _f:
    FIXTURE = json.load(_f)


def _golden(case):
    """racon's answer for a generated case (read when a test needs it: the generator below makes the file)"""
    with open(os.path.join(ROOT, "tests", "golden", "read_groups_cases.json")) as f:
        return json.load(f)[case]

BASES = np.frombuffer(b"ACGT", np.uint8)


# ---- the generated multi-contig case ----------------------------------------------------------------------------------
def _mutate(rng, seq, p_sub, p_ins, p_del):
    """seq (codes 0..3) through substitutions, insertions and deletions -> (codes, position in the output of every input
    base, plus the end)"""
    r = rng.random(len(seq))
    dele = r < p_del
    sub = (r >= p_del) & (r < p_del + p_sub)
    ins = (r >= p_del + p_sub) & (r < p_del + p_sub + p_ins)
    emit = np.where(dele, 0, np.where(ins, 2, 1))
    pos = np.cumsum(emit) - emit
    out = np.empty(int(emit.sum()), np.uint8)
    base = np.where(sub, (seq + rng.integers(1, 4, len(seq))) % 4, seq).astype(np.uint8)
    out[pos[ins]] = rng.integers(0, 4, int(ins.sum()))
    keep = ~dele
    out[pos[keep] + ins[keep]] = base[keep]
    return out, np.append(pos, len(out))


def multi_contig_layout(n_contigs=24, contig_len=3000):
    """Which contigs get no reads: every fourth, never two side by side.  They are 40 times longer than the others, so
    that a group of one of them and a neighbour costs more than any single target (one target per group is then a budget
    the planner can be given)."""
    empty = [c % 4 == 2 for c in range(n_contigs)]
    lengths = [contig_len * (40 if e else 1) for e in empty]
    return empty, lengths


def write_multi_contig(d, n_contigs=24, contig_len=3000, coverage=30, read_len=1500, seed=5, min_part=150):
    """A genome cut into n_contigs consecutive contigs (drafts: the genome with 3 % substitutions), some without any read
    (multi_contig_layout); FASTQ reads with 10 % error sampled on both strands from the rest, some across the boundary of
    two neighbouring contigs: such a read has one PAF line per contig (each part at least min_part bases) and racon's
    one-overlap-per-read filter keeps the longer, whichever group it falls in.  Writes reads.fastq, overlaps.paf and
    contigs.fasta into d; returns their paths."""
    rng = np.random.default_rng(seed)
    empty, lengths = multi_contig_layout(n_contigs, contig_len)
    start = np.concatenate([[0], np.cumsum(lengths)])
    genome = rng.integers(0, 4, int(start[-1])).astype(np.uint8)
    with open(os.path.join(d, "contigs.fasta"), "wb") as f:
        for c in range(n_contigs):
            truth = genome[start[c]:start[c + 1]]
            draft = np.where(rng.random(len(truth)) < 0.03, (truth + rng.integers(1, 4, len(truth))) % 4, truth)
            f.write(b">contig%d\n" % c + BASES[draft].tobytes() + b"\n")
    reads, paf = [], []
    spanning = {"first": 0, "second": 0}   # reads over a boundary whose longer part is on the first / second contig
    n_reads = int(coverage * contig_len * sum(1 for e in empty if not e) / read_len)
    while len(reads) < n_reads:
        c = int(rng.integers(n_contigs))
        if empty[c]:
            continue
        length = int(rng.integers(read_len // 2, read_len * 3 // 2))
        s = int(rng.integers(start[c] - length // 2, start[c + 1] - length // 2))
        s, e = max(s, 0), min(s + length, int(start[-1]))
        touched = [k for k in range(n_contigs) if start[k] < e and s < start[k + 1]]
        if any(empty[k] for k in touched) or e - s < min_part:
            continue
        codes, pos = _mutate(rng, genome[s:e], 0.04, 0.03, 0.03)
        L = len(codes)
        rev = bool(rng.random() < 0.5)
        name = b"read%d" % len(reads)
        seq = BASES[3 - codes[::-1]] if rev else BASES[codes]
        qual = (rng.integers(8, 40, L) + 33).astype(np.uint8)
        reads.append(b"@" + name + b"\n" + seq.tobytes() + b"\n+\n" + qual.tobytes() + b"\n")
        parts = []
        for k in touched:
            g0, g1 = max(s, int(start[k])), min(e, int(start[k + 1]))
            if g1 - g0 < min_part:
                continue
            p0, p1 = int(pos[g0 - s]), int(pos[g1 - s])
            q0, q1 = (L - p1, L - p0) if rev else (p0, p1)
            t0, t1 = g0 - int(start[k]), g1 - int(start[k])
            parts.append(g1 - g0)
            paf.append(b"%s\t%d\t%d\t%d\t%s\tcontig%d\t%d\t%d\t%d\t%d\t%d\t60\n" % (
                name, L, q0, q1, b"-" if rev else b"+", k, lengths[k], t0, t1, min(q1 - q0, t1 - t0),
                max(q1 - q0, t1 - t0)))
        if len(parts) == 2:
            spanning["first" if parts[0] > parts[1] else "second"] += 1
    # the edges the case is for
    assert sum(empty) >= 2 and spanning["first"] > 0 and spanning["second"] > 0, spanning
    with open(os.path.join(d, "reads.fastq"), "wb") as f:
        f.write(b"".join(reads))
    with open(os.path.join(d, "overlaps.paf"), "wb") as f:
        f.write(b"".join(paf))
    return [os.path.join(d, n) for n in ("reads.fastq", "overlaps.paf", "contigs.fasta")]


# ---- helpers ----------------------------------------------------------------------------------------------------------
def _options(opts):
    frag = "-f" in opts
    e = float(opts[opts.index("-e") + 1]) if "-e" in opts else 0.3
    return frag, e


def _plan_input(paths, opts):
    """(n_targets, lengths, has_quality, q_id, t_id) of the input after racon's filter"""
    frag, e = _options(opts)
    inp = api.InputFiles(*paths, fragment_correction=frag, error_threshold=e)
    try:
        return (inp.n_targets, np.diff(inp.seq_off.astype(np.int64)), inp.seq_has_qual.copy(),
                inp.overlaps[:, 0].copy(), inp.overlaps[:, 1].copy())
    finally:
        inp.close()


def _single_target_need(plan):
    """the largest store one target needs on its own"""
    n_targets, lengths, has_q, q_id, t_id = plan
    need = 0
    for t in range(n_targets):
        ids = np.unique(np.append(q_id[t_id == t], t))
        need = max(need, api.read_store_bytes(lengths[ids], has_q[ids]))
    return need


def _groups(plan, budget):
    return len(api.plan_read_groups(*plan, budget)[1])


def _budget_for(plan, n_groups):
    """the smallest budget under which the planner makes at most n_groups groups"""
    lo, hi = _single_target_need(plan), api.read_store_bytes(plan[1], plan[2])
    while lo < hi:
        mid = (lo + hi) // 2
        if _groups(plan, mid) <= n_groups:
            hi = mid
        else:
            lo = mid + 1
    return lo


def _check(want, status, out, err):
    assert status == 0, err
    lines = out.split(b"\n")
    names, seqs = lines[0:-1:2], lines[1:-1:2]
    assert len(seqs) == want["count"]
    assert sum(len(s) for s in seqs) == want["bases"]
    assert [n[1:].decode() for n in names] == want["names"]
    assert hashlib.md5(out).hexdigest() == want["md5"]


# ---- the sample cases under the smallest budget -------------------------------------------------------------------------
@pytest.mark.parametrize("case", sorted(k for k in FIXTURE if "generator" not in FIXTURE[k]))
def test_sample_cases_under_the_smallest_budget_give_racons_output(case):
    """RP_READ_STORE_BYTES = the largest store a single target needs: as many groups as that allows, racon's bytes"""
    paths = sample(*FIXTURE[case]["files"])
    plan = _plan_input(paths, FIXTURE[case]["options"])
    budget = _single_target_need(plan)
    if "-f" in FIXTURE[case]["options"]:
        assert plan[0] == 236 and _groups(plan, budget) >= 3
    _check(FIXTURE[case], *run_cli(FIXTURE[case]["options"] + paths, env={"RP_READ_STORE_BYTES": str(budget)}))


# ---- the generated multi-contig case ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def multi_contig(tmp_path_factory):
    paths = write_multi_contig(str(tmp_path_factory.mktemp("multi_contig")))
    assert [os.path.basename(p) for p in paths] == _golden("multi_contig")["files"]
    return paths, _plan_input(paths, _golden("multi_contig")["options"])


def _budgets(plan):
    """budget -> groups: one group, two groups, one target per group"""
    whole = api.read_store_bytes(plan[1], plan[2])
    single = _single_target_need(plan)
    out = {whole: 1, _budget_for(plan, 2): 2, single: plan[0]}
    for budget, n in out.items():
        assert _groups(plan, budget) == n
    return out


def test_multi_contig_in_one_two_and_one_target_per_group(multi_contig):
    paths, plan = multi_contig
    for budget in _budgets(plan):
        _check(_golden("multi_contig"), *run_cli(_golden("multi_contig")["options"] + paths,
                                        env={"RP_READ_STORE_BYTES": str(budget)}))


def test_multi_contig_on_two_lanes_per_gpu(multi_contig):
    paths, plan = multi_contig
    budget = _budget_for(plan, 2)
    _check(_golden("multi_contig"), *run_cli(["-c", "2"] + _golden("multi_contig")["options"] + paths,
                                    env={"RP_READ_STORE_BYTES": str(budget)}))


def test_polish_files_on_two_lanes_uploads_the_planned_stores(multi_contig, tmp_path):
    """api.polish_files(device=[0, 0]) in each grouping: racon's bytes, and every group's store is as large as planned"""
    paths, plan = multi_contig
    want = _golden("multi_contig")
    for budget, n_groups in _budgets(plan).items():
        out = str(tmp_path / "polished.fasta")
        n, fo, fw = api.polish_files(*paths, out, device=[0, 0], read_store_bytes=budget)
        assert (n, fo, fw) == (want["count"], 0, 0)
        assert hashlib.md5(open(out, "rb").read()).hexdigest() == want["md5"]
        run = api.last_grouped_run()
        assert run["group_bytes"] == [int(b) for b in api.plan_read_groups(*plan, budget)[1]]
        assert len(run["group_bytes"]) == n_groups


def test_a_target_over_the_budget_is_an_error(multi_contig, tmp_path):
    paths, plan = multi_contig
    budget = _single_target_need(plan) - 1
    status, out, err = run_cli(_golden("multi_contig")["options"] + paths, env={"RP_READ_STORE_BYTES": str(budget)})
    assert status == 1 and out == b""
    assert "needs a read store of %d bytes, over the budget of %d bytes per device" % (budget + 1, budget) in err, err
    with pytest.raises(api.RaconB200Error, match="over the budget"):
        api.polish_files(*paths, str(tmp_path / "o.fasta"), read_store_bytes=budget)
    assert not os.path.exists(tmp_path / "o.fasta")


# ---- refused overlaps keep their whole-run indices ---------------------------------------------------------------------
def _write_refused_three_contigs(d):
    """Three 1.2 kb contigs, three exact copies of each as reads, and on the middle contig a fourth read with 17 distinct
    letters — one more than the aligner takes (the read of tests/test_gpu_cli.py)."""
    rng = np.random.default_rng(17)
    contigs = [bytes(b"ACGT"[i] for i in rng.integers(4, size=1200)) for _ in range(3)]
    odd = bytearray(contigs[1])
    for k, c in enumerate(b"BDEFHIJKLMNOP"):
        odd[50 + 70 * k] = c
    with open(os.path.join(d, "t.fasta"), "wb") as f:
        f.write(b"".join(b">contig%d\n%s\n" % (c, s) for c, s in enumerate(contigs)))
    reads = [(b"r%d_%d" % (c, i), c, s) for c, s in enumerate(contigs) for i in range(3)] + [(b"odd", 1, bytes(odd))]
    with open(os.path.join(d, "r.fasta"), "wb") as f:
        f.write(b"".join(b">" + n + b"\n" + s + b"\n" for n, _, s in reads))
    with open(os.path.join(d, "o.paf"), "wb") as f:
        f.write(b"".join(b"%s\t1200\t0\t1200\t+\tcontig%d\t1200\t0\t1200\t1200\t1200\t60\n" % (n, c) for n, c, _ in reads))
    return [os.path.join(d, n) for n in ("r.fasta", "o.paf", "t.fasta")]


def test_refused_overlap_keeps_its_index_under_groups(tmp_path):
    paths = _write_refused_three_contigs(str(tmp_path))
    plan = _plan_input(paths, [])
    single = _single_target_need(plan)
    assert _groups(plan, single) == 3
    runs = {}
    for budget in (0, single):
        out = str(tmp_path / ("o%d.fasta" % budget))
        n, fo, fw = api.polish_files(*paths, out, read_store_bytes=budget)
        runs[budget] = (open(out, "rb").read(), api.last_grouped_run())
        assert len(runs[budget][1]["group_bytes"]) == (1 if budget == 0 else 3)
    assert runs[0][0] == runs[single][0]
    assert runs[0][1]["failed_overlaps"] == runs[single][1]["failed_overlaps"] == [9]   # the odd read's, in file order
    assert runs[0][1]["failed_windows"] == runs[single][1]["failed_windows"]
    status, out, err = run_cli(paths, env={"RP_READ_STORE_BYTES": str(single)})
    assert status == 2 and "refused 1 overlap(s)" in err, err
    assert out == runs[0][0]


# ---- the read store's size rule and the automatic budget --------------------------------------------------------------
def test_read_store_bytes_follow_the_documented_rule():
    rng = np.random.default_rng(3)
    for with_quality in (False, True):
        n = 40
        seqs = [bytes(BASES[rng.integers(0, 4, int(rng.integers(0, 3000)))]) for _ in range(n)]
        absent = rng.random(n) < 0.3
        seqs = [b"" if a else s for a, s in zip(absent, seqs)]
        quals = [b"5" * len(s) for s in seqs] if with_quality else None
        store = api.ReadStore(seqs, quals)
        try:
            assert store.device_bytes() == api.read_store_bytes([len(s) for s in seqs], [with_quality] * n)
        finally:
            store.close()


def write_small_multi_contig(d):
    """The multi-contig case shrunk to 300-base contigs and 150-base reads, and two 13 Mb contigs without reads at the end:
    under a budget of a few MB their store alone fills a group."""
    paths = write_multi_contig(d, n_contigs=12, contig_len=300, read_len=150, min_part=30)
    rng = np.random.default_rng(8)
    with open(paths[2], "ab") as f:
        for k in range(2):
            f.write(b">long%d\n" % k + BASES[rng.integers(0, 4, 13_000_000)].tobytes() + b"\n")
    return paths


def test_automatic_budget_gives_the_one_group_file(tmp_path):
    """read_store_bytes=0: half of the free device memory (rp_device_memory) before anything is allocated — the groups the
    planner makes under it, and the file of a one-group run"""
    paths = write_small_multi_contig(str(tmp_path))
    plan = _plan_input(paths, [])
    automatic = api.device_memory(0)[0] // 2
    files = {}
    for name, budget in (("one", api.read_store_bytes(plan[1], plan[2])), ("auto", 0)):
        out = str(tmp_path / (name + ".fasta"))
        n, fo, fw = api.polish_files(*paths, out, read_store_bytes=budget)
        assert n > 0 and (fo, fw) == (0, 0)
        files[name] = open(out, "rb").read()
        groups = api.last_grouped_run()["group_bytes"]
        assert len(groups) == (1 if name == "one" else _groups(plan, automatic))
    assert files["auto"] == files["one"]
