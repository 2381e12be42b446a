"""The racon_b200 command line end to end on the device: for racon's option set on the lambda-phage sample files, stdout
equals what racon's own command line prints on its CPU path (tests/golden/cli_cases.json, made by
tests/golden/make_cli_cases.py from the reference's src/main.cpp): md5, record count, bases, names and tags.  The CUDA
options and the number of GPUs change nothing in the bytes; items the device refuses give exit status 2; a failed write
gives exit status 1."""
import hashlib
import json
import os

import pytest

from tests.test_cli import CONTIG, ROOT, run_cli, sample

pytestmark = pytest.mark.gpu

with open(os.path.join(ROOT, "tests", "golden", "cli_cases.json")) as _f:
    FIXTURE = json.load(_f)


def _check(case, status, out, err):
    want = FIXTURE[case]
    assert status == want.get("expected_status", 0), err
    if status == 0:
        assert "refused" not in err and "exceeded device limit" not in err, err
    lines = out.split(b"\n")
    names, seqs = lines[0:-1:2], lines[1:-1:2]
    assert len(seqs) == want["count"]
    assert sum(len(s) for s in seqs) == want["bases"]
    assert [n[1:].decode() for n in names] == want["names"]
    assert hashlib.md5(out).hexdigest() == want["md5"]


def _args(case):
    return FIXTURE[case]["options"] + sample(*FIXTURE[case]["files"])


@pytest.mark.parametrize("case", sorted(k for k in FIXTURE if "generator" not in FIXTURE[k]))
def test_stdout_equals_racons(case):
    """the sample-file cases; those whose inputs a generator writes are run by the generator's own test module"""
    _check(case, *run_cli(_args(case)))


CUDA_OPTIONS = {
    "paths_then_-c": sample(*CONTIG) + ["-c"],   # first, "-c" would take the reads path for its count
    "-c_2": ["-c", "2"] + sample(*CONTIG),
    "-c2": ["-c2"] + sample(*CONTIG),
    "-c_-b": ["-c", "-b"] + sample(*CONTIG),   # the next word is an option: one lane
    "--cudapoa-batches=2": ["--cudapoa-batches=2"] + sample(*CONTIG),
    "paths_then_-c_2": sample(*CONTIG) + ["-c", "2"],
    "-b": ["-b"] + sample(*CONTIG),
    "-c_2_-b": ["-c", "2", "-b"] + sample(*CONTIG),
    "--cudaaligner-batches_1": ["--cudaaligner-batches", "1"] + sample(*CONTIG),
    "--cudaaligner-band-width_100": ["--cudaaligner-band-width", "100"] + sample(*CONTIG),
    "-t_4": ["-t", "4"] + sample(*CONTIG),
}


@pytest.mark.parametrize("name", sorted(CUDA_OPTIONS))
def test_cuda_options_do_not_change_the_output(name):
    """-c (lanes per GPU), -b (banded consensus) and the aligner options racon takes: the default run's bytes"""
    _check("fastq_paf", *run_cli(CUDA_OPTIONS[name]))


@pytest.mark.parametrize("case", ["fastq_paf", "frag_fastq_paf"])
def test_every_visible_gpu_gives_the_bytes_of_gpu_0(case):
    everyone = run_cli(_args(case))
    one = run_cli(_args(case), env={"CUDA_VISIBLE_DEVICES": "0"})
    _check(case, *one)
    assert everyone[:2] == one[:2]


def _write_refused_case(tmp_path):
    """A 1.2 kb FASTA target, three exact copies of it as reads, and a fourth read over the same span that uses 17 distinct
    letters — one more than the aligner takes (RP_ALN_ALPHABET_LIMIT)."""
    import numpy as np
    rng = np.random.default_rng(17)
    target = bytes(b"ACGT"[i] for i in rng.integers(4, size=1200))
    odd = bytearray(target)
    for k, c in enumerate(b"BDEFHIJKLMNOP"):   # 13 more letters: 17 in all
        odd[50 + 70 * k] = c
    (tmp_path / "t.fasta").write_bytes(b">contig\n" + target + b"\n")
    reads = [(b"r%d" % i, target) for i in range(3)] + [(b"odd", bytes(odd))]
    (tmp_path / "r.fasta").write_bytes(b"".join(b">" + n + b"\n" + s + b"\n" for n, s in reads))
    (tmp_path / "o.paf").write_bytes(b"".join(b"%s\t1200\t0\t1200\t+\tcontig\t1200\t0\t1200\t1200\t1200\t60\n" % n
                                              for n, _ in reads))
    return [str(tmp_path / "r.fasta"), str(tmp_path / "o.paf"), str(tmp_path / "t.fasta")]


def test_refused_overlap_gives_status_2_and_still_writes_the_output(tmp_path):
    status, out, err = run_cli(_write_refused_case(tmp_path))
    assert status == 2, err
    summary = [line for line in err.splitlines() if "refused" in line]
    assert len(summary) == 1, err
    refused_overlaps = int(summary[0].split("refused ")[1].split(" overlap")[0])
    assert refused_overlaps >= 1
    assert out.startswith(b">contig LN:i:") and out.count(b"\n") == 2


@pytest.mark.parametrize("case", ["fastq_paf", "frag_fastq_paf"])
def test_failed_write_exits_1(case):
    """a full disk (/dev/full) and a pipe whose reader has gone: status 1 with the write error.  The contig's one record
    fails at the final flush, the -f run's 1.4 MB fail in mid-stream, while batches are still on the device."""
    with open("/dev/full", "wb") as full:
        status, _, err = run_cli(_args(case), stdout=full)
    assert status == 1 and "writing the output failed: No space left on device" in err, err
    r, w = os.pipe()
    os.close(r)
    try:
        status, _, err = run_cli(_args(case), stdout=w)
    finally:
        os.close(w)
    assert status == 1 and "writing the output failed: Broken pipe" in err, err
