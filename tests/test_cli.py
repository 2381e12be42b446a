"""The racon_b200 command line (racon_b200/csrc/racon_main.cpp) up to the point where it needs a device: help and version,
racon's option parsing, and racon's checks of the arguments and input files, in racon's order.  Runs without a GPU: every
case here ends before a device is used (tests/test_gpu_cli.py runs the program to the end on the H100)."""
import os
import signal
import subprocess

import pytest

from racon_b200 import api
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "racon_b200", "lib", "racon_b200")
CONTIG = ("sample_reads.fastq.gz", "sample_overlaps.paf.gz", "sample_layout.fasta.gz")


def run_cli(args, timeout=600, env=None, stdout=subprocess.PIPE):
    """The program in a session of its own, killed with its whole group when it overruns.  env: variables set on top of
    this process's environment.  Returns (exit status, stdout bytes, stderr text)."""
    p = subprocess.Popen([CLI] + list(args), stdin=subprocess.DEVNULL, stdout=stdout, stderr=subprocess.PIPE,
                         env=dict(os.environ, **(env or {})), start_new_session=True)
    try:
        out, err = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        try:
            os.killpg(p.pid, signal.SIGKILL)
        except ProcessLookupError:
            pass
        p.communicate()
        raise
    return p.returncode, out, err.decode(errors="replace")


def sample(*names):
    d = util.sample_data_dir()
    return [os.path.join(d, n) for n in names]


NO_DEVICE = {"CUDA_VISIBLE_DEVICES": ""}   # an empty device list, on any machine


def test_cli_is_built_next_to_its_libraries():
    assert os.access(CLI, os.X_OK)
    for lib in ("libracon_b200.so", "libracon_b200_host.so"):
        assert os.path.exists(os.path.join(os.path.dirname(CLI), lib))


@pytest.mark.parametrize("flag", ["-h", "--help"])
def test_help_prints_the_usage_and_exits_0(flag):
    status, out, err = run_cli([flag])
    assert status == 0, err
    text = out.decode()
    assert text.startswith("usage: racon_b200 [options ...] <sequences> <overlaps> <target sequences>\n")
    for option in ("--include-unpolished", "--fragment-correction", "--window-length", "--quality-threshold",
                   "--error-threshold", "--no-trimming", "--match", "--mismatch", "--gap", "--threads", "--version",
                   "--cudapoa-batches", "--cuda-banded-alignment", "--cudaaligner-batches", "--cudaaligner-band-width"):
        assert option in text, option


def test_version_prints_the_library_version_and_exits_0():
    status, out, err = run_cli(["--version"])
    assert status == 0, err
    assert out.decode() == api.load(build_if_missing=False).rp_version().decode() + "\n"


@pytest.mark.parametrize("args", [["-v"], ["--verbose"], ["-z"], ["-w"], ["--cudaaligner-batches"]],
                         ids=["-v", "--verbose", "-z", "-w-without-value", "--cudaaligner-batches-without-value"])
def test_unknown_option_or_missing_value_exits_1(args):
    """racon has no -v (only --version): getopt_long refuses it like any unknown option"""
    status, out, err = run_cli(sample(*CONTIG) + args, env=NO_DEVICE)   # last: a value cannot come from a path
    assert status == 1 and out == b""
    assert "no CUDA device" not in err


@pytest.mark.parametrize("n", [0, 1, 2])
def test_fewer_than_three_paths_exits_1(n):
    status, out, err = run_cli(sample(*CONTIG)[:n], env=NO_DEVICE)
    assert status == 1 and out == b""
    assert "missing input file(s)!" in err and "usage: racon_b200" in err


def test_c_takes_the_next_word_as_its_count():
    """racon's -c rule: without an attached value the next word is the count unless it starts with '-'"""
    files = sample(*CONTIG)
    status, _, err = run_cli(["-c"] + files, env=NO_DEVICE)      # the reads path becomes the count: two paths left
    assert status == 1 and "missing input file(s)!" in err
    for args in (["-c", "2"] + files, files + ["-c", "2"], ["-c", "-u"] + files, ["-c3"] + files,
                 ["--cudapoa-batches=2"] + files, ["--cudapoa-batches", "2"] + files):
        status, out, err = run_cli(args, env=NO_DEVICE)         # three paths: the run gets as far as the device
        assert status == 1 and out == b"" and "no CUDA device" in err, (args, err)


@pytest.mark.parametrize("args", [["-t", "8"], ["--threads=8"], ["-b"], ["--cudaaligner-batches", "4"],
                                  ["--cudaaligner-band-width", "100"], ["-u", "--no-trimming", "-f", "-w", "300",
                                                                        "-q", "20", "-e", "0.1", "-m", "8", "-x", "-6",
                                                                        "-g", "-8"]])
def test_racon_options_are_accepted(args):
    status, out, err = run_cli(args + sample(*CONTIG), env=NO_DEVICE)
    assert status == 1 and out == b"" and "no CUDA device" in err, err


@pytest.mark.parametrize("position", [0, 1, 2])
def test_unsupported_extension_exits_1_with_racons_message(position, tmp_path):
    files = sample(*CONTIG)
    bad = str(tmp_path / "input.txt")
    open(bad, "w").close()
    files[position] = bad
    status, out, err = run_cli(files, env=NO_DEVICE)
    assert status == 1 and out == b""
    assert "error: file %s has unsupported format extension (valid extensions: " % bad in err


def test_window_length_0_exits_1_before_the_files_are_looked_at(tmp_path):
    for files in (sample(*CONTIG), [str(tmp_path / "r.txt"), str(tmp_path / "o.txt"), str(tmp_path / "t.txt")]):
        status, out, err = run_cli(["-w", "0"] + files, env=NO_DEVICE)
        assert status == 1 and out == b""
        assert "invalid window length!" in err and "extension" not in err


def test_extensions_are_checked_before_any_file_is_read(tmp_path):
    """racon checks the three extensions before it reads anything: a missing reads file with a good extension does not
    hide a bad target extension"""
    missing = str(tmp_path / "missing.fastq")
    bad = str(tmp_path / "targets.txt")
    status, out, err = run_cli([missing, sample(CONTIG[1])[0], bad], env=NO_DEVICE)
    assert status == 1 and out == b""
    assert "unsupported format extension" in err and "unable to open" not in err


@pytest.mark.parametrize("position", [0, 1, 2])
def test_missing_file_exits_1(position, tmp_path):
    files = sample(*CONTIG)
    files[position] = str(tmp_path / ("missing" + os.path.basename(files[position])[len("sample"):]))
    status, out, err = run_cli(files, env=NO_DEVICE)
    assert status == 1 and out == b""
    assert "unable to open file %s" % files[position] in err


def test_without_a_device_exits_1_and_prints_nothing():
    """valid arguments and files, an empty device list: the library's error, status 1, nothing on stdout (no CPU path)"""
    status, out, err = run_cli(sample(*CONTIG), env=NO_DEVICE)
    assert status == 1 and out == b""
    assert "no CUDA device (this library has no CPU fallback)" in err
