"""Polishing on a list of devices (racon_b200::Polisher's lanes, host_mirror.hpp): one lane per entry of `device`, batches
handed out from a shared cursor, collected in whatever order the devices finish them, stitched back into window order.
The output must not depend on the list: every run here is checked against the reference's bytes or the one-lane run.
A one-GPU machine runs the multi-lane code with a repeated index ([0, 0] = two lanes on GPU 0); only the last test needs
two GPUs.  The stitch cursor and the argument checks are host logic and run without a GPU."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from racon_b200 import api, build
from tests.lambda_overlaps import LambdaOverlaps
from tests.test_reads_io import CASES, DATA, GOLD
from tests.test_zz_files_pipeline import _records

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _files(case):
    reads, overlaps, target, frag, e = CASES[case]
    return [os.path.join(DATA, f) for f in (reads, overlaps, target)], dict(fragment_correction=frag, error_threshold=e)


# ---- host logic: the stitch cursor ------------------------------------------------------------------------------------
def _check_stitch_order(counts, completion):
    counts = np.asarray(counts, np.int64)
    order, step = api.stitch_order(counts, completion)
    assert np.array_equal(order, np.arange(counts.sum())), "every window once, in window order"
    position = np.empty(len(counts), np.int64)
    position[np.asarray(completion)] = np.arange(len(counts))
    # range r's windows are stitched by the finish that completes ranges 0..r — not before, and not later
    due = np.maximum.accumulate(position)
    assert np.array_equal(step, np.repeat(due, counts))


@pytest.mark.parametrize("seed", range(40))
def test_stitch_cursor_emits_windows_in_order_whatever_the_completion_order(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 201))
    _check_stitch_order(rng.integers(1, 50, n), rng.permutation(n))


@pytest.mark.parametrize("n", [1, 2, 200])
def test_stitch_cursor_at_the_extremes_of_completion_order(n):
    counts = np.arange(n) % 7 + 1
    _check_stitch_order(counts, np.arange(n))           # in order: every finish stitches its own range
    _check_stitch_order(counts, np.arange(n)[::-1])     # reversed: nothing is stitched before the last finish
    _check_stitch_order(counts, np.roll(np.arange(n), -1))   # range 0 last: everything waits for it


# ---- argument checks ----------------------------------------------------------------------------------------------
def test_an_empty_device_list_is_a_clean_error(tmp_path):
    paths, kw = _files("fastq_sam")
    for empty in ([], (), range(0)):
        with pytest.raises(api.RaconB200Error, match="empty device list"):
            api.polish_files(*paths, str(tmp_path / "o.fasta"), device=empty, **kw)
        with pytest.raises(api.RaconB200Error, match="empty device list"):
            api.MirrorPolisher.from_files(*paths, device=empty, **kw)
    assert not os.path.exists(tmp_path / "o.fasta")


def test_a_device_index_that_does_not_exist_is_a_clean_error(tmp_path, monkeypatch):
    """With two visible devices, index 2 does not exist (nor does a negative one); the list is refused before any device
    is touched."""
    monkeypatch.setattr(api, "device_count", lambda: 2)
    paths, kw = _files("fastq_sam")
    for bad in ([0, 2], [2], 7, -1, [0, -1], ["0"], [0.0]):
        with pytest.raises(api.RaconB200Error):
            api.polish_files(*paths, str(tmp_path / "o.fasta"), device=bad, **kw)
    assert not os.path.exists(tmp_path / "o.fasta")
    assert list(api._device_list(range(2))) == [0, 1] and list(api._device_list([1, 1, 0])) == [1, 1, 0]
    assert list(api._device_list(np.int64(1))) == [1]


_OPEN_ON = """
import ctypes as C, os, sys
import numpy as np
from racon_b200 import api
from tests.test_reads_io import CASES, DATA
reads, overlaps, target, _, _ = CASES["fastq_sam"]
lib = api.load()
devices = np.array([int(d) for d in sys.argv[1].split(",")], np.uint32)
err = C.create_string_buffer(1024)
h = lib.rp_mirror_polisher_open_files(*[os.fsencode(os.path.join(DATA, f)) for f in (reads, overlaps, target)], 0, 500,
                                      10.0, 0.3, 1, 3, -5, -4, devices.ctypes.data, len(devices), 0, err, 1024)
print("opened" if h else err.value.decode())
"""


def test_the_host_layer_itself_refuses_a_device_index_past_the_visible_devices():
    """racon_b200::Polisher, called past the Python checks: over the simulated runtime playing two devices, [0, 1] opens the
    SAM files (which need no device to build their windows) and [0, 2] ends the process with the polisher's message."""
    env = dict(os.environ, RACON_B200_LIB=build.build_simapi(), RP_SIM_DEVICES="2")
    run = [subprocess.run([sys.executable, "-c", _OPEN_ON, devices], cwd=ROOT, env=env, stdout=subprocess.PIPE,
                          stderr=subprocess.PIPE, text=True, timeout=300) for devices in ("0,1", "0,2")]
    assert run[0].returncode == 0 and run[0].stdout.strip() == "opened", run[0].stderr
    assert run[1].returncode == 1 and "opened" not in run[1].stdout
    assert "[racon_b200::Polisher] error: device 2 out of range (2 CUDA devices)!" in run[1].stderr


# ---- on the device ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_a_device_index_past_the_visible_devices_is_a_clean_error(tmp_path):
    paths, kw = _files("fastq_paf")
    with pytest.raises(api.RaconB200Error, match="out of range"):
        api.polish_files(*paths, str(tmp_path / "o.fasta"), device=[0, api.device_count()], **kw)


@pytest.mark.gpu
def test_query_reports_a_finished_run_without_blocking():
    """rp_aln_query / rp_poa_query: RP_ERR_STATE before a run, RP_OK once the run has finished (after a sync at the
    latest), RP_ERR_STATE again after a reset."""
    a = api.AlnBatch()
    try:
        with pytest.raises(api.RaconB200Error, match="query before run"):
            a.ready()
        assert a.add(b"ACGTACGTTACG" * 20, b"ACGTACGTACG" * 20)
        a.run()
        a.ready()                       # True or False: it only must not fail or block
        a.sync()
        assert a.ready()
        a.reset()
        with pytest.raises(api.RaconB200Error, match="query before run"):
            a.ready()
    finally:
        a.close()
    p = api.PoaBatch(window_length=100)
    try:
        with pytest.raises(api.RaconB200Error, match="query before run"):
            p.ready()
        backbone = b"ACGTTGCA" * 10
        assert p.add_window([(backbone, None, 0, 0)] + [(backbone[1:], None, 1, 79)] * 3) == api.RP_OK
        p.run()
        p.ready()
        p.sync()
        assert p.ready()
        assert p.fetch(0)[0]
    finally:
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("resident", [False, True], ids=["copied", "resident"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_files_on_two_lanes_of_one_gpu_give_the_reference_records(case, resident, tmp_path):
    """Every file combination of the reference's tests, both read modes, on two lanes of GPU 0: the reference's records
    (count, bases, md5, names and tags), nothing refused."""
    g = np.load(GOLD)
    paths, kw = _files(case)
    out = str(tmp_path / "polished.fasta")
    n, fo, fw = api.polish_files(*paths, out, device=[0, 0], drop_unpolished=False, resident_reads=resident, **kw)
    assert (fo, fw) == (0, 0)
    names, seqs = _records(out)
    count, bases = (int(x) for x in g[case + "/polished"])
    assert n == count == len(seqs)
    assert sum(len(s) for s in seqs) == bases
    assert hashlib.md5(b"".join(seqs)).hexdigest() == g[case + "/polished_md5"].tobytes().decode()
    assert names == g[case + "/polished_names"].tobytes().decode().split("\n")


def _frag_polisher(device):
    lam = LambdaOverlaps("lambda_frag_overlaps.npz")
    m, x, g = (int(v) for v in lam.z["scores"])
    pol = api.MirrorPolisher(lam.bases, lam.quals, lam.seq_off, lam.seq_has_qual, n_targets=len(lam.seq_off) - 1,
                             overlaps=lam.ov, window_length=lam.window_length, quality_threshold=lam.quality_threshold,
                             trim=True, match=m, mismatch=x, gap=g, window_type_tgs=True, fragment_correction=True,
                             device=device)
    return lam, pol


@pytest.mark.gpu
def test_many_batches_on_three_lanes_give_the_reference_reads(tmp_path):
    """racon -f on the lambda sample with a 40 MB budget per batch object: dozens of batches over six objects on three
    lanes of GPU 0, collected out of order; the 236 corrected reads come out in target order with the reference's bytes,
    and nothing is refused — as on one lane."""
    failed = {}
    for device in ([0, 0, 0], [0]):
        lam, pol = _frag_polisher(device)
        n_seq = len(lam.seq_off) - 1
        out = str(tmp_path / ("corrected_%d.fasta" % len(device)))
        try:
            n = pol.stream_fasta(out, ["read%d" % i for i in range(n_seq)], drop_unpolished=False, mem_bytes=40 << 20)
            failed[len(device)] = pol.failed()
        finally:
            pol.close()
        assert n == 236
        lines = open(out, "rb").read().split(b"\n")
        data = b"".join(lines[1::2])
        assert len(data) == 1658216
        assert hashlib.md5(data).hexdigest() == lam.z["polished_md5"].tobytes().decode()
    assert failed[3] == failed[1] == (0, 0)


@pytest.mark.gpu
def test_breaking_points_on_two_lanes_equal_one_lane_and_the_reference():
    """The 7 780 all-vs-all overlaps of the -f flow aligned on two lanes of GPU 0: per overlap the breaking points of the
    one-lane run, which are the reference's."""
    got = {}
    for device in ([0], [0, 0]):
        lam, pol = _frag_polisher(device)
        try:
            got[len(device)] = pol.breaking_points()
            assert pol.failed()[0] == 0
        finally:
            pol.close()
    assert lam.n_overlaps() == 7780
    (off1, bp1), (off2, bp2) = got[1], got[2]
    assert np.array_equal(off1, off2) and np.array_equal(bp1, bp2)
    assert np.array_equal(off1, lam.bp_off) and np.array_equal(bp1, lam.bp.reshape(-1, 2))


@pytest.mark.gpu
def test_every_visible_gpu_gives_the_one_gpu_fasta(tmp_path):
    """device=range(device_count()): the same file, byte for byte, as device=[0]."""
    if api.device_count() < 2:
        pytest.skip("needs at least two visible GPUs")
    paths, kw = _files("frag_fastq_paf")
    md5 = {}
    for name, device in (("one", [0]), ("all", range(api.device_count()))):
        out = str(tmp_path / (name + ".fasta"))
        n, fo, fw = api.polish_files(*paths, out, device=device, mem_bytes=64 << 20, **kw)
        assert n > 0 and (fo, fw) == (0, 0)
        md5[name] = hashlib.md5(open(out, "rb").read()).hexdigest()
    assert md5["all"] == md5["one"]
