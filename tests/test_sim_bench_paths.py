"""The POA batch object's per-launch DP counters (rp_poa_info [5]-[7]) and a relaunched resident batch, on a machine without
a GPU: the C ABI over the simulated CUDA runtime (build.build_simapi), in a process of its own with RACON_B200_LIB pointing at
it.  The counters are the bytes bench.py's roofline divides by the kernel time; every launch must count that launch alone,
whatever ran on the object before, and equal what the oracle counts on the same windows.  The full set of these checks
runs on the device in tests/test_gpu_bench_paths.py."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle_counts(ws):
    from oracle import bindings as ob
    out = np.zeros(12, np.uint64)
    ob.oracle_lib().oracle_poa_stats(out.ctypes.data)      # reading the oracle's counters zeroes them
    cons, pol, _ = ob.oracle_consensus(ws, window_length=100)
    ob.oracle_lib().oracle_poa_stats(out.ctypes.data)
    return [int(v) for v in out[:3]], cons, pol


def _counts(b):
    i = b.info()
    return [i["alignments"], i["dp_cells"], i["pred_cells"]]


def _results(b, n):
    out, lens, pol, st = b.fetch_all(512)
    return [out[w, :lens[w]].tobytes().decode() for w in range(n)], [bool(p) for p in pol], [int(s) for s in st]


def figures():
    """Runs in the child process: what the counters and the results were after each way of driving one batch object."""
    from racon_b200 import api
    from tests import util
    ws = util.make_set(3, 4, wlen=80, depth=6, err=0.1, partial_frac=0.3)
    ws2 = util.make_set(4, 3, wlen=60, depth=5, err=0.1, partial_frac=0.3)
    want, cons, pol = _oracle_counts(ws)
    want2, _, _ = _oracle_counts(ws2)
    r = {"oracle": want, "oracle_other_batch": want2,
         "oracle_results": [[c.decode() for c in cons], [bool(p) for p in pol], [0] * ws.n_windows]}
    b = api.PoaBatch(window_length=100)
    try:
        b.add_window_set(ws)
        b.run()                      # counters off
        b.sync()
        r["off"] = _counts(b)
        b.enable_counters(True)
        b.run()
        b.sync()
        r["run"] = _counts(b)
        r["run_results"] = _results(b, ws.n_windows)
        b.run()
        b.sync()
        r["run_again"] = _counts(b)
        b.upload()                   # bench.py's resident relaunches
        b.launch()
        b.launch()
        b.download()
        b.sync()
        r["relaunch"] = _counts(b)
        r["relaunch_results"] = _results(b, ws.n_windows)
        r["launches"] = b.info()["launches"]
        b.reset()
        b.add_window_set(ws)
        b.run()
        b.sync()
        r["reset_same"] = _counts(b)
        b.reset()
        b.add_window_set(ws2)
        b.run()
        b.sync()
        r["reset_other"] = _counts(b)
    finally:
        b.close()
    return r


def test_counters_count_each_launch_alone_over_the_simulated_runtime():
    from racon_b200 import build
    env = dict(os.environ, RACON_B200_LIB=build.build_simapi())
    code = ("import sys, json; sys.path.insert(0, %r)\n"
            "from tests.test_sim_bench_paths import figures\n"
            "print('FIGURES ' + json.dumps(figures()))\n" % ROOT)
    p = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=900)
    lines = [l for l in p.stdout.splitlines() if l.startswith("FIGURES ")]
    assert p.returncode == 0 and len(lines) == 1, p.stdout[-3000:]
    r = json.loads(lines[0][len("FIGURES "):])
    want = r["oracle"]
    assert want[0] > 0 and r["off"] == [0, 0, 0], r
    table = {k: r[k] for k in ("run", "run_again", "relaunch", "reset_same")}
    assert all(v == want for v in table.values()), "alignments / DP cells / predecessor cells %s, oracle %s" % (table, want)
    assert r["reset_other"] == r["oracle_other_batch"], r
    assert r["launches"] == 5, r      # one kernel launch per run / launch: nothing went through the escalation pass
    assert r["run_results"] == r["oracle_results"] and r["relaunch_results"] == r["run_results"], r
