#!/usr/bin/env python3
"""Files -> polished FASTA (api.polish_files' flow: MirrorPolisher.from_files + stream_fasta) on 1, 2, ... GPUs.

Workload: a seeded synthetic fragment-correction run (racon -f), written to a temporary directory — reads sampled from a
random genome on both strands with ONT-like error (12 %: 5 % substitutions, 3 % insertions, 4 % deletions) as FASTQ, and a
PAF of every pair of reads whose genome intervals overlap by at least --min-overlap bases, with coordinates taken from the
known sampling positions (each pair once, query and target chosen at random).

Runs: device=[0], [0, 1], ..., up to every visible GPU; with one visible GPU, [0] and [0, 0] (two lanes on one GPU).  One
JSON line per run: wall time per stage (load, align + breaking points + window building, consensus + FASTA; they add up to
total_s, which is one parse + the device stages, as in polish_files), overlaps (after racon's filter) per second and windows
per second, speedup and scaling efficiency against [0] from total_s, the CPU time of the driving thread, the md5 of the
FASTA (the same in every row), and the card's name and power limit.

With --read-store-bytes B: on device [0] only, api.polish_files in target groups, alternating runs under the automatic
budget (one group here) and under B bytes per device, three of each.  One JSON line per run: the load alone, the whole
grouped run (parse, plan, and per group: store upload, alignment, window building, consensus + FASTA), the groups and their
store bytes, the md5 of the FASTA.

  python tools/bench_polish_devices.py [--genome-mb 16] [--coverage 30] [--seed 1] [--read-store-bytes B]
"""
import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from racon_b200 import api  # noqa: E402

BASES = np.frombuffer(b"ACGT", np.uint8)
P_SUB, P_INS, P_DEL = 0.05, 0.03, 0.04


def _read(rng, seg):
    """seg (codes 0..3) through the error model -> (read codes, read position of every genome base + the end)"""
    r = rng.random(len(seg))
    dele = r < P_DEL
    sub = (r >= P_DEL) & (r < P_DEL + P_SUB)
    ins = (r >= P_DEL + P_SUB) & (r < P_DEL + P_SUB + P_INS)
    emit = np.where(dele, 0, np.where(ins, 2, 1))
    pos = np.cumsum(emit) - emit
    out = np.empty(int(emit.sum()), np.uint8)
    base = np.where(sub, (seg + rng.integers(1, 4, len(seg))) % 4, seg).astype(np.uint8)
    out[pos[ins]] = rng.integers(0, 4, int(ins.sum()))
    keep = ~dele
    out[pos[keep] + ins[keep]] = base[keep]
    return out, np.append(pos, len(out))


def make_workload(d, genome_mb, coverage, read_len, min_overlap, seed):
    rng = np.random.default_rng(seed)
    g = int(genome_mb * 1e6)
    genome = rng.integers(0, 4, g).astype(np.uint8)
    n = int(g * coverage / read_len)
    length = rng.integers(int(read_len * 0.6), int(read_len * 1.4), n)
    start = np.sort(rng.integers(0, g - length.max(), n))
    end = start + length
    rev = rng.random(n) < 0.5
    # every pair (i < j by start) whose intervals overlap by min_overlap or more
    pa, pb = [], []
    for i in range(n):
        j1 = np.searchsorted(start, end[i] - min_overlap, side="right")
        js = np.arange(i + 1, j1)
        js = js[np.minimum(end[i], end[js]) - start[js] >= min_overlap]
        pa.append(np.full(len(js), i))
        pb.append(js)
    pa, pb = np.concatenate(pa), np.concatenate(pb)
    gs, ge = np.maximum(start[pa], start[pb]), np.minimum(end[pa], end[pb])
    # read coordinates of the pair boundaries, read by read
    coord = {}
    by_read = [[] for _ in range(n)]
    for k in range(len(pa)):
        by_read[pa[k]].append(k)
        by_read[pb[k]].append(k)
    read_len_out = np.zeros(n, np.int64)
    with open(os.path.join(d, "reads.fastq"), "wb") as f:
        for i in range(n):
            codes, pos = _read(rng, genome[start[i]:end[i]])
            L = len(codes)
            read_len_out[i] = L
            seq = BASES[codes]
            if rev[i]:
                seq = BASES[3 - codes[::-1]]
            qual = (rng.integers(8, 26, L) + 33).astype(np.uint8)
            f.write(b"@r%d\n" % i + seq.tobytes() + b"\n+\n" + qual.tobytes() + b"\n")
            for k in by_read[i]:
                p0, p1 = int(pos[gs[k] - start[i]]), int(pos[ge[k] - start[i]])
                coord[(k, i)] = (L - p1, L - p0) if rev[i] else (p0, p1)
    swap = rng.random(len(pa)) < 0.5
    with open(os.path.join(d, "overlaps.paf"), "w") as f:
        for k in range(len(pa)):
            q, t = (pb[k], pa[k]) if swap[k] else (pa[k], pb[k])
            q0, q1 = coord[(k, q)]
            t0, t1 = coord[(k, t)]
            span = (min(q1 - q0, t1 - t0), max(q1 - q0, t1 - t0))
            f.write("r%d\t%d\t%d\t%d\t%s\tr%d\t%d\t%d\t%d\t%d\t%d\t255\n" % (
                q, read_len_out[q], q0, q1, "-" if rev[q] != rev[t] else "+", t, read_len_out[t], t0, t1, span[0],
                span[1]))
    return dict(genome_bases=g, coverage=coverage, reads=n, read_bases=int(read_len_out.sum()), paf_lines=len(pa),
                error_rate=P_SUB + P_INS + P_DEL, min_overlap=min_overlap, seed=seed)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        return [line.strip() for line in out.splitlines() if line.strip()]
    except Exception:
        return ["unknown"]


def polish(d, devices, out):
    """What polish_files does (from_files, then stream_fasta), timed from t1 to t3.  from_files parses the files and then
    aligns and builds the windows; the parse alone is timed beforehand (t0 to t1, not part of the total), and the align
    stage is from_files' time minus it, so that the three stages add up to the total."""
    files = [os.path.join(d, f) for f in ("reads.fastq", "overlaps.paf", "reads.fastq")]
    t0, c0 = time.perf_counter(), time.thread_time()
    inp = api.InputFiles(*files, fragment_correction=True)      # the load alone (parse + overlap filter)
    n_overlaps = len(inp.overlaps)
    inp.close()
    t1, c1 = time.perf_counter(), time.thread_time()
    pol = api.MirrorPolisher.from_files(*files, fragment_correction=True, device=devices, resident_reads=True)
    t2, c2 = time.perf_counter(), time.thread_time()
    counts = (ctypes.c_uint64 * 3)()
    pol.lib.rp_mirror_polisher_counts(pol.h, counts)   # windows, pieces, bases
    try:
        n = pol.stream_fasta(out, None, drop_unpolished=True, resident_reads=True)
        failed = pol.failed()
    finally:
        pol.close()
    t3, c3 = time.perf_counter(), time.thread_time()
    load, load_cpu = t1 - t0, c1 - c0
    return dict(load_s=load, align_breaking_points_s=(t2 - t1) - load, consensus_fasta_s=t3 - t2, total_s=t3 - t1,
                cpu_s=dict(load=load_cpu, align_breaking_points=(c2 - c1) - load_cpu, consensus_fasta=c3 - c2,
                           total=c3 - c1),
                overlaps=n_overlaps, windows=int(counts[0]), records=n, failed=list(failed),
                md5=hashlib.md5(open(out, "rb").read()).hexdigest())


def polish_grouped(d, budget, out):
    """api.polish_files(read_store_bytes=budget) on device [0], timed; the load alone is timed beforehand"""
    files = [os.path.join(d, f) for f in ("reads.fastq", "overlaps.paf", "reads.fastq")]
    t0 = time.perf_counter()
    api.InputFiles(*files, fragment_correction=True).close()
    t1 = time.perf_counter()
    n, fo, fw = api.polish_files(*files, out, fragment_correction=True, device=[0], read_store_bytes=budget)
    t2 = time.perf_counter()
    groups = api.last_grouped_run()["group_bytes"]
    return dict(read_store_bytes=budget, load_s=round(t1 - t0, 3), grouped_total_s=round(t2 - t1, 3),
                groups=len(groups), group_store_bytes=groups, records=n, failed=[fo, fw],
                md5=hashlib.md5(open(out, "rb").read()).hexdigest())


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--genome-mb", type=float, default=16.0)
    ap.add_argument("--coverage", type=float, default=30.0)
    ap.add_argument("--read-len", type=int, default=10000)
    ap.add_argument("--min-overlap", type=int, default=1000)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--read-store-bytes", type=int, default=None,
                    help="compare target groups under this budget with the automatic budget, on device [0]")
    args = ap.parse_args()
    n_gpus = api.device_count()
    if n_gpus < 1:
        raise SystemExit("no CUDA device: this measures GPUs")
    runs = [list(range(k)) for k in range(1, n_gpus + 1)] if n_gpus > 1 else [[0], [0, 0]]
    gpus = card()
    with tempfile.TemporaryDirectory() as d:
        t = time.perf_counter()
        size = make_workload(d, args.genome_mb, args.coverage, args.read_len, args.min_overlap, args.seed)
        size["generate_s"] = round(time.perf_counter() - t, 1)
        warm = os.path.join(d, "warm")
        os.makedirs(warm)
        make_workload(warm, 0.2, 10, 5000, 1000, args.seed + 1)     # CUDA contexts and modules on every device
        polish(warm, sorted(set(sum(runs, []))), os.path.join(warm, "o.fasta"))
        if args.read_store_bytes is not None:
            for budget in (0, args.read_store_bytes) * 3:
                row = dict(workload=size, cards=gpus[:1], **polish_grouped(d, budget, os.path.join(d, "polished.fasta")))
                print(json.dumps(row), flush=True)
            return
        base = None
        for devices in runs:
            r = polish(d, devices, os.path.join(d, "polished.fasta"))
            if base is None:
                base = r["total_s"]
            distinct = len(set(devices))
            cards = [gpus[i] if i < len(gpus) else "?" for i in sorted(set(devices))]
            row = dict(devices=devices, workload=size, cards=cards,
                       stages_s={k: round(r[k], 3) for k in ("load_s", "align_breaking_points_s", "consensus_fasta_s",
                                                             "total_s")},
                       overlaps=r["overlaps"], overlaps_per_s=round(r["overlaps"] / r["align_breaking_points_s"], 1),
                       windows=r["windows"], windows_per_s=round(r["windows"] / r["consensus_fasta_s"], 1),
                       speedup_vs_one=round(base / r["total_s"], 3),
                       scaling_efficiency=round(base / r["total_s"] / distinct, 3),
                       driver_thread_cpu_s={k: round(v, 3) for k, v in r["cpu_s"].items()},
                       records=r["records"], failed=r["failed"], md5=r["md5"])
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
