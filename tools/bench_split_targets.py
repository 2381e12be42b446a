#!/usr/bin/env python3
"""What polishing one contig in parts costs: files -> polished FASTA (api.polish_files on device [0]) under a read store
budget that holds the whole input, and under 1/2, 1/4 and 1/8 of it with split_targets, where the contig is polished in
parts of consecutive windows.

Workload: a seeded synthetic single contig, written to a temporary directory — a random genome of --genome-mb, the draft
with 3 % substitutions, and --coverage x of FASTQ reads of about --read-len bases sampled from both strands with ONT-like
error (12 %: 5 % substitutions, 3 % insertions, 4 % deletions), one PAF line per read from the known sampling positions.

One JSON line per run: the budget and its fraction of the whole store, wall time per stage (load: parse + racon's overlap
filter, timed alone beforehand; plan: api.plan_read_groups with the window length; polish: the whole api.polish_files
call, which parses again, plans, and per group uploads the store, aligns, builds windows and polishes), the groups and parts,
each group's store bytes, the overlaps aligned (the same sum in every row), the md5 of the FASTA (the same in every row),
and the card's name and power limit.  --repeats N runs the four budgets N times, in turn.

  python tools/bench_split_targets.py [--genome-mb 20] [--coverage 30] [--read-len 10000] [--seed 1] [--repeats 1]
"""
import argparse
import hashlib
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from racon_b200 import api  # noqa: E402
from tools.bench_polish_devices import BASES, P_DEL, P_INS, P_SUB, _read, card  # noqa: E402

WINDOW = 500


def make_workload(d, genome_mb, coverage, read_len, seed):
    rng = np.random.default_rng(seed)
    g = int(genome_mb * 1e6)
    genome = rng.integers(0, 4, g).astype(np.uint8)
    draft = np.where(rng.random(g) < 0.03, (genome + rng.integers(1, 4, g)) % 4, genome).astype(np.uint8)
    with open(os.path.join(d, "contig.fasta"), "wb") as f:
        f.write(b">contig\n" + BASES[draft].tobytes() + b"\n")
    del draft
    n = int(g * coverage / read_len)
    length = rng.integers(int(read_len * 0.6), int(read_len * 1.4), n)
    start = rng.integers(0, g - length + 1)
    rev = rng.random(n) < 0.5
    read_bases = 0
    with open(os.path.join(d, "reads.fastq"), "wb") as fq, open(os.path.join(d, "overlaps.paf"), "w") as paf:
        for i in range(n):
            codes, _ = _read(rng, genome[start[i]:start[i] + length[i]])
            L = len(codes)
            read_bases += L
            seq = BASES[3 - codes[::-1]] if rev[i] else BASES[codes]
            qual = (rng.integers(8, 26, L) + 33).astype(np.uint8)
            fq.write(b"@r%d\n" % i + seq.tobytes() + b"\n+\n" + qual.tobytes() + b"\n")
            paf.write("r%d\t%d\t0\t%d\t%s\tcontig\t%d\t%d\t%d\t%d\t%d\t255\n" % (
                i, L, L, "-" if rev[i] else "+", g, start[i], start[i] + length[i], min(L, length[i]),
                max(L, length[i])))
    return dict(genome_bases=g, coverage=coverage, reads=n, read_bases=read_bases, error_rate=P_SUB + P_INS + P_DEL,
                seed=seed)


def files(d):
    return [os.path.join(d, f) for f in ("reads.fastq", "overlaps.paf", "contig.fasta")]


def plan_input(d):
    inp = api.InputFiles(*files(d))
    try:
        ov = inp.overlaps
        return (inp.n_targets, np.diff(inp.seq_off.astype(np.int64)), inp.seq_has_qual.copy(), ov[:, 0].copy(),
                ov[:, 1].copy(), ov[:, 6].copy(), ov[:, 7].copy())
    finally:
        inp.close()


def run(d, budget, out):
    t0 = time.perf_counter()
    plan = plan_input(d)
    t1 = time.perf_counter()
    groups = api.plan_read_groups(*plan[:5], budget, t_begin=plan[5], t_end=plan[6], window_length=WINDOW)
    t2 = time.perf_counter()
    n, fo, fw = api.polish_files(*files(d), out, device=[0], read_store_bytes=budget, split_targets=True)
    t3 = time.perf_counter()
    last = api.last_grouped_run()
    return dict(load_s=round(t1 - t0, 3), plan_s=round(t2 - t1, 3), polish_s=round(t3 - t2, 3),
                groups=len(last["group_bytes"]), parts=int(np.count_nonzero(groups[5])),
                group_store_bytes=last["group_bytes"], planned=last["group_bytes"] == [int(b) for b in groups[1]],
                aligned=sum(last["group_aligned"]), records=n, failed=[fo, fw],
                md5=hashlib.md5(open(out, "rb").read()).hexdigest())


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--genome-mb", type=float, default=20.0)
    ap.add_argument("--coverage", type=float, default=30.0)
    ap.add_argument("--read-len", type=int, default=10000)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=1)
    args = ap.parse_args()
    if api.device_count() < 1:
        raise SystemExit("no CUDA device: this measures a GPU")
    gpus = card()
    with tempfile.TemporaryDirectory() as d:
        t = time.perf_counter()
        size = make_workload(d, args.genome_mb, args.coverage, args.read_len, args.seed)
        size["generate_s"] = round(time.perf_counter() - t, 1)
        warm = os.path.join(d, "warm")
        os.makedirs(warm)
        make_workload(warm, 0.2, 10, 5000, args.seed + 1)   # the CUDA context and modules
        api.polish_files(*files(warm), os.path.join(warm, "o.fasta"), device=[0])
        plan = plan_input(d)
        whole = api.read_store_bytes(plan[1], plan[2])
        md5 = set()
        for _ in range(args.repeats):
            for fraction in (1, 2, 4, 8):
                budget = whole // fraction
                r = run(d, budget, os.path.join(d, "polished.fasta"))
                md5.add(r["md5"])
                print(json.dumps(dict(read_store_bytes=budget, fraction="1/%d" % fraction, workload=size,
                                      cards=gpus[:1], **r)), flush=True)
        if len(md5) != 1:
            raise SystemExit("the FASTA differs between budgets: %s" % sorted(md5))


if __name__ == "__main__":
    main()
