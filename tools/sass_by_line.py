#!/usr/bin/env python
"""Static instruction counts of one kernel by source line / function, from the SASS (no GPU needed).

  python tools/sass_by_line.py [--kernel 'rp_poa_kernelILi32ELi16ELi3E'] [--lines poa_core.cuh:1300-1520] [--top 40]

cuobjdump extracts the sm_90a cubin of racon_b200/lib/libracon_b200.so, `nvdisasm -g` annotates every instruction with
the source line it was generated for (the library is built with -lineinfo).  The counts are STATIC (instructions in the
binary, not executed ones): they are what a change of the source can be checked against before any GPU time is spent —
together with `ncu_by_line.py`'s dynamic counts from a capture.  --lines prints the listing of a source range."""
import argparse
import collections
import os
import re
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def disassemble(lib, kernel):
    with tempfile.TemporaryDirectory(prefix="sass_") as tmp:
        subprocess.run(["cuobjdump", "-xelf", "all", lib], cwd=tmp, check=True, stdout=subprocess.DEVNULL)
        cubin = [os.path.join(tmp, f) for f in os.listdir(tmp) if f.endswith(".cubin")][0]
        out = subprocess.run(["nvdisasm", "-g", cubin], stdout=subprocess.PIPE, text=True, check=True).stdout
    sect, keep = None, []
    for line in out.splitlines():
        m = re.match(r"\s*\.section\s+\.text\.(\S+?),", line)
        if m:
            sect = m.group(1)
            continue
        if line.startswith("//-----") or re.match(r"\s*\.section", line):
            sect = None if not m else sect
        if sect and kernel in sect and not sect.startswith("$"):
            keep.append(line)
    return keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "racon_b200", "lib", "libracon_b200.so"))
    ap.add_argument("--kernel", default="rp_poa_kernelILi32ELi16ELi3E")
    ap.add_argument("--lines", help="file.cuh:first-last : print the SASS generated for that source range")
    ap.add_argument("--top", type=int, default=40)
    ap.add_argument("--range", help="lo-hi (hex addresses): plain listing of that address range, source lines beside it")
    ap.add_argument("--where", help="file.cuh:line : address ranges (clusters) of the instructions generated for that line, "
                                    "e.g. a loop statement -> the extent of each copy of the loop")
    ap.add_argument("--grep", help="regular expression over the instruction text: list the matches with their source lines")
    args = ap.parse_args()
    lines = disassemble(args.lib, args.kernel)
    cur = ("?", 0)
    per_line = collections.Counter()
    listing = []
    n = 0
    for ln in lines:
        m = re.search(r'//## File "([^"]+)", line (\d+)', ln)
        if m:
            cur = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = re.match(r"\s*/\*([0-9a-f]+)\*/\s+(.*?);", ln)
        if m:
            per_line[cur] += 1
            n += 1
            listing.append((cur, m.group(1), m.group(2).strip()))
    print("kernel %s: %d instructions" % (args.kernel, n))
    if args.range:
        lo, _, hi = args.range.partition("-")
        lo, hi = int(lo, 16), int(hi, 16)
        for (cf, cl), addr, ins in listing:
            if lo <= int(addr, 16) <= hi:
                print("/*%s*/  %-60s // %s:%d" % (addr, ins + " ;", cf, cl))
        return
    if args.where:
        f, _, ln = args.where.partition(":")
        ads = sorted(int(addr, 16) for (cf, cl), addr, ins in listing if cf == f and cl == int(ln))
        start = prev = None
        for a in ads:
            if start is None or a - prev > 0x3000:
                if start is not None:
                    print("0x%x-0x%x" % (start, prev))
                start = a
            prev = a
        if start is not None:
            print("0x%x-0x%x" % (start, prev))
        return
    if args.grep:
        for (cf, cl), addr, ins in listing:
            if re.search(args.grep, ins):
                print("%s:%-5d /*%s*/ %s" % (cf, cl, addr, ins))
        return
    if args.lines:
        f, _, rng = args.lines.partition(":")
        a, _, b = rng.partition("-")
        a, b = int(a), int(b or a)
        tot = 0
        for (cf, cl), addr, ins in listing:
            if cf == f and a <= cl <= b:
                print("%s:%-5d /*%s*/ %s" % (cf, cl, addr, ins))
                tot += 1
        print("-- %d instructions for %s" % (tot, args.lines))
        return
    for (f, l), c in per_line.most_common(args.top):
        print("%6d  %s:%d" % (c, f, l))


if __name__ == "__main__":
    main()
