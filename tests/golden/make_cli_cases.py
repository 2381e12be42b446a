"""Fixture for the racon_b200 command line (racon_b200/csrc/racon_main.cpp): what racon's own command line prints on its
CPU path — oracle/_ref/racon_cpu, the reference's src/main.cpp built by oracle/refcli.mk — for the lambda-phage
sample files (tests/golden/data) over racon's option set:
  the seven file combinations of tests/test_reads_io.py::CASES with their own -f / -e, at racon's defaults;
  on the contig FASTQ + PAF case: -u, --no-trimming, -u --no-trimming, -w 200, -w 1000, -q 20, -u -q 20, -e 0.1,
  -m 5 -x -4 -g -8 and medaka's recommended scores -m 8 -x -6 -g -8;
  on the fragment-correction FASTQ + PAF case: -f -u, -f --no-trimming -w 300 and -f -u -m 1 -x -1 -g -1 (the run
  of racon's own tests).
Generated inputs, whose files are written by a function of the test suite and never committed (the case records the
function as "generator"): a deep amplicon, 66 000 reads through one window (tests/test_gpu_poa_depth.py).
Per case: the options and the three files, the record count, the total bases, the md5 of stdout
and the header lines (name + tags).  racon's output does not depend on its thread count, so it runs with -t 8 here.
Stored in tests/golden/cli_cases.json.  Run on a machine with the reference sources:  python tests/golden/make_cli_cases.py
[case ...] (only the named cases are remade, the others are kept)"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refcli  # noqa: E402
from tests import test_gpu_poa_depth as depth, util  # noqa: E402
from tests.test_reads_io import CASES  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "cli_cases.json")
CONTIG = "fastq_paf"
FRAG = "frag_fastq_paf"
# name: (file combination of CASES, options beyond the combination's own)
VARIANTS = {
    "fastq_paf_u": (CONTIG, ["-u"]),
    "fastq_paf_no_trimming": (CONTIG, ["--no-trimming"]),
    "fastq_paf_u_no_trimming": (CONTIG, ["-u", "--no-trimming"]),
    "fastq_paf_w200": (CONTIG, ["-w", "200"]),
    "fastq_paf_w1000": (CONTIG, ["-w", "1000"]),
    "fastq_paf_q20": (CONTIG, ["-q", "20"]),   # no window of the sample is polished: no record
    "fastq_paf_u_q20": (CONTIG, ["-u", "-q", "20"]),
    "fastq_paf_e0.1": (CONTIG, ["-e", "0.1"]),
    "fastq_paf_m5_x-4_g-8": (CONTIG, ["-m", "5", "-x", "-4", "-g", "-8"]),
    "fastq_paf_m8_x-6_g-8": (CONTIG, ["-m", "8", "-x", "-6", "-g", "-8"]),   # medaka's recommended racon scores
    "frag_fastq_paf_u": (FRAG, ["-u"]),
    "frag_fastq_paf_no_trimming_w300": (FRAG, ["--no-trimming", "-w", "300"]),
    # the scores of racon's own fragment-correction tests (test/racon_test.cpp: 236 reads, 1 658 216 bases)
    "frag_fastq_paf_u_m1_x-1_g-1": (FRAG, ["-u", "-m", "1", "-x", "-1", "-g", "-1"]),
}


def cases():
    """name -> (options, [reads, overlaps, targets]) in a fixed order"""
    out = {}
    for name in sorted(CASES):
        reads, overlaps, target, frag, e = CASES[name]
        out[name] = ((["-f"] if frag else []) + (["-e", repr(e)] if e != 0.3 else []), [reads, overlaps, target])
    for name, (base, extra) in VARIANTS.items():
        opts, files = out[base]
        out[name] = (opts + extra, files)
    return out


# name: (options, function that writes the three files into a directory and returns their paths)
GENERATED = {"deep_amplicon": ([], depth.write_deep_amplicon)}


def summary(stdout):
    """count, bases, md5 of the whole stdout, header lines (without '>') of a FASTA with one line per sequence"""
    lines = stdout.split(b"\n")
    assert lines[-1] == b"" and len(lines) % 2 == 1, "not one line per record"
    names, seqs = lines[0:-1:2], lines[1:-1:2]
    assert all(n.startswith(b">") for n in names)
    return {"count": len(seqs), "bases": sum(len(s) for s in seqs), "md5": hashlib.md5(stdout).hexdigest(),
            "names": [n[1:].decode() for n in names]}


def _run(exe, name, opts, paths):
    r = subprocess.run([exe] + opts + ["-t", "8"] + paths, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                       timeout=3600)
    assert r.returncode == 0, (name, r.returncode)
    rec = summary(r.stdout)
    print("%-34s %3d records %9d bases  %s" % (name, rec["count"], rec["bases"], rec["md5"]))
    return rec


def main(only=()):
    exe = refcli.build_refcli()
    assert exe, "the reference's command line needs the reference sources"
    data = util.sample_data_dir()
    fixture = {}
    if only:
        with open(OUT) as f:
            fixture = json.load(f)
    for name, (opts, files) in cases().items():
        if not only or name in only:
            fixture[name] = dict({"options": opts, "files": files},
                                 **_run(exe, name, opts, [os.path.join(data, f) for f in files]))
    for name, (opts, gen) in GENERATED.items():
        if not only or name in only:
            with tempfile.TemporaryDirectory() as d:
                paths = gen(d)
                fixture[name] = dict({"options": opts, "generator": "%s.%s" % (gen.__module__, gen.__name__),
                                      "files": [os.path.basename(p) for p in paths]}, **_run(exe, name, opts, paths))
    with open(OUT, "w") as f:
        json.dump(fixture, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1:])
