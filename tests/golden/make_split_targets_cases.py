"""Fixture for the split-target tests (tests/test_gpu_split_targets.py): what racon's own command line prints on its CPU
path — oracle/_ref/racon_cpu, the reference's src/main.cpp built by oracle/refcli.mk — for inputs a function of the test
suite generates (the case records the function as "generator"; the files are never committed):
  long_contig: a 60 kb contig between two 3 kb ones, FASTQ reads on both strands (write_long_contig).
Per case the same record as tests/golden/cli_cases.json: options, file names, record count, total bases, md5 of stdout and
the header lines.  Stored in tests/golden/split_targets_cases.json.  Run on a machine with the reference sources:
python tests/golden/make_split_targets_cases.py"""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refcli  # noqa: E402
from tests import test_gpu_split_targets as split  # noqa: E402
from tests.golden.make_cli_cases import _run  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "split_targets_cases.json")
# name: (options, function that writes the three files into a directory and returns their paths)
GENERATED = {"long_contig": ([], split.write_long_contig)}


def main():
    exe = refcli.build_refcli()
    assert exe, "the reference's command line needs the reference sources"
    fixture = {}
    for name, (opts, gen) in GENERATED.items():
        with tempfile.TemporaryDirectory() as d:
            paths = gen(d)
            fixture[name] = dict({"options": opts, "generator": "%s.%s" % (gen.__module__, gen.__name__),
                                  "files": [os.path.basename(p) for p in paths]}, **_run(exe, name, opts, paths))
    with open(OUT, "w") as f:
        json.dump(fixture, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
