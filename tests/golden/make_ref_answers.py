"""Generates tests/golden/ref_answers.json: what the UNMODIFIED reference (oracle/_ref, built by oracle/Makefile) answers
on the inputs of tests/test_oracle.py (spoa consensus through Window::generate_consensus), on one seed of each tie-rich
window generator of tests/test_gpu_poa_ties.py, and on those of tests/test_myers_oracle.py (edlib CIGARs), so that those comparisons also run where oracle/_ref is not built.  Run where it is:
    python tests/golden/make_ref_answers.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import bindings as ob  # noqa: E402
from tests import test_gpu_poa_ties as tt, test_myers_oracle as tm, test_oracle as to, util  # noqa: E402


def main():
    assert ob.have_ref(), "oracle/_ref/libracon_ref.so is not built"
    poa = {}
    for name in sorted(to.CASES):
        for scores in to.SCORES:
            poa["%s/%d,%d,%d" % ((name,) + scores)] = util.consensus_answer(*to.equals_reference_case(name, scores)(
                ob.ref_consensus))
    for name in sorted(to.EXTREME_SCORES):
        for scores in to.EXTREME_SCORES[name]:
            poa["%s/%d,%d,%d" % ((name,) + scores)] = util.consensus_answer(*to.equals_reference_case(name, scores)(
                ob.ref_consensus))
    poa["partial/no_trim"] = util.consensus_answer(*to.no_trim_case()(ob.ref_consensus))
    for kind in sorted(tt.KINDS):
        case = tt.pinned_case(kind)
        for scores in tt.SCORES:
            poa[tt.pinned_key(kind, scores)] = util.consensus_answer(*case(ob.ref_consensus, scores))
    edlib = {}
    for n, err, count in tm.TRACEBACK:
        edlib["traceback/%d" % n] = [util.cigar_answer(ob.ref_edlib_cigar(q, t)) for q, t in tm.traceback_pairs(n, err, count)]
    for n, err, count in tm.HIRSCHBERG:
        edlib["hirschberg/%d" % n] = [util.cigar_answer(ob.ref_edlib_cigar(q, t))
                                      for q, t in tm.hirschberg_pairs(n, err, count)]
    edlib["degenerate"] = [util.cigar_answer(ob.ref_edlib_cigar(q, t)) for q, t in tm.DEGENERATE]
    for n in tm.TIES_TRACEBACK + tm.TIES_HIRSCHBERG:
        edlib["ties/%d" % n] = [util.cigar_answer(ob.ref_edlib_cigar(q, t)) for q, t in tm.tie_pairs(n)]
    with open(os.path.join(ROOT, "tests", "golden", "ref_answers.json"), "w") as f:
        json.dump({"source": "oracle/_ref (the unmodified reference)", "poa": poa, "edlib": edlib}, f,
                  separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
