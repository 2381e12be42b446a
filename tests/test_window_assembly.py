"""Host logic of the pipeline without a GPU: racon_b200::Polisher::build_windows (src/polisher.cpp:383-461 — layer
length and mean-quality filters, window ids, window-relative positions, strand handling) fed with the reference's own
breaking points must rebuild the reference's own window set (both fixtures come from the unmodified reference)."""
import os

import numpy as np

from tests.lambda_overlaps import LambdaOverlaps

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _build(lam, ref, n_targets, fragment):
    from racon_b200 import api
    pol = api.MirrorPolisher(lam.bases, lam.quals, lam.seq_off, lam.seq_has_qual, n_targets=n_targets, overlaps=lam.ov,
                             window_length=lam.window_length, quality_threshold=lam.quality_threshold,
                             window_type_tgs=bool(ref["win_type"][0]), fragment_correction=fragment,
                             breaking_points=(lam.bp_off, lam.bp))
    got = pol.export()
    pol.close()
    return got


def test_windows_from_reference_breaking_points_contig():
    lam = LambdaOverlaps()
    ref = np.load(os.path.join(GOLD, "lambda_windows.npz"))
    got = _build(lam, ref, 1, False)
    for k in ("win_first", "win_type", "win_target", "win_rank", "seq_off", "seq_begin", "seq_end", "seq_has_qual",
              "bases", "quals"):
        assert np.array_equal(got[k], ref[k]), k


def test_windows_from_reference_breaking_points_fragment_correction():
    lam = LambdaOverlaps("lambda_frag_overlaps.npz")
    ref = np.load(os.path.join(GOLD, "lambda_frag_windows.npz"))
    got = _build(lam, ref, len(lam.seq_off) - 1, True)
    assert len(got["win_type"]) == int(ref["total_windows"][0])
    nw = len(ref["win_type"])
    ns = int(ref["win_first"][nw])
    nb = int(ref["seq_off"][ns])
    assert np.array_equal(got["win_first"][:nw + 1], ref["win_first"])
    for k in ("seq_begin", "seq_end", "seq_has_qual"):
        assert np.array_equal(got[k][:ns], ref[k]), k
    assert np.array_equal(got["seq_off"][:ns + 1], ref["seq_off"])
    assert np.array_equal(got["bases"][:nb], ref["bases"]) and np.array_equal(got["quals"][:nb], ref["quals"])


def test_fasta_record_format_reproduces_racon_stdout():
    """racon_b200::format_fasta on the reference's polished lambda contig + tags == racon's stdout (golden md5)."""
    import ctypes as C
    import hashlib
    from racon_b200 import api
    lib = api.load()
    ref = np.load(os.path.join(GOLD, "lambda_windows.npz"))
    full = ref["polished_name"].tobytes()
    cut = full.index(b" LN:i:")
    name, tags, data = full[:cut], full[cut:], ref["polished"].tobytes()
    n = lib.rp_mirror_format_fasta(name, tags, data, len(data), None, 0)
    buf = C.create_string_buffer(n)
    assert lib.rp_mirror_format_fasta(name, tags, data, len(data), buf, n) == n
    assert hashlib.md5(buf.raw[:n]).hexdigest() == "b0e2a2788440a4982e544e2e9b3bf378"
