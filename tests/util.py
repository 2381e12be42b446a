"""Shared test helpers: random window makers (numpy RNG; test-only) and checker access."""
import atexit
import os
import shutil
import struct
import tempfile
import zlib

import numpy as np

from racon_b200 import windows

BASES = b"ACGT"
GOLDEN_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "data")
_sample_dir = []


def sample_data_dir():
    """The reference's lambda-phage sample files (tests/golden/data) as a directory of whole files.  No stored file exceeds
    1 MB, so the larger ones are kept as NAME.part0, NAME.part1 ...: they are joined here, into a temporary directory that
    is removed when the process exits."""
    if not _sample_dir:
        d = tempfile.mkdtemp(prefix="racon_b200_samples_")
        atexit.register(shutil.rmtree, d, True)
        for f in sorted(os.listdir(GOLDEN_DATA)):
            with open(os.path.join(GOLDEN_DATA, f), "rb") as src, open(os.path.join(d, f.rsplit(".part", 1)[0]), "ab") as dst:
                dst.write(src.read())
        _sample_dir.append(d)
    return _sample_dir[0]


def ref_answers():
    """What the unmodified reference answered on the oracle tests' inputs (tests/golden/make_ref_answers.py)."""
    import json
    with open(os.path.join(os.path.dirname(GOLDEN_DATA), "ref_answers.json")) as f:
        return json.load(f)


def cigar_answer(res):
    """(CIGAR, edit distance) as stored: [CRC-32 of the CIGAR, edit distance]."""
    return [zlib.crc32(res[0].encode()), int(res[1])]


def consensus_answer(cons, polished):
    """Per window, as stored: [CRC-32 of the consensus, polished flag]."""
    return [[zlib.crc32(c), int(p)] for c, p in zip(cons, polished)]


def mutate(rng, t, err, alphabet=BASES):
    out = bytearray()
    p = err / 3.0
    for ch in t:
        while True:
            u = rng.random()
            if u < p:
                break
            if u < 2 * p:
                out.append(alphabet[rng.integers(len(alphabet))])
                continue
            if u < 3 * p:
                c = ch
                while c == ch:
                    c = alphabet[rng.integers(len(alphabet))]
                out.append(c)
                break
            out.append(ch)
            break
    return bytes(out)


def rand_qual(rng, n, lo=5, hi=40):
    return bytes((rng.integers(lo, hi + 1, size=n) + 33).astype(np.uint8))


def make_window(rng, wlen=500, depth=32, err=0.12, partial_frac=0.0, with_qual=False, backbone_qual=False,
                alphabet=BASES, min_piece=20):
    """One window as [(bases, quals|None, begin, end), ...]; layers may be partial-span."""
    truth = bytes(alphabet[i] for i in rng.integers(len(alphabet), size=wlen))
    bb = mutate(rng, truth, err, alphabet)[:wlen] or truth[:1]
    win = [(bb, rand_qual(rng, len(bb)) if backbone_qual else None, 0, 0)]
    bl = len(bb)
    for _ in range(depth):
        if bl >= 2 * min_piece and rng.random() < partial_frac:
            b = int(rng.integers(0, bl - min_piece))
            e = int(rng.integers(b + min_piece - 1, bl))
            if rng.random() < 0.5:
                b = 0 if rng.random() < 0.5 else b
                e = bl - 1 if b != 0 else e
        else:
            b, e = 0, bl - 1
        if e <= b:
            continue
        piece = mutate(rng, bb[b:e + 1], err, alphabet)
        if not piece:
            continue
        win.append((piece, rand_qual(rng, len(piece)) if with_qual else None, b, e))
    return win


def make_set(seed, n, types=None, **kw):
    rng = np.random.default_rng(seed)
    wins = [make_window(rng, **kw) for _ in range(n)]
    return windows.from_lists(wins, types)


def window_crcs(r):
    """one CRC-32 per window over its sequences: bases, qualities (where present), begin, end — same function on the
    reference's window arrays and on MirrorPolisher.export()"""
    out = []
    for w in range(len(r["win_first"]) - 1):
        c = zlib.crc32(bytes([int(r["win_type"][w])]))
        for s in range(int(r["win_first"][w]), int(r["win_first"][w + 1])):
            a, b = int(r["seq_off"][s]), int(r["seq_off"][s + 1])
            c = zlib.crc32(r["bases"][a:b].tobytes(), c)
            if r["seq_has_qual"][s]:
                c = zlib.crc32(r["quals"][a:b].tobytes(), c)
            c = zlib.crc32(struct.pack("<II", int(r["seq_begin"][s]), int(r["seq_end"][s])), c)
        out.append(c)
    return np.asarray(out, np.uint32)
