"""ctypes binding of the C ABI (include/racon_b200.h) — used by tests/, bench.py and __graft_entry__.py.

The product is libracon_b200.so (C ABI + sm_90a kernels + C++ host mirror); this module only calls it.
Loading fails loudly when the library is missing; creating a batch fails loudly without a CUDA device.
"""
import ctypes as C
import os

import numpy as np

from . import build

_lib = None

RP_OK = 0
RP_BATCH_FULL = 1


class RaconB200Error(RuntimeError):
    pass


def lib_path():
    return os.environ.get("RACON_B200_LIB") or os.path.join(build.LIBDIR, "libracon_b200.so")


def load(build_if_missing=True):
    """Loads libracon_b200.so (building it in-tree first if the sources are newer)."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if build_if_missing and not os.environ.get("RACON_B200_LIB"):
        try:
            path = build.build_cuda()
        except Exception:
            if not os.path.exists(path):
                raise
    if not os.path.exists(path):
        raise RaconB200Error("libracon_b200.so is missing: run __graft_entry__.build() (no CPU fallback exists)")
    lib = C.CDLL(path)
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    lib.rp_strerror.restype = C.c_char_p
    lib.rp_strerror.argtypes = [C.c_int32]
    lib.rp_last_error.restype = C.c_char_p
    lib.rp_version.restype = C.c_char_p
    lib.rp_device_count.restype = C.c_int
    lib.rp_poa_create.restype = C.c_int32
    lib.rp_poa_create.argtypes = [C.POINTER(vp), C.c_int, C.c_size_t, C.c_int8, C.c_int8, C.c_int8, C.c_int, u32, u32]
    lib.rp_poa_destroy.restype = None
    lib.rp_poa_destroy.argtypes = [vp]
    lib.rp_poa_add_window.restype = C.c_int32
    lib.rp_poa_add_window.argtypes = [vp, u32, vp, vp, vp, vp, vp, C.c_int, C.c_int]
    lib.rp_poa_add_window_set.restype = C.c_int32
    lib.rp_poa_add_window_set.argtypes = [vp, u32, u32, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp]
    lib.rp_poa_size.restype = u32
    lib.rp_poa_size.argtypes = [vp]
    for name in ("rp_poa_run", "rp_poa_sync", "rp_poa_upload", "rp_poa_launch", "rp_poa_download", "rp_poa_reset"):
        getattr(lib, name).restype = C.c_int32
        getattr(lib, name).argtypes = [vp]
    lib.rp_poa_fetch.restype = C.c_int32
    lib.rp_poa_fetch.argtypes = [vp, u32, vp, vp, vp, vp]
    lib.rp_poa_window_status.restype = C.c_int32
    lib.rp_poa_window_status.argtypes = [vp, u32, vp]
    lib.rp_poa_fetch_all.restype = C.c_int32
    lib.rp_poa_fetch_all.argtypes = [vp, vp, u32, vp, vp, vp]
    lib.rp_poa_set_stream.restype = C.c_int32
    lib.rp_poa_set_stream.argtypes = [vp, vp]
    lib.rp_poa_info.restype = C.c_int32
    lib.rp_poa_info.argtypes = [vp, vp]
    lib.rp_poa_enable_counters.restype = C.c_int32
    lib.rp_poa_enable_counters.argtypes = [vp, C.c_int]
    lib.rp_poa_band_info.restype = C.c_int32
    lib.rp_poa_band_info.argtypes = [vp, vp]
    _bind_aln(lib, C, vp, u32)
    # the C++ host layer and its hooks live in a library of their own (it links against the product, not vice versa)
    host_path = os.path.join(os.path.dirname(path), "libracon_b200_host.so")
    if os.path.exists(host_path):
        host = C.CDLL(host_path)
        for name in ("rp_mirror_align", "rp_mirror_consensus", "rp_mirror_polisher_open", "rp_mirror_polisher_open_with_bp",
                     "rp_mirror_polisher_counts", "rp_mirror_polisher_export", "rp_mirror_polisher_polish",
                     "rp_mirror_polisher_window_consensus", "rp_mirror_polisher_polished", "rp_mirror_polisher_close",
                     "rp_mirror_polisher_failed", "rp_mirror_format_fasta", "rp_mirror_polisher_stream_fasta",
                     "rp_mirror_input_open", "rp_mirror_input_counts", "rp_mirror_input_export",
                     "rp_mirror_input_cigar_breaking_points", "rp_mirror_input_close", "rp_mirror_polisher_open_files"):
            if hasattr(host, name):
                setattr(lib, name, getattr(host, name))
    if hasattr(lib, "rp_mirror_align"):
        lib.rp_mirror_align.restype = C.c_int
        lib.rp_mirror_align.argtypes = [u32, vp, vp, vp, vp, vp, u32, u32, vp, u32]
    if hasattr(lib, "rp_mirror_consensus"):
        lib.rp_mirror_consensus.restype = C.c_double
        lib.rp_mirror_consensus.argtypes = [u32] + [vp] * 8 + [C.c_int8, C.c_int8, C.c_int8, u32, C.c_int, u32, vp,
                                                               u32, vp, vp]
    _lib = lib
    return lib


def _bind_aln(lib, C, vp, u32):
    lib.rp_aln_create.restype = C.c_int32
    lib.rp_aln_create.argtypes = [C.POINTER(vp), C.c_int, C.c_size_t, u32]
    lib.rp_aln_destroy.restype = None
    lib.rp_aln_destroy.argtypes = [vp]
    lib.rp_aln_add.restype = C.c_int32
    lib.rp_aln_add.argtypes = [vp, C.c_char_p, u32, C.c_char_p, u32]
    lib.rp_aln_set_window_length.restype = C.c_int32
    lib.rp_aln_set_window_length.argtypes = [vp, u32]
    lib.rp_aln_add_overlap.restype = C.c_int32
    lib.rp_aln_add_overlap.argtypes = [vp, C.c_char_p, u32, C.c_char_p, u32, u32, u32]
    lib.rp_aln_fetch_breaking_points.restype = C.c_int32
    lib.rp_aln_fetch_breaking_points.argtypes = [vp, u32, vp, vp]
    lib.rp_aln_size.restype = u32
    lib.rp_aln_size.argtypes = [vp]
    for name in ("rp_aln_run", "rp_aln_sync", "rp_aln_upload", "rp_aln_launch", "rp_aln_download", "rp_aln_reset"):
        getattr(lib, name).restype = C.c_int32
        getattr(lib, name).argtypes = [vp]
    lib.rp_aln_fetch_cigar.restype = C.c_int32
    lib.rp_aln_fetch_cigar.argtypes = [vp, u32, vp, vp, vp, vp]
    lib.rp_aln_set_stream.restype = C.c_int32
    lib.rp_aln_set_stream.argtypes = [vp, vp]
    lib.rp_aln_info.restype = C.c_int32
    lib.rp_aln_info.argtypes = [vp, vp]


def _check(lib, st, what):
    if st < 0:
        raise RaconB200Error("%s: %s (%s)" % (what, lib.rp_strerror(st).decode(), lib.rp_last_error().decode()))
    return st


def _ptr(a):
    return None if a is None else a.ctypes.data


class ReadStore:
    """Device-resident sequences (rp_reads): uploaded once; windows then name their layers as slices of them
    (PoaBatch.add_window_refs).  sequences: list of bytes; qualities: list of bytes / None (or None for no qualities)."""

    def __init__(self, sequences, qualities=None, device=0):
        self.lib = load()
        n = len(sequences)
        self._keep = (list(sequences), list(qualities) if qualities is not None else None)
        sp = (C.c_char_p * n)(*sequences)
        qp = None
        if qualities is not None:
            qp = (C.c_char_p * n)(*[q if q else None for q in qualities])
        ln = (C.c_uint32 * n)(*[len(x) for x in sequences])
        self._arrays = (sp, qp, ln)
        self.h = C.c_void_p()
        f = self.lib.rp_reads_create
        f.restype = C.c_int32
        f.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        _check(self.lib, f(C.byref(self.h), device, n, sp, qp, ln), "rp_reads_create")

    @classmethod
    def from_flat(cls, bases, seq_off, quals=None, seq_has_qual=None, device=0):
        """Store over flat arrays (numpy uint8 bases / quals, uint64 offsets): sequence i = bases[seq_off[i]:seq_off[i+1]]."""
        self = cls.__new__(cls)
        self.lib = load()
        n = len(seq_off) - 1
        base = bases.ctypes.data
        off = np.asarray(seq_off, dtype=np.uint64)
        ptrs = np.ascontiguousarray(off[:-1] + np.uint64(base))
        qptrs = None
        if quals is not None and seq_has_qual is not None and np.any(seq_has_qual):
            qptrs = np.ascontiguousarray(np.where(np.asarray(seq_has_qual) != 0, off[:-1] + np.uint64(quals.ctypes.data),
                                                  np.uint64(0)).astype(np.uint64))
        ln = np.ascontiguousarray(np.diff(off).astype(np.uint32))
        self._keep = (bases, quals, ptrs, qptrs, ln)
        self._arrays = None
        self.h = C.c_void_p()
        f = self.lib.rp_reads_create
        f.restype = C.c_int32
        f.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        _check(self.lib, f(C.byref(self.h), device, n, _ptr(ptrs), _ptr(qptrs), _ptr(ln)), "rp_reads_create")
        return self

    def device_bytes(self):
        self.lib.rp_reads_bytes.restype = C.c_uint64
        self.lib.rp_reads_bytes.argtypes = [C.c_void_p]
        return int(self.lib.rp_reads_bytes(self.h))

    def close(self):
        if self.h:
            self.lib.rp_reads_destroy.restype = None
            self.lib.rp_reads_destroy.argtypes = [C.c_void_p]
            self.lib.rp_reads_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PoaBatch:
    """racon::CUDABatchProcessor-shaped batch object (add windows -> run -> fetch)."""

    def __init__(self, device=0, mem_bytes=0, match=3, mismatch=-5, gap=-4, banded=False, window_length=500,
                 max_depth=0):
        self.lib = load()
        self.h = C.c_void_p()
        _check(self.lib, self.lib.rp_poa_create(C.byref(self.h), device, mem_bytes, match, mismatch, gap,
                                                1 if banded else 0, window_length, max_depth), "rp_poa_create")

    def close(self):
        if self.h:
            self.lib.rp_poa_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add_window_set(self, ws, first=0, count=None, trim=True):
        """Adds windows [first, first+count) of a WindowSet; returns how many fit."""
        if count is None:
            count = ws.n_windows - first
        added = C.c_uint32(0)
        st = self.lib.rp_poa_add_window_set(self.h, first, count, _ptr(ws.bases), _ptr(ws.quals), _ptr(ws.seq_off),
                                            _ptr(ws.seq_has_qual), _ptr(ws.seq_begin), _ptr(ws.seq_end),
                                            _ptr(ws.win_first), _ptr(ws.win_type), 1 if trim else 0, C.byref(added))
        _check(self.lib, st, "rp_poa_add_window_set")
        return added.value

    def add_window(self, seqs, window_type=1, trim=True):
        """seqs: [(bases, quals|None, begin, end), ...], backbone first.  Returns RP_OK or RP_BATCH_FULL."""
        n = len(seqs)
        keep = []
        sp = (C.c_char_p * n)()
        qp = (C.c_char_p * n)()
        ln = (C.c_uint32 * n)()
        bg = (C.c_uint32 * n)()
        en = (C.c_uint32 * n)()
        for i, (b, q, s, e) in enumerate(seqs):
            keep.append((b, q))
            sp[i] = b
            qp[i] = q
            ln[i] = len(b)
            bg[i] = s
            en[i] = e
        st = self.lib.rp_poa_add_window(self.h, n, sp, ln, qp, bg, en, window_type, 1 if trim else 0)
        return _check(self.lib, st, "rp_poa_add_window")

    def add_window_refs(self, store, pieces, window_type=1, trim=True):
        """pieces: [(sequence id in `store`, offset, length, reverse, begin, end), ...], backbone first — the window's
        layers named as slices of a device-resident ReadStore.  Returns RP_OK or RP_BATCH_FULL."""
        a = np.ascontiguousarray(np.asarray(pieces, dtype=np.int64).reshape(-1, 6))
        cols = [np.ascontiguousarray(a[:, k].astype(np.uint32)) for k in (0, 1, 2)]
        rev = np.ascontiguousarray(a[:, 3].astype(np.uint8))
        bg, en = (np.ascontiguousarray(a[:, k].astype(np.uint32)) for k in (4, 5))
        f = self.lib.rp_poa_add_window_refs
        f.restype = C.c_int32
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_void_p] * 6 + [C.c_int, C.c_int]
        st = f(self.h, store.h, len(a), _ptr(cols[0]), _ptr(cols[1]), _ptr(cols[2]), _ptr(rev), _ptr(bg), _ptr(en),
               window_type, 1 if trim else 0)
        return _check(self.lib, st, "rp_poa_add_window_refs")

    def add_window_set_refs(self, store, refs, first=0, count=None, trim=True):
        """Bulk add_window_refs.  refs: dict of flat arrays seq_id, offset, length, reverse (uint8), begin, end (one entry
        per piece) + win_first (windows + 1) and optionally win_type.  Returns how many windows fit."""
        if count is None:
            count = len(refs["win_first"]) - 1 - first
        f = self.lib.rp_poa_add_window_set_refs
        f.restype = C.c_int32
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 8 + [C.c_int, C.c_void_p]
        added = C.c_uint32(0)
        st = f(self.h, store.h, first, count, _ptr(refs["seq_id"]), _ptr(refs["offset"]), _ptr(refs["length"]),
               _ptr(refs.get("reverse")), _ptr(refs["begin"]), _ptr(refs["end"]), _ptr(refs["win_first"]),
               _ptr(refs.get("win_type")), 1 if trim else 0, C.byref(added))
        _check(self.lib, st, "rp_poa_add_window_set_refs")
        return added.value

    def size(self):
        return self.lib.rp_poa_size(self.h)

    def set_stream(self, cuda_stream):
        _check(self.lib, self.lib.rp_poa_set_stream(self.h, C.c_void_p(cuda_stream)), "rp_poa_set_stream")

    def upload(self):
        _check(self.lib, self.lib.rp_poa_upload(self.h), "rp_poa_upload")

    def launch(self):
        _check(self.lib, self.lib.rp_poa_launch(self.h), "rp_poa_launch")

    def download(self):
        _check(self.lib, self.lib.rp_poa_download(self.h), "rp_poa_download")

    def run(self):
        _check(self.lib, self.lib.rp_poa_run(self.h), "rp_poa_run")

    def sync(self):
        _check(self.lib, self.lib.rp_poa_sync(self.h), "rp_poa_sync")

    def reset(self):
        _check(self.lib, self.lib.rp_poa_reset(self.h), "rp_poa_reset")

    def enable_counters(self, on=True):
        _check(self.lib, self.lib.rp_poa_enable_counters(self.h, 1 if on else 0), "rp_poa_enable_counters")

    def info(self):
        a = (C.c_uint64 * 8)()
        _check(self.lib, self.lib.rp_poa_info(self.h, a), "rp_poa_info")
        keys = ["launches", "h2d_bytes", "d2h_bytes", "workers", "scratch_bytes_per_worker", "alignments",
                "dp_cells", "pred_cells"]
        return dict(zip(keys, [int(v) for v in a]))

    def band_info(self):
        """racon -b bookkeeping of the last run: alignments tried inside the band / redone with the full matrix."""
        a = (C.c_uint64 * 8)()
        _check(self.lib, self.lib.rp_poa_band_info(self.h, a), "rp_poa_band_info")
        return {"banded": bool(a[0]), "band_alignments": int(a[1]), "band_redone_full": int(a[2]),
                "band_width": int(a[3]), "band_audit_mismatches": int(a[4]), "band_layout_in_use": bool(a[5])}

    def fetch_all(self, stride):
        n = self.size()
        out = np.zeros((n, stride), dtype=np.uint8)
        lens = np.zeros(n, dtype=np.uint32)
        pol = np.zeros(n, dtype=np.uint8)
        st = np.zeros(n, dtype=np.uint32)
        _check(self.lib, self.lib.rp_poa_fetch_all(self.h, out.ctypes.data, stride, lens.ctypes.data,
                                                   pol.ctypes.data, st.ctypes.data), "rp_poa_fetch_all")
        return out, lens, pol.astype(bool), st

    def fetch(self, i):
        c = C.c_char_p()
        l = C.c_uint32()
        cov = C.POINTER(C.c_uint16)()
        pol = C.c_int()
        _check(self.lib, self.lib.rp_poa_fetch(self.h, i, C.byref(c), C.byref(l), C.byref(cov), C.byref(pol)),
               "rp_poa_fetch")
        cons = C.string_at(c, l.value) if l.value else b""
        coverage = np.ctypeslib.as_array(cov, shape=(l.value,)).copy() if (l.value and cov) else np.zeros(0, np.uint16)
        return cons, coverage, bool(pol.value)


class AlnBatch:
    """racon::CUDABatchAligner's shape (src/cuda/cudaaligner.hpp:21-92) over the rp_aln_* C ABI."""

    def __init__(self, device=0, mem_bytes=0, max_len=0):
        self.lib = load()
        self.h = C.c_void_p()
        _check(self.lib, self.lib.rp_aln_create(C.byref(self.h), device, mem_bytes, max_len), "rp_aln_create")

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.lib.rp_aln_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_window_length(self, window_length):
        _check(self.lib, self.lib.rp_aln_set_window_length(self.h, window_length), "rp_aln_set_window_length")

    def fetch_breaking_points(self, i):
        """(n, 2) uint32 (t, q) points of overlap i, as Overlap::breaking_points_ (overlap.cpp:226-292)."""
        p = C.c_void_p()
        n = C.c_uint32()
        _check(self.lib, self.lib.rp_aln_fetch_breaking_points(self.h, i, C.byref(p), C.byref(n)),
               "rp_aln_fetch_breaking_points")
        if n.value == 0:
            return np.zeros((0, 2), np.uint32)
        a = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint32)), shape=(n.value * 2,))
        return a.reshape(n.value, 2).copy()

    def add(self, query, target, t_begin=0, q_start=0):
        """addOverlap: True if taken, False if the batch is full (cudaaligner.cpp:51-78)."""
        st = self.lib.rp_aln_add_overlap(self.h, query, len(query), target, len(target), t_begin, q_start)
        if st == 1:
            return False
        _check(self.lib, st, "rp_aln_add")
        return True

    def add_ref(self, store, q_id, q_start, q_len, q_reverse, t_id, t_begin, t_len):
        """The overlap named as slices of a device-resident ReadStore (rp_aln_add_overlap_ref): query = q_len bases of
        sequence q_id from q_start on (of its reverse complement when q_reverse), target = t_len bases of t_id from
        t_begin on.  False = batch full (like add)."""
        f = self.lib.rp_aln_add_overlap_ref
        f.restype = C.c_int32
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_uint32,
                      C.c_uint32]
        return _check(self.lib, f(self.h, store.h, q_id, q_start, q_len, 1 if q_reverse else 0, t_id, t_begin, t_len),
                      "rp_aln_add_overlap_ref") == RP_OK

    def size(self):
        return self.lib.rp_aln_size(self.h)

    def set_stream(self, cuda_stream):
        _check(self.lib, self.lib.rp_aln_set_stream(self.h, C.c_void_p(cuda_stream)), "rp_aln_set_stream")

    def upload(self):
        _check(self.lib, self.lib.rp_aln_upload(self.h), "rp_aln_upload")

    def launch(self):
        _check(self.lib, self.lib.rp_aln_launch(self.h), "rp_aln_launch")

    def download(self):
        _check(self.lib, self.lib.rp_aln_download(self.h), "rp_aln_download")

    def run(self):
        _check(self.lib, self.lib.rp_aln_run(self.h), "rp_aln_run")

    def sync(self):
        _check(self.lib, self.lib.rp_aln_sync(self.h), "rp_aln_sync")

    def reset(self):
        _check(self.lib, self.lib.rp_aln_reset(self.h), "rp_aln_reset")

    def info(self):
        a = (C.c_uint64 * 8)()
        _check(self.lib, self.lib.rp_aln_info(self.h, a), "rp_aln_info")
        return {"launches": a[0], "h2d_bytes": a[1], "d2h_bytes": a[2], "workers": a[3], "scratch_per_warp": a[4]}

    def fetch(self, i):
        """(cigar bytes, edit distance, status) of overlap i."""
        p = C.c_char_p()
        n = C.c_uint32()
        d = C.c_int32()
        st = C.c_uint32()
        _check(self.lib, self.lib.rp_aln_fetch_cigar(self.h, i, C.byref(p), C.byref(n), C.byref(d), C.byref(st)),
               "rp_aln_fetch_cigar")
        return (p.value or b"")[: n.value], d.value, st.value


def align(pairs, device=0, max_len=0):
    """CIGARs for [(query, target), ...] as Overlap::align_overlaps would get them from edlib (overlap.cpp:205-224)."""
    b = AlnBatch(device=device, max_len=max_len)
    out = []
    try:
        i = 0
        while i < len(pairs):
            b.reset()
            first = i
            while i < len(pairs) and b.add(*pairs[i]):
                i += 1
            if i == first:
                raise RaconB200Error("pair %d does not fit an empty batch" % i)
            b.run()
            b.sync()
            out.extend(b.fetch(k) for k in range(i - first))
    finally:
        b.close()
    return out


def mirror_align(pairs, max_alignments=0, device=0):
    """CIGARs through the C++ mirror of CUDABatchAligner (host_mirror.hpp), driven like
    CUDAPolisher::find_overlap_breaking_points drives the reference's batches (cudapolisher.cpp:100-213)."""
    lib = load()
    n = len(pairs)
    blob = b"".join(q + t for q, t in pairs)
    q_off = np.zeros(n, np.uint64)
    t_off = np.zeros(n, np.uint64)
    q_len = np.array([len(q) for q, _ in pairs], np.uint32)
    t_len = np.array([len(t) for _, t in pairs], np.uint32)
    o = 0
    for i, (q, t) in enumerate(pairs):
        q_off[i] = o
        t_off[i] = o + len(q)
        o += len(q) + len(t)
    stride = int(max((len(q) + len(t)) for q, t in pairs) * 4 + 16) if n else 16
    out = np.zeros(max(n, 1) * stride, np.uint8)
    buf = np.frombuffer(blob if blob else b"\0", np.uint8)
    r = lib.rp_mirror_align(n, _ptr(buf), _ptr(q_off), _ptr(q_len), _ptr(t_off), _ptr(t_len), max_alignments, device,
                            _ptr(out), stride)
    if r != 0:
        raise RaconB200Error("rp_mirror_align failed: %d" % r)
    res = []
    for i in range(n):
        row = out[i * stride:(i + 1) * stride].tobytes()
        res.append(row[: row.index(b"\0")])
    return res


class MirrorPolisher:
    """Drives racon_b200::Polisher (host_mirror.hpp) through its test hooks: overlaps -> device alignment + breaking
    points -> windows -> device consensus -> stitched sequences.  Same call shape as oracle/ref_polisher_harness.cpp."""

    def __init__(self, bases, quals, seq_off, seq_has_qual, n_targets, overlaps, window_length=500,
                 quality_threshold=10.0, trim=True, match=3, mismatch=-5, gap=-4, window_type_tgs=True,
                 fragment_correction=False, device=0, breaking_points=None):
        """breaking_points=(bp_off, bp): skip the device alignment and build the windows from given breaking points
        (host logic only; no GPU needed, polish() is then not available)."""
        self.lib = load()
        L = self.lib
        vp = C.c_void_p
        L.rp_mirror_polisher_open.restype = vp
        L.rp_mirror_polisher_open.argtypes = [C.c_uint32, vp, vp, vp, vp, C.c_uint32, C.c_int, C.c_int, C.c_uint32, vp,
                                              C.c_uint32, C.c_double, C.c_int, C.c_int8, C.c_int8, C.c_int8, C.c_uint32]
        L.rp_mirror_polisher_counts.restype = None
        L.rp_mirror_polisher_counts.argtypes = [vp, vp]
        L.rp_mirror_polisher_export.restype = None
        L.rp_mirror_polisher_export.argtypes = [vp] * 11
        L.rp_mirror_polisher_polish.restype = C.c_uint32
        L.rp_mirror_polisher_polish.argtypes = [vp, C.c_int]
        L.rp_mirror_polisher_window_consensus.restype = C.c_uint32
        L.rp_mirror_polisher_window_consensus.argtypes = [vp, C.c_uint32, vp, C.c_uint32]
        L.rp_mirror_polisher_polished.restype = C.c_uint64
        L.rp_mirror_polisher_polished.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, vp, C.c_uint64]
        L.rp_mirror_polisher_close.restype = None
        L.rp_mirror_polisher_close.argtypes = [vp]
        # keep the sequence bytes alive: the windows point into them
        self._bases = np.ascontiguousarray(np.frombuffer(bases, np.uint8))
        self._quals = np.ascontiguousarray(np.frombuffer(quals, np.uint8))
        self._off = np.ascontiguousarray(seq_off, dtype=np.uint64)
        self._hq = np.ascontiguousarray(seq_has_qual, dtype=np.uint8)
        ov = np.ascontiguousarray(overlaps, dtype=np.uint32)
        if breaking_points is not None:
            L.rp_mirror_polisher_open_with_bp.restype = vp
            L.rp_mirror_polisher_open_with_bp.argtypes = [C.c_uint32, vp, vp, vp, vp, C.c_uint32, C.c_int, C.c_int,
                                                          C.c_uint32, vp, vp, vp, C.c_uint32, C.c_double]
            bp_off = np.ascontiguousarray(breaking_points[0], dtype=np.uint64)
            bp = np.ascontiguousarray(breaking_points[1], dtype=np.uint32)
            self.h = L.rp_mirror_polisher_open_with_bp(len(self._off) - 1, _ptr(self._bases), _ptr(self._quals),
                                                       _ptr(self._off), _ptr(self._hq), n_targets,
                                                       1 if window_type_tgs else 0, 1 if fragment_correction else 0,
                                                       len(ov), _ptr(ov), _ptr(bp_off), _ptr(bp), window_length,
                                                       quality_threshold)
            return
        self.h = L.rp_mirror_polisher_open(len(self._off) - 1, _ptr(self._bases), _ptr(self._quals), _ptr(self._off),
                                           _ptr(self._hq), n_targets, 1 if window_type_tgs else 0,
                                           1 if fragment_correction else 0, len(ov), _ptr(ov), window_length,
                                           quality_threshold, 1 if trim else 0, match, mismatch, gap, device)

    @classmethod
    def from_files(cls, reads, overlaps, targets, fragment_correction=False, window_length=500, quality_threshold=10.0,
                   error_threshold=0.3, trim=True, match=3, mismatch=-5, gap=-4, device=0, resident_reads=False):
        """createPolisher + initialize on files (reads_io.hpp): parse, filter, align + breaking points on the device
        (SAM input keeps its own alignments and needs no device here), build the windows.  resident_reads: the sequences
        are uploaded once and the aligner (and later the consensus) name their inputs instead of copying them."""
        self = cls.__new__(cls)
        self.lib = load()
        L = self.lib
        vp = C.c_void_p
        L.rp_mirror_polisher_open_files.restype = vp
        L.rp_mirror_polisher_open_files.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.c_uint32, C.c_double,
                                                    C.c_double, C.c_int, C.c_int8, C.c_int8, C.c_int8, C.c_uint32, C.c_int,
                                                    vp, C.c_uint32]
        L.rp_mirror_polisher_counts.restype = None
        L.rp_mirror_polisher_counts.argtypes = [vp, vp]
        L.rp_mirror_polisher_export.restype = None
        L.rp_mirror_polisher_export.argtypes = [vp] * 11
        L.rp_mirror_polisher_polish.restype = C.c_uint32
        L.rp_mirror_polisher_polish.argtypes = [vp, C.c_int]
        L.rp_mirror_polisher_window_consensus.restype = C.c_uint32
        L.rp_mirror_polisher_window_consensus.argtypes = [vp, C.c_uint32, vp, C.c_uint32]
        L.rp_mirror_polisher_polished.restype = C.c_uint64
        L.rp_mirror_polisher_polished.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, vp, C.c_uint64]
        L.rp_mirror_polisher_close.restype = None
        L.rp_mirror_polisher_close.argtypes = [vp]
        err = C.create_string_buffer(1024)
        self.h = L.rp_mirror_polisher_open_files(os.fsencode(reads), os.fsencode(overlaps), os.fsencode(targets),
                                                 1 if fragment_correction else 0, window_length, quality_threshold,
                                                 error_threshold, 1 if trim else 0, match, mismatch, gap, device,
                                                 1 if resident_reads else 0, err, 1024)
        if not self.h:
            raise RuntimeError(err.value.decode(errors="replace"))
        return self

    def export(self):
        c = (C.c_uint64 * 3)()
        self.lib.rp_mirror_polisher_counts(self.h, c)
        nw, ns, nb = int(c[0]), int(c[1]), int(c[2])
        r = dict(bases=np.zeros(nb, np.uint8), quals=np.zeros(nb, np.uint8), seq_off=np.zeros(ns + 1, np.uint64),
                 seq_has_qual=np.zeros(ns, np.uint8), seq_begin=np.zeros(ns, np.uint32), seq_end=np.zeros(ns, np.uint32),
                 win_first=np.zeros(nw + 1, np.uint32), win_type=np.zeros(nw, np.uint8),
                 win_target=np.zeros(nw, np.uint64), win_rank=np.zeros(nw, np.uint32))
        self.lib.rp_mirror_polisher_export(self.h, *[_ptr(r[k]) for k in (
            "bases", "quals", "seq_off", "seq_has_qual", "seq_begin", "seq_end", "win_first", "win_type", "win_target",
            "win_rank")])
        return r

    def polish(self, drop_unpolished=False):
        n = self.lib.rp_mirror_polisher_polish(self.h, 1 if drop_unpolished else 0)
        c = (C.c_uint64 * 3)()
        self.lib.rp_mirror_polisher_counts(self.h, c)
        buf = C.create_string_buffer(1 << 20)
        cons = []
        for w in range(int(c[0])):
            k = self.lib.rp_mirror_polisher_window_consensus(self.h, w, buf, len(buf))
            cons.append(buf.raw[:k])
        out = []
        data = C.create_string_buffer(1 << 27)
        tags = C.create_string_buffer(4096)
        for i in range(n):
            tid = C.c_uint64()
            k = self.lib.rp_mirror_polisher_polished(self.h, i, C.byref(tid), tags, len(tags), data, len(data))
            out.append((tid.value, tags.value.decode(), data.raw[:k]))
        return cons, out

    def stream_fasta(self, path, names, drop_unpolished=False, mem_bytes=0, banded=False, resident_reads=False):
        """Polisher::polish_streaming into a FASTA file: two batch objects in flight, every polished sequence written the
        moment its last window is collected (polisher.cpp:504-537 + main.cpp:159-161).  names: target names by id
        (None: the names of the files a from_files() polisher was opened on).  resident_reads: every sequence is
        uploaded once and the windows are added by reference (layers extracted on the device)."""
        f = self.lib.rp_mirror_polisher_stream_fasta
        f.restype = C.c_uint32
        f.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.c_uint64, C.c_int, C.c_int]
        blob = None if names is None else b"".join(n.encode() + b"\0" for n in names) + b"\0"
        return f(self.h, 1 if drop_unpolished else 0, os.fsencode(path), blob, mem_bytes, 1 if banded else 0,
                 1 if resident_reads else 0)

    def failed(self):
        """(overlaps, windows) the device could not finish (see host_mirror.hpp: Polisher::failed_overlaps/windows)."""
        a = (C.c_uint64 * 2)()
        self.lib.rp_mirror_polisher_failed.restype = None
        self.lib.rp_mirror_polisher_failed.argtypes = [C.c_void_p, C.c_void_p]
        self.lib.rp_mirror_polisher_failed(self.h, a)
        return int(a[0]), int(a[1])

    def close(self):
        if self.h:
            self.lib.rp_mirror_polisher_close(self.h)
            self.h = None


def consensus(ws, match=3, mismatch=-5, gap=-4, trim=True, window_length=500, device=0, want_coverage=False,
              mem_bytes=0, banded=False, band_stats=None):
    """Convenience: whole WindowSet through PoaBatch (multiple batches if needed).
    Returns (consensus list, polished bool array, status uint32 array[, coverages]).
    band_stats: optional dict that receives the summed rp_poa_band_info counters."""
    batch = PoaBatch(device=device, mem_bytes=mem_bytes, match=match, mismatch=mismatch, gap=gap,
                     window_length=window_length, banded=banded)
    n = ws.n_windows
    lens_in = np.diff(ws.seq_off.astype(np.int64))
    stride = int(2 * (lens_in.max() if len(lens_in) else 1) + 64)
    cons, pol, st, covs = [], [], [], []
    first = 0
    try:
        while first < n:
            batch.reset()
            took = batch.add_window_set(ws, first, n - first, trim=trim)
            if took == 0:
                raise RaconB200Error("window %d does not fit an empty batch" % first)
            batch.run()
            batch.sync()
            out, lens, p, s = batch.fetch_all(stride)
            if band_stats is not None:
                for k, v in batch.band_info().items():
                    band_stats[k] = v if k in ("banded", "band_width", "band_layout_in_use") else band_stats.get(k, 0) + v
                band_stats["batches"] = band_stats.get("batches", 0) + 1
            for i in range(took):
                cons.append(out[i, :lens[i]].tobytes())
                if want_coverage:
                    covs.append(batch.fetch(i)[1])
            pol.append(p)
            st.append(s)
            first += took
    finally:
        batch.close()
    pol = np.concatenate(pol) if pol else np.zeros(0, bool)
    st = np.concatenate(st) if st else np.zeros(0, np.uint32)
    if want_coverage:
        return cons, pol, st, covs
    return cons, pol, st


def mirror_consensus(ws, match=3, mismatch=-5, gap=-4, trim=True, window_length=500, device=0):
    """Drives the C++ host mirror (createWindow/add_layer/BatchProcessor) through its test hook."""
    lib = load()
    n = ws.n_windows
    lens_in = np.diff(ws.seq_off.astype(np.int64))
    stride = int(2 * (lens_in.max() if len(lens_in) else 1) + 64)
    out = np.zeros((n, stride), dtype=np.uint8)
    lens = np.zeros(n, dtype=np.uint32)
    pol = np.zeros(n, dtype=np.uint8)
    r = lib.rp_mirror_consensus(n, _ptr(ws.bases), _ptr(ws.quals), _ptr(ws.seq_off), _ptr(ws.seq_has_qual),
                                _ptr(ws.seq_begin), _ptr(ws.seq_end), _ptr(ws.win_first), _ptr(ws.win_type), match,
                                mismatch, gap, window_length, 1 if trim else 0, device, out.ctypes.data, stride,
                                lens.ctypes.data, pol.ctypes.data)
    if r < 0:
        raise RaconB200Error("rp_mirror_consensus failed (%r)" % r)
    return [out[w, :lens[w]].tobytes() for w in range(n)], pol.astype(bool)


class InputFiles:
    """The input layer of the C++ host layer (reads_io.hpp): sequence + overlap files -> what racon::Polisher::initialize
    holds before it looks for breaking points — targets first, then the reads that are not a target; overlaps turned into
    indices and filtered (racon -e, one overlap per read unless -f)."""

    def __init__(self, reads, overlaps, targets, fragment_correction=False, error_threshold=0.3):
        self.lib = load()
        L = self.lib
        vp = C.c_void_p
        L.rp_mirror_input_open.restype = vp
        L.rp_mirror_input_open.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.c_double, vp, C.c_uint32]
        L.rp_mirror_input_counts.restype = None
        L.rp_mirror_input_counts.argtypes = [vp, vp]
        L.rp_mirror_input_export.restype = None
        L.rp_mirror_input_export.argtypes = [vp] * 8
        L.rp_mirror_input_cigar_breaking_points.restype = C.c_uint32
        L.rp_mirror_input_cigar_breaking_points.argtypes = [vp, C.c_uint32, C.c_uint32, vp, C.c_uint32]
        L.rp_mirror_input_close.restype = None
        L.rp_mirror_input_close.argtypes = [vp]
        err = C.create_string_buffer(1024)
        self.h = L.rp_mirror_input_open(os.fsencode(reads), os.fsencode(overlaps), os.fsencode(targets),
                                        1 if fragment_correction else 0, float(error_threshold), err, 1024)
        if not self.h:
            raise RuntimeError(err.value.decode(errors="replace"))
        c = (C.c_uint64 * 7)()
        L.rp_mirror_input_counts(self.h, c)
        ns, self.n_targets, nb, no = int(c[0]), int(c[1]), int(c[2]), int(c[3])
        self.window_type_tgs = bool(c[4])
        self.bases = np.zeros(nb, np.uint8)
        self.quals = np.zeros(nb, np.uint8)
        self.seq_off = np.zeros(ns + 1, np.uint64)
        self.seq_has_qual = np.zeros(ns, np.uint8)
        names = np.zeros(max(1, int(c[5])), np.uint8)
        self.overlaps = np.zeros((no, 9), np.uint32)
        cigars = np.zeros(max(1, int(c[6])), np.uint8)
        L.rp_mirror_input_export(self.h, _ptr(self.bases), _ptr(self.quals), _ptr(self.seq_off), _ptr(self.seq_has_qual),
                                 _ptr(names), _ptr(self.overlaps), _ptr(cigars))
        self.names = names.tobytes()[:int(c[5])].split(b"\0")[:ns]
        self.cigars = cigars.tobytes()[:int(c[6])].split(b"\0")[:no]

    def cigar_breaking_points(self, index, window_length=500):
        """(t, q) breaking points of an overlap that came with a CIGAR (SAM input), from the host layer"""
        n = self.lib.rp_mirror_input_cigar_breaking_points(self.h, index, window_length, None, 0)
        out = np.zeros((n, 2), np.uint32)
        self.lib.rp_mirror_input_cigar_breaking_points(self.h, index, window_length, _ptr(out), n)
        return out

    def close(self):
        if self.h:
            self.lib.rp_mirror_input_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def polish_files(reads, overlaps, targets, out_path, fragment_correction=False, window_length=500, quality_threshold=10.0,
                 error_threshold=0.3, trim=True, match=3, mismatch=-5, gap=-4, device=0, drop_unpolished=True,
                 mem_bytes=0, banded=False, resident_reads=True):
    """racon's whole run through the C++ host layer: files in, polished FASTA out (alignment, breaking points and
    consensus on the device).  Returns (records written, overlaps the device refused, windows the device refused)."""
    pol = MirrorPolisher.from_files(reads, overlaps, targets, fragment_correction=fragment_correction,
                                    window_length=window_length, quality_threshold=quality_threshold,
                                    error_threshold=error_threshold, trim=trim, match=match, mismatch=mismatch, gap=gap,
                                    device=device, resident_reads=resident_reads)
    try:
        n = pol.stream_fasta(out_path, None, drop_unpolished=drop_unpolished, mem_bytes=mem_bytes, banded=banded,
                             resident_reads=resident_reads)
        return (n,) + pol.failed()
    finally:
        pol.close()
