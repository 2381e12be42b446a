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
RP_NOT_READY = 2


class RaconB200Error(RuntimeError):
    pass


_vp, _u32, _u64, _int, _st = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_int32
_i8, _str, _size = C.c_int8, C.c_char_p, C.c_size_t

# name: (restype, argtypes) of every function of the C ABI (include/racon_b200.h)
SIGNATURES = {
    "rp_strerror": (_str, [_st]),
    "rp_last_error": (_str, []),
    "rp_device_count": (_int, []),
    "rp_device_memory": (_st, [_int, _vp, _vp]),
    "rp_version": (_str, []),
    "rp_poa_create": (_st, [C.POINTER(_vp), _int, _size, _i8, _i8, _i8, _int, _u32, _u32]),
    "rp_poa_destroy": (None, [_vp]),
    "rp_poa_add_window": (_st, [_vp, _u32, _vp, _vp, _vp, _vp, _vp, _int, _int]),
    "rp_reads_create": (_st, [C.POINTER(_vp), _int, _u32, _vp, _vp, _vp]),
    "rp_reads_destroy": (None, [_vp]),
    "rp_reads_bytes": (_u64, [_vp]),
    "rp_poa_add_window_refs": (_st, [_vp, _vp, _u32] + [_vp] * 6 + [_int, _int]),
    "rp_poa_add_window_set_refs": (_st, [_vp, _vp, _u32, _u32] + [_vp] * 8 + [_int, _vp]),
    "rp_poa_add_window_set": (_st, [_vp, _u32, _u32] + [_vp] * 8 + [_int, _vp]),
    "rp_poa_size": (_u32, [_vp]),
    "rp_poa_run": (_st, [_vp]),
    "rp_poa_sync": (_st, [_vp]),
    "rp_poa_query": (_st, [_vp]),
    "rp_poa_upload": (_st, [_vp]),
    "rp_poa_launch": (_st, [_vp]),
    "rp_poa_download": (_st, [_vp]),
    "rp_poa_fetch": (_st, [_vp, _u32, _vp, _vp, _vp, _vp]),
    "rp_poa_window_status": (_st, [_vp, _u32, _vp]),
    "rp_poa_fetch_all": (_st, [_vp, _vp, _u32, _vp, _vp, _vp]),
    "rp_poa_reset": (_st, [_vp]),
    "rp_poa_set_stream": (_st, [_vp, _vp]),
    "rp_poa_info": (_st, [_vp, _vp]),
    "rp_poa_enable_counters": (_st, [_vp, _int]),
    "rp_poa_band_info": (_st, [_vp, _vp]),
    "rp_aln_create": (_st, [C.POINTER(_vp), _int, _size, _u32]),
    "rp_aln_destroy": (None, [_vp]),
    "rp_aln_add": (_st, [_vp, _str, _u32, _str, _u32]),
    "rp_aln_set_window_length": (_st, [_vp, _u32]),
    "rp_aln_add_overlap": (_st, [_vp, _str, _u32, _str, _u32, _u32, _u32]),
    "rp_aln_add_overlap_ref": (_st, [_vp, _vp, _u32, _u32, _u32, _int, _u32, _u32, _u32]),
    "rp_aln_fetch_breaking_points": (_st, [_vp, _u32, _vp, _vp]),
    "rp_aln_size": (_u32, [_vp]),
    "rp_aln_run": (_st, [_vp]),
    "rp_aln_sync": (_st, [_vp]),
    "rp_aln_query": (_st, [_vp]),
    "rp_aln_upload": (_st, [_vp]),
    "rp_aln_launch": (_st, [_vp]),
    "rp_aln_download": (_st, [_vp]),
    "rp_aln_fetch_cigar": (_st, [_vp, _u32, _vp, _vp, _vp, _vp]),
    "rp_aln_reset": (_st, [_vp]),
    "rp_aln_set_stream": (_st, [_vp, _vp]),
    "rp_aln_info": (_st, [_vp, _vp]),
}

# the test hooks of the C++ host layer (libracon_b200_host.so, host_mirror.cpp / reads_io.cpp), bound when present
HOST_SIGNATURES = {
    "rp_mirror_align": (_int, [_u32, _vp, _vp, _vp, _vp, _vp, _u32, _u32, _vp, _u32]),
    "rp_mirror_consensus": (C.c_double, [_u32] + [_vp] * 8 + [_i8, _i8, _i8, _u32, _int, _u32, _vp, _u32, _vp, _vp]),
    "rp_mirror_polisher_open": (_vp, [_u32, _vp, _vp, _vp, _vp, _u32, _int, _int, _u32, _vp, _u32, C.c_double, _int,
                                      _i8, _i8, _i8, _vp, _u32]),
    "rp_mirror_polisher_open_with_bp": (_vp, [_u32, _vp, _vp, _vp, _vp, _u32, _int, _int, _u32, _vp, _vp, _vp, _u32,
                                              C.c_double]),
    "rp_mirror_polisher_open_files": (_vp, [_str, _str, _str, _int, _u32, C.c_double, C.c_double, _int, _i8, _i8, _i8,
                                            _vp, _u32, _int, _vp, _u32]),
    "rp_mirror_polisher_counts": (None, [_vp, _vp]),
    "rp_mirror_polisher_export": (None, [_vp] * 11),
    "rp_mirror_polisher_polish": (_u32, [_vp, _int]),
    "rp_mirror_polisher_window_consensus": (_u32, [_vp, _u32, _vp, _u32]),
    "rp_mirror_polisher_polished": (_u64, [_vp, _u32, _vp, _vp, _u32, _vp, _u64]),
    "rp_mirror_polisher_close": (None, [_vp]),
    "rp_mirror_polisher_failed": (None, [_vp, _vp]),
    "rp_mirror_polisher_breaking_points": (_u64, [_vp, _vp, _vp]),
    "rp_mirror_polisher_stream_fasta": (_u32, [_vp, _int, _str, _str, _u64, _int, _int]),
    "rp_mirror_polish_files_grouped": (_int, [_str, _str, _str, _int, _u32, C.c_double, C.c_double, _int, _i8, _i8, _i8,
                                              _vp, _u32, _int, _u64, _int, _u64, _int, _str, _vp, _vp, _u32]),
    "rp_mirror_last_grouped_run": (None, [_vp, _vp, _vp, _vp]),
    "rp_mirror_last_grouped_run_windows": (None, [_vp, _vp]),
    "rp_mirror_plan_read_groups": (C.c_int64, [_u64, _u32, _vp, _vp, _u64, _vp, _vp, _vp, _vp, _u32, _u64, _vp, _vp,
                                               _vp, _vp, _vp, _vp, _vp, _vp, _vp, _u32]),
    "rp_mirror_format_fasta": (_u64, [_str, _str, _str, _u64, _str, _u64]),
    "rp_mirror_stitch_order": (_u64, [_u32, _vp, _vp, _vp, _vp]),
    "rp_mirror_input_open": (_vp, [_str, _str, _str, _int, C.c_double, _vp, _u32]),
    "rp_mirror_input_counts": (None, [_vp, _vp]),
    "rp_mirror_input_export": (None, [_vp] * 8),
    "rp_mirror_input_cigar_breaking_points": (_u32, [_vp, _u32, _u32, _vp, _u32]),
    "rp_mirror_input_close": (None, [_vp]),
}


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
    for name, (restype, argtypes) in SIGNATURES.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = restype, argtypes
    # the C++ host layer and its hooks live in a library of their own (it links against the product, not vice versa)
    host_path = os.path.join(os.path.dirname(path), "libracon_b200_host.so")
    if os.path.exists(host_path):
        host = C.CDLL(host_path)
        for name, (restype, argtypes) in HOST_SIGNATURES.items():
            if hasattr(host, name):
                f = getattr(host, name)
                f.restype, f.argtypes = restype, argtypes
                setattr(lib, name, f)
    _lib = lib
    return lib


def _check(lib, st, what):
    if st < 0:
        raise RaconB200Error("%s: %s (%s)" % (what, lib.rp_strerror(st).decode(), lib.rp_last_error().decode()))
    return st


def _ptr(a):
    return None if a is None else a.ctypes.data


def device_count():
    """CUDA devices the library sees (rp_device_count; 0 without one): device=range(device_count()) uses them all."""
    return max(0, int(load().rp_device_count()))


def _device_list(device):
    """device: one CUDA device index or a sequence of them, one lane each (an index may repeat: [0, 0] = two lanes on
    GPU 0) -> the uint32 array the host layer takes.  Raises RaconB200Error on an empty list or an index that no visible
    device has; without any device nothing can be checked here and the first device call fails instead ("no CUDA
    device", as for a single index)."""
    devices = [device] if isinstance(device, (int, np.integer)) else list(device)
    if not devices:
        raise RaconB200Error("empty device list")
    n = device_count()
    for d in devices:
        if isinstance(d, bool) or not isinstance(d, (int, np.integer)):
            raise RaconB200Error("device index %r is not an integer" % (d,))
        if d < 0 or (n > 0 and d >= n):
            raise RaconB200Error("device index %d out of range: %d CUDA device(s) visible" % (d, n))
    return np.ascontiguousarray(devices, dtype=np.uint32)


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
        _check(self.lib, self.lib.rp_reads_create(C.byref(self.h), device, n, sp, qp, ln), "rp_reads_create")

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
        _check(self.lib, self.lib.rp_reads_create(C.byref(self.h), device, n, _ptr(ptrs), _ptr(qptrs), _ptr(ln)),
               "rp_reads_create")
        return self

    def device_bytes(self):
        return int(self.lib.rp_reads_bytes(self.h))

    def close(self):
        if self.h:
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
        st = self.lib.rp_poa_add_window_refs(self.h, store.h, len(a), _ptr(cols[0]), _ptr(cols[1]), _ptr(cols[2]),
                                             _ptr(rev), _ptr(bg), _ptr(en), window_type, 1 if trim else 0)
        return _check(self.lib, st, "rp_poa_add_window_refs")

    def add_window_set_refs(self, store, refs, first=0, count=None, trim=True):
        """Bulk add_window_refs.  refs: dict of flat arrays seq_id, offset, length, reverse (uint8), begin, end (one entry
        per piece) + win_first (windows + 1) and optionally win_type.  Returns how many windows fit."""
        if count is None:
            count = len(refs["win_first"]) - 1 - first
        added = C.c_uint32(0)
        st = self.lib.rp_poa_add_window_set_refs(
            self.h, store.h, first, count, _ptr(refs["seq_id"]), _ptr(refs["offset"]), _ptr(refs["length"]),
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

    def ready(self):
        """True when the last run has finished, False while it is in flight (rp_poa_query; never blocks)."""
        return _check(self.lib, self.lib.rp_poa_query(self.h), "rp_poa_query") == RP_OK

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
        st = self.lib.rp_aln_add_overlap_ref(self.h, store.h, q_id, q_start, q_len, 1 if q_reverse else 0, t_id, t_begin,
                                             t_len)
        return _check(self.lib, st, "rp_aln_add_overlap_ref") == RP_OK

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

    def ready(self):
        """True when the last run has finished, False while it is in flight (rp_aln_query; never blocks)."""
        return _check(self.lib, self.lib.rp_aln_query(self.h), "rp_aln_query") == RP_OK

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
        """device: a CUDA device index or a sequence of them (one lane each, see host_mirror.hpp's Polisher; an index may
        repeat).  breaking_points=(bp_off, bp): skip the device alignment and build the windows from given breaking
        points (host logic only; no GPU needed, `device` is not used and polish() is then not available)."""
        self.lib = load()
        L = self.lib
        # keep the sequence bytes alive: the windows point into them
        self._bases = np.ascontiguousarray(np.frombuffer(bases, np.uint8))
        self._quals = np.ascontiguousarray(np.frombuffer(quals, np.uint8))
        self._off = np.ascontiguousarray(seq_off, dtype=np.uint64)
        self._hq = np.ascontiguousarray(seq_has_qual, dtype=np.uint8)
        ov = np.ascontiguousarray(overlaps, dtype=np.uint32)
        self._n_overlaps = len(ov)
        if breaking_points is not None:
            bp_off = np.ascontiguousarray(breaking_points[0], dtype=np.uint64)
            bp = np.ascontiguousarray(breaking_points[1], dtype=np.uint32)
            self.h = L.rp_mirror_polisher_open_with_bp(len(self._off) - 1, _ptr(self._bases), _ptr(self._quals),
                                                       _ptr(self._off), _ptr(self._hq), n_targets,
                                                       1 if window_type_tgs else 0, 1 if fragment_correction else 0,
                                                       len(ov), _ptr(ov), _ptr(bp_off), _ptr(bp), window_length,
                                                       quality_threshold)
            return
        devices = _device_list(device)
        self.h = L.rp_mirror_polisher_open(len(self._off) - 1, _ptr(self._bases), _ptr(self._quals), _ptr(self._off),
                                           _ptr(self._hq), n_targets, 1 if window_type_tgs else 0,
                                           1 if fragment_correction else 0, len(ov), _ptr(ov), window_length,
                                           quality_threshold, 1 if trim else 0, match, mismatch, gap, _ptr(devices),
                                           len(devices))

    @classmethod
    def from_files(cls, reads, overlaps, targets, fragment_correction=False, window_length=500, quality_threshold=10.0,
                   error_threshold=0.3, trim=True, match=3, mismatch=-5, gap=-4, device=0, resident_reads=False):
        """createPolisher + initialize on files (reads_io.hpp): parse, filter, align + breaking points on the device
        (SAM input keeps its own alignments and needs no device here), build the windows.  device: a CUDA device index
        or a sequence of them, one lane each (an index may repeat); both device stages spread their batches over the
        lanes.  resident_reads: the sequences are uploaded once per device and the aligner (and later the consensus) name
        their inputs instead of copying them."""
        self = cls.__new__(cls)
        self.lib = load()
        self._n_overlaps = None
        devices = _device_list(device)
        err = C.create_string_buffer(1024)
        self.h = self.lib.rp_mirror_polisher_open_files(os.fsencode(reads), os.fsencode(overlaps), os.fsencode(targets),
                                                        1 if fragment_correction else 0, window_length, quality_threshold,
                                                        error_threshold, 1 if trim else 0, match, mismatch, gap,
                                                        _ptr(devices), len(devices), 1 if resident_reads else 0, err, 1024)
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
        """Polisher::polish_streaming into a FASTA file: two batch objects in flight per device lane, every polished
        sequence written in target order the moment its last window is stitched (polisher.cpp:504-537 +
        main.cpp:159-161).  names: target names by id (None: the names of the files a from_files() polisher was opened
        on).  resident_reads: every sequence is uploaded once per device and the windows are added by reference (layers
        extracted on the device)."""
        blob = None if names is None else b"".join(n.encode() + b"\0" for n in names) + b"\0"
        return self.lib.rp_mirror_polisher_stream_fasta(self.h, 1 if drop_unpolished else 0, os.fsencode(path), blob,
                                                        mem_bytes, 1 if banded else 0, 1 if resident_reads else 0)

    def breaking_points(self):
        """(bp_off, bp) of a polisher opened on arrays: the (t, q) breaking points of overlap i are
        bp[bp_off[i]:bp_off[i + 1]] — what the aligner stage produced (empty for an overlap the device refused)."""
        if self._n_overlaps is None:
            raise RaconB200Error("breaking_points: only for a polisher opened on arrays")
        n = int(self.lib.rp_mirror_polisher_breaking_points(self.h, None, None))
        off = np.zeros(self._n_overlaps + 1, np.uint64)
        bp = np.zeros((max(n, 1), 2), np.uint32)
        self.lib.rp_mirror_polisher_breaking_points(self.h, _ptr(off), _ptr(bp))
        return off, bp[:n]

    def failed(self):
        """(overlaps, windows) the device could not finish (see host_mirror.hpp: Polisher::failed_overlaps/windows)."""
        a = (C.c_uint64 * 2)()
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


def stitch_order(counts, completion):
    """The polisher's stitch cursor (host logic only): contiguous ranges of counts[r] windows finish in the order
    `completion`.  Returns (windows in the order they were stitched, for each the index into `completion` of the finish
    that stitched it)."""
    lib = load()
    counts = np.ascontiguousarray(counts, dtype=np.uint32)
    completion = np.ascontiguousarray(completion, dtype=np.uint32)
    total = int(counts.sum())
    order = np.zeros(max(total, 1), np.uint64)
    step = np.zeros(max(total, 1), np.uint32)
    n = lib.rp_mirror_stitch_order(len(counts), _ptr(counts), _ptr(completion), _ptr(order), _ptr(step))
    return order[:n], step[:n]


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


def device_memory(device=0):
    """(free bytes, total bytes) of a CUDA device (rp_device_memory)."""
    lib = load()
    free, total = C.c_uint64(), C.c_uint64()
    _check(lib, lib.rp_device_memory(device, C.byref(free), C.byref(total)), "rp_device_memory")
    return free.value, total.value


def read_store_bytes(lengths, has_quality):
    """What rp_reads_create allocates for sequences of these lengths (include/racon_b200.h, rp_reads_bytes)."""
    lengths = np.asarray(lengths, dtype=np.uint64)
    quality = bool(np.any((np.asarray(has_quality) != 0) & (lengths > 0)))
    return (int(lengths.sum()) + 16) * (2 if quality else 1)


def plan_read_groups(n_targets, lengths, has_quality, q_id, t_id, budget, *, t_begin=None, t_end=None,
                     window_length=None):
    """The target groups the host layer polishes in under a read store budget of `budget` bytes per device (host only):
    sequences of `lengths` (the first n_targets are the targets) with a quality string where has_quality, overlap k from
    sequence q_id[k] onto target t_id[k].  Returns (first_target: group g = targets [first_target[g],
    first_target[g + 1]), bytes: predicted store bytes per group, overlap_first, overlap_order: group g's overlaps are
    overlap_order[overlap_first[g]:overlap_first[g + 1]]).  Raises RaconB200Error when one target does not fit.

    With window_length (and every overlap's target span [t_begin[k], t_end[k])) a target that does not fit is split
    into parts of consecutive windows, as polish_files(split_targets=True) polishes it.  The result then also carries
    first_window, end_window (group g is windows [first_window[g], end_window[g]) of its one target when it is a part;
    0, 0 for a group of whole targets) and aligned_in (the group that aligns overlap k: the first it is in); an overlap
    is in every part it touches.  Raises RaconB200Error when one window does not fit."""
    lib = load()
    lengths = np.ascontiguousarray(lengths, dtype=np.uint32)
    has_quality = np.ascontiguousarray(has_quality, dtype=np.uint8)
    q_id = np.ascontiguousarray(q_id, dtype=np.uint32)
    t_id = np.ascontiguousarray(t_id, dtype=np.uint32)
    err = C.create_string_buffer(1024)
    split = window_length is not None
    if split:
        t_begin = np.ascontiguousarray(t_begin, dtype=np.uint32)
        t_end = np.ascontiguousarray(t_end, dtype=np.uint32)
        if len(t_begin) != len(q_id) or len(t_end) != len(q_id):
            raise ValueError("t_begin and t_end need one entry per overlap")
    inputs = (n_targets, len(lengths), _ptr(lengths), _ptr(has_quality), len(q_id), _ptr(q_id), _ptr(t_id),
              _ptr(t_begin) if split else None, _ptr(t_end) if split else None, window_length or 0, budget)
    sizes = np.zeros(2, np.uint64)
    n = lib.rp_mirror_plan_read_groups(*inputs, _ptr(sizes), *([None] * 7), err, len(err))
    if n < 0:
        raise RaconB200Error(err.value.decode(errors="replace"))
    n_groups, n_order = int(sizes[0]), int(sizes[1])
    out = [np.zeros(n_groups + 1, np.uint64), np.zeros(max(n_groups, 1), np.uint64),
           np.zeros(n_groups + 1, np.uint64), np.zeros(max(n_order, 1), np.uint64),
           np.zeros(max(n_groups, 1), np.uint32), np.zeros(max(n_groups, 1), np.uint32),
           np.zeros(max(len(q_id), 1), np.uint64)]
    lib.rp_mirror_plan_read_groups(*inputs, _ptr(sizes), *[_ptr(a) for a in out], err, len(err))
    plan = (out[0], out[1][:n_groups], out[2], out[3][:n_order], out[4][:n_groups], out[5][:n_groups],
            out[6][:len(q_id)])
    return plan if split else plan[:4]


def last_grouped_run():
    """The last polish_files run of this process (with resident_reads): rp_reads_bytes of each target group's read store,
    the whole-run indices of the overlaps and windows the device refused, and per group its whole-run windows
    [first, end) (group_windows) and the number of overlaps it sent to the aligner (group_aligned)."""
    lib = load()
    counts = np.zeros(3, np.uint64)
    lib.rp_mirror_last_grouped_run(_ptr(counts), None, None, None)
    out = [np.zeros(max(int(n), 1), np.uint64) for n in counts]
    lib.rp_mirror_last_grouped_run(_ptr(counts), *[_ptr(a) for a in out])
    run = {k: [int(v) for v in a[:int(n)]]
           for k, a, n in zip(("group_bytes", "failed_overlaps", "failed_windows"), out, counts)}
    n_groups = int(counts[0])
    windows, aligned = np.zeros(max(2 * n_groups, 1), np.uint64), np.zeros(max(n_groups, 1), np.uint64)
    lib.rp_mirror_last_grouped_run_windows(_ptr(windows), _ptr(aligned))
    run["group_windows"] = [(int(windows[2 * g]), int(windows[2 * g + 1])) for g in range(n_groups)]
    run["group_aligned"] = [int(v) for v in aligned[:n_groups]]
    return run


def polish_files(reads, overlaps, targets, out_path, fragment_correction=False, window_length=500, quality_threshold=10.0,
                 error_threshold=0.3, trim=True, match=3, mismatch=-5, gap=-4, device=0, drop_unpolished=True,
                 mem_bytes=0, banded=False, resident_reads=True, read_store_bytes=0, split_targets=False):
    """racon's whole run through the C++ host layer: files in, polished FASTA out (alignment, breaking points and
    consensus on the device).  device: a CUDA device index or a sequence of them — device=range(device_count()) runs on
    every visible GPU; the file is byte-identical whatever the list.  With resident_reads (the default) the targets are
    polished in consecutive groups whose sequences fit a device read store of read_store_bytes per device (0 = half of
    the smallest free device memory); the file is the same whatever the groups.  A target whose own sequences do not fit
    is an error, or with split_targets is polished in parts of consecutive windows that fit (plan_read_groups with the
    window length), with the same file.  Returns (records written, overlaps the device refused, windows the device
    refused)."""
    if split_targets and not resident_reads:
        raise ValueError("split_targets polishes in target groups, which need resident_reads")
    if resident_reads:
        lib = load()
        devices = _device_list(device)
        err = C.create_string_buffer(1024)
        result = np.zeros(3, np.uint64)
        st = lib.rp_mirror_polish_files_grouped(
            os.fsencode(reads), os.fsencode(overlaps), os.fsencode(targets), 1 if fragment_correction else 0,
            window_length, quality_threshold, error_threshold, 1 if trim else 0, match, mismatch, gap, _ptr(devices),
            len(devices), 1 if drop_unpolished else 0, mem_bytes, 1 if banded else 0, read_store_bytes,
            1 if split_targets else 0, os.fsencode(out_path), _ptr(result), err, len(err))
        if st != 0:
            raise RaconB200Error(err.value.decode(errors="replace"))
        return tuple(int(v) for v in result)
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
