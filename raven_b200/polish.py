"""Host-side mirror of the reference's polishing call over the C++ facade:
``racon::Polisher::Create(pool, q, e, w, trim, m, n, g, ...)->Polish(targets,
sequences, false)`` (RavenLib/src/polish.cc:43-51) through
raven_b200/libraven_b200_host.so (raven_b200/host/host_api.cc).  GPU: read-to-target
mapping, alignment paths and window cuts, racon's layer rules, the window layers and
their consensus (POA); host: best overlap per read and stitching.  There is no CPU
path."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import seqio

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def _load():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "libraven_b200_host.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: run `python __graft_entry__.py`")
        lib = C.CDLL(path)
        u64p, u32p, u8p = (C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8))
        lib.rvnh_polish.restype = C.c_void_p
        lib.rvnh_polish.argtypes = [u64p, u64p, u32p, C.c_uint32, u64p, u64p, u32p, u8p, u64p,
                                    C.c_uint32, C.c_double, C.c_double, C.c_uint32, C.c_int,
                                    C.c_int, C.c_int, C.c_int, C.c_uint32]
        for name, res in (("rvnh_polish_error", C.c_char_p), ("rvnh_polish_count", C.c_uint32),
                          ("rvnh_polish_words", C.c_void_p), ("rvnh_polish_word_off", C.c_void_p),
                          ("rvnh_polish_lens", C.c_void_p), ("rvnh_polish_names", C.c_char_p),
                          ("rvnh_polish_stats", C.POINTER(C.c_double)),
                          ("rvnh_polish_free", None)):
            getattr(lib, name).restype = res
            getattr(lib, name).argtypes = [C.c_void_p]
        _LIB = lib
    return _LIB


def polish(targets, sequences, q=0.0, e=0.3, w=500, trim=True, m=3, n=-5, g=-4, threads=4):
    """Polished targets (ReadSet with names) and stats: windows, polished windows,
    windows on the wide consensus kernel (deeper than the 16-bit kernels take), the
    window batches of the consensus, seconds in the consensus phase (device layer
    build + POA kernels + D2H), total seconds."""
    lib = _load()
    u64p, u32p, u8p = (C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8))

    def flat(rs):
        words = np.ascontiguousarray(rs.words, dtype=np.uint64)
        if words.size == 0:
            words = np.zeros(1, np.uint64)
        return (words, np.ascontiguousarray(rs.word_off, dtype=np.uint64),
                np.ascontiguousarray(rs.lens, dtype=np.uint32))

    tw, to, tl = flat(targets)
    sw, so, sl = flat(sequences)
    bq = bqo = None
    if sequences.block_quality is not None:
        bq = np.ascontiguousarray(sequences.block_quality, dtype=np.uint8)
        bqo = np.ascontiguousarray(sequences.bq_off, dtype=np.uint64)
    h = lib.rvnh_polish(tw.ctypes.data_as(u64p), to.ctypes.data_as(u64p), tl.ctypes.data_as(u32p),
                        targets.n, sw.ctypes.data_as(u64p), so.ctypes.data_as(u64p),
                        sl.ctypes.data_as(u32p),
                        bq.ctypes.data_as(u8p) if bq is not None else None,
                        bqo.ctypes.data_as(u64p) if bqo is not None else None, sequences.n,
                        q, e, w, int(trim), m, n, g, threads)
    try:
        err = lib.rvnh_polish_error(h).decode()
        if err:
            raise (ValueError if "invalid" in err or "must be" in err else RuntimeError)(err)
        cnt = lib.rvnh_polish_count(h)

        def view(ptr, k, dt):
            if k == 0:
                return np.zeros(0, dt)
            buf = (C.c_uint8 * (k * np.dtype(dt).itemsize)).from_address(ptr)
            return np.frombuffer(buf, dtype=dt).copy()

        woff = view(lib.rvnh_polish_word_off(h), cnt + 1, np.uint64)
        rs = seqio.ReadSet(view(lib.rvnh_polish_words(h), int(woff[-1]) if cnt else 0, np.uint64),
                           woff, view(lib.rvnh_polish_lens(h), cnt, np.uint32))
        rs.names = lib.rvnh_polish_names(h).decode().split("\n")[:-1]
        st = lib.rvnh_polish_stats(h)
        stats = dict(windows=int(st[0]), polished_windows=int(st[1]),
                     wide_windows=int(st[10]), window_batches=int(st[11]),
                     poa_seconds=st[2],
                     seconds=st[3],
                     phases_s=dict(map=st[4], align=st[5], pack=st[6], consensus=st[7],
                                   stitch=st[8], pieces=st[9]))
        return rs, stats
    finally:
        lib.rvnh_polish_free(h)
