"""ctypes bindings of the CPU oracle (oracle/liboracle.so) and, when present,
of the compiled reference (oracle/_ref/libraven_ref.so).  TEST INFRASTRUCTURE:
only tests/, __graft_entry__.smoke() and bench.py's CPU legs import this."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
_U64P = C.POINTER(C.c_uint64)
_U32P = C.POINTER(C.c_uint32)
_U16P = C.POINTER(C.c_uint16)
_U8P = C.POINTER(C.c_uint8)


def build_oracle(quiet=True):
    """Compile oracle/ (and oracle/_ref when /root/reference is present)."""
    subprocess.run(["make", "-C", ORACLE_DIR, "-j4"], check=True,
                   stdout=subprocess.DEVNULL if quiet else None)


def _ptr(a, typ):
    return a.ctypes.data_as(typ) if a is not None else None


class _Flat:
    """Common plumbing: bags of named arrays + read sets."""

    def __init__(self, path, prefix):
        self.lib = C.CDLL(path)
        self.p = prefix
        L = self.lib
        g = lambda n: getattr(L, prefix + n)
        g("_bag_len").restype = C.c_int64
        g("_bag_len").argtypes = [C.c_void_p, C.c_char_p]
        g("_bag_ptr").restype = C.c_void_p
        g("_bag_ptr").argtypes = [C.c_void_p, C.c_char_p]
        g("_bag_free").argtypes = [C.c_void_p]
        g("_reads_create").restype = C.c_void_p
        g("_reads_create").argtypes = [_U64P, _U64P, _U32P, C.c_uint32, _U8P, _U64P]
        g("_reads_free").argtypes = [C.c_void_p]

    def reads(self, rs):
        words = np.ascontiguousarray(rs.words, dtype=np.uint64)
        if words.size == 0:
            words = np.zeros(1, np.uint64)
        woff = np.ascontiguousarray(rs.word_off, dtype=np.uint64)
        lens = np.ascontiguousarray(rs.lens, dtype=np.uint32)
        bq = bqo = None
        if rs.block_quality is not None:
            bq = np.ascontiguousarray(rs.block_quality, dtype=np.uint8)
            bqo = np.ascontiguousarray(rs.bq_off, dtype=np.uint64)
        h = getattr(self.lib, self.p + "_reads_create")(
            _ptr(words, _U64P), _ptr(woff, _U64P), _ptr(lens, _U32P), rs.n,
            _ptr(bq, _U8P), _ptr(bqo, _U64P))
        return _Handle(h, getattr(self.lib, self.p + "_reads_free"))

    def unbag(self, bag, spec):
        out = {}
        for name, dt in spec.items():
            n = getattr(self.lib, self.p + "_bag_len")(bag, name.encode())
            if n < 0:
                continue
            ptr = getattr(self.lib, self.p + "_bag_ptr")(bag, name.encode())
            if n == 0:
                out[name] = np.zeros(0, dtype=dt)
            else:
                buf = (C.c_uint8 * n).from_address(ptr)
                out[name] = np.frombuffer(buf, dtype=dt).copy()
        getattr(self.lib, self.p + "_bag_free")(bag)
        return out


class _Handle:
    def __init__(self, h, free):
        self.h, self._free = h, free

    def __del__(self):
        if self.h:
            self._free(self.h)
            self.h = None


_STAGE1 = dict(overlaps=np.uint32, ovl_off=np.uint64, pile=np.uint16,
               pile_off=np.uint64, occurrences=np.uint32, num_mapped=np.uint64,
               seconds=np.float64)


class Oracle(_Flat):
    def __init__(self):
        path = os.path.join(ORACLE_DIR, "liboracle.so")
        if not os.path.exists(path):
            build_oracle()
        super().__init__(path, "orc")
        L = self.lib
        L.orc_engine_create.restype = C.c_void_p
        L.orc_engine_create.argtypes = [C.c_uint32] * 7
        L.orc_engine_free.argtypes = [C.c_void_p]
        L.orc_sketch.restype = C.c_void_p
        L.orc_sketch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]
        L.orc_engine_minimize.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]
        L.orc_engine_filter.restype = C.c_int
        L.orc_engine_filter.argtypes = [C.c_void_p, C.c_double, _U32P]
        L.orc_engine_keys.restype = C.c_void_p
        L.orc_engine_keys.argtypes = [C.c_void_p]
        L.orc_engine_map.restype = C.c_void_p
        L.orc_engine_map.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                     C.c_int, C.c_int, C.c_int, C.c_int]
        L.orc_engine_chain.restype = C.c_void_p
        L.orc_engine_chain.argtypes = [C.c_void_p, C.c_uint32, _U64P, _U64P, C.c_uint64]
        L.orc_stage1.restype = C.c_void_p
        L.orc_stage1.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_uint64, C.c_int,
                                 C.c_uint64, C.c_uint64]
        L.orc_pile_add_layers.argtypes = [C.c_uint32, _U16P, C.c_uint32, _U32P, C.c_uint64]
        L.orc_truncate.restype = C.c_uint64
        L.orc_truncate.argtypes = [_U32P, C.c_uint64, C.c_uint64]
        L.orc_edit_distance.restype = C.c_int
        L.orc_edit_distance.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int]

    def engine(self, k=15, w=5, bandwidth=500, chain=4, matches=100, gap=10000,
               threads=1):
        h = self.lib.orc_engine_create(k, w, bandwidth, chain, matches, gap, threads)
        return _Handle(h, self.lib.orc_engine_free)

    def sketch(self, eng, reads, first, last, minhash):
        bag = self.lib.orc_sketch(eng.h, reads.h, first, last, int(minhash))
        return self.unbag(bag, dict(value=np.uint64, origin=np.uint64, offsets=np.uint64))

    def minimize(self, eng, reads, first, last, minhash):
        self.lib.orc_engine_minimize(eng.h, reads.h, first, last, int(minhash))

    def filter(self, eng, f):
        occ = C.c_uint32(0)
        if self.lib.orc_engine_filter(eng.h, f, C.byref(occ)) != 0:
            raise ValueError("[ram::MinimizerEngine::Filter] error: invalid frequency")
        return occ.value

    def keys(self, eng):
        return self.unbag(self.lib.orc_engine_keys(eng.h),
                          dict(values=np.uint64, counts=np.uint32, totals=np.uint64))

    def map(self, eng, reads, first, last, avoid_equal=True, avoid_symmetric=True,
            minhash=False, want_matches=False):
        bag = self.lib.orc_engine_map(eng.h, reads.h, first, last, int(avoid_equal),
                                      int(avoid_symmetric), int(minhash), int(want_matches))
        r = self.unbag(bag, dict(overlaps=np.uint32, ovl_off=np.uint64, filtered=np.uint32,
                                 filt_off=np.uint64, match_group=np.uint64,
                                 match_pos=np.uint64, match_off=np.uint64))
        r["overlaps"] = r["overlaps"].reshape(-1, 8)
        return r

    def chain(self, eng, lhs_id, group, positions):
        g = np.ascontiguousarray(group, dtype=np.uint64)
        p = np.ascontiguousarray(positions, dtype=np.uint64)
        bag = self.lib.orc_engine_chain(eng.h, lhs_id, _ptr(g, _U64P), _ptr(p, _U64P), g.size)
        return self.unbag(bag, dict(overlaps=np.uint32))["overlaps"].reshape(-1, 8)

    def stage1(self, eng, reads, freq=0.001, max_overlaps=32, minhash=False,
               index_batch_bases=1 << 32, query_batch_bases=1 << 30):
        bag = self.lib.orc_stage1(eng.h, reads.h, freq, max_overlaps, int(minhash),
                                  index_batch_bases, query_batch_bases)
        r = self.unbag(bag, _STAGE1)
        r["overlaps"] = r["overlaps"].reshape(-1, 8)
        return r

    def pile_add_layers(self, read_id, data, overlaps):
        d = np.ascontiguousarray(data, dtype=np.uint16).copy()
        o = np.ascontiguousarray(overlaps, dtype=np.uint32).reshape(-1, 8)
        self.lib.orc_pile_add_layers(read_id, _ptr(d, _U16P), d.size, _ptr(o, _U32P), o.shape[0])
        return d

    def truncate(self, overlaps, max_overlaps=32):
        o = np.ascontiguousarray(overlaps, dtype=np.uint32).reshape(-1, 8).copy()
        n = self.lib.orc_truncate(_ptr(o, _U32P), o.shape[0], max_overlaps)
        return o[:n]

    def kmer_complexity(self, reads, read_index, positions, k):
        ri = np.ascontiguousarray(read_index, dtype=np.uint32)
        po = np.ascontiguousarray(positions, dtype=np.uint32)
        keep = np.zeros(ri.size, dtype=np.uint8)
        self.lib.orc_kmer_complexity.argtypes = [C.c_void_p, _U32P, _U32P, C.c_uint64,
                                                 C.c_uint32, _U8P]
        self.lib.orc_kmer_complexity(reads.h, _ptr(ri, _U32P), _ptr(po, _U32P), ri.size, k,
                                     _ptr(keep, _U8P))
        return keep

    def poa_batch(self, w, m=3, n=-5, g=-4, trim=True, tgs=True, threads=4):
        """racon window consensus over the flat window batch `w` (synth.make_windows)."""
        L = self.lib
        L.orc_poa_batch.restype = C.c_void_p
        L.orc_poa_batch.argtypes = [C.c_uint32, _U32P, _U64P, C.c_char_p, C.c_char_p, _U32P,
                                    _U32P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_uint32]
        wf = np.ascontiguousarray(w["win_first"], dtype=np.uint32)
        so = np.ascontiguousarray(w["seq_off"], dtype=np.uint64)
        ba = np.ascontiguousarray(w["bases"], dtype=np.uint8)
        qu = None if w.get("quals") is None else np.ascontiguousarray(w["quals"], dtype=np.uint8)
        sb = np.ascontiguousarray(w["seq_begin"], dtype=np.uint32)
        se = np.ascontiguousarray(w["seq_end"], dtype=np.uint32)
        bag = L.orc_poa_batch(wf.size - 1, _ptr(wf, _U32P), _ptr(so, _U64P),
                              ba.ctypes.data_as(C.c_char_p),
                              qu.ctypes.data_as(C.c_char_p) if qu is not None else None,
                              _ptr(sb, _U32P), _ptr(se, _U32P), m, n, g, int(trim), int(tgs),
                              threads)
        return self.unbag(bag, dict(consensus=np.uint8, cons_off=np.uint64, coverage=np.uint32,
                                    cov_off=np.uint64, status=np.uint8, cells=np.uint64,
                                    seconds=np.float64))

    def polish(self, targets, sequences, q=0.0, e=0.3, w=500, trim=True, m=3, n=-5, g=-4,
               threads=4):
        """racon::Polisher (oracle): polished targets as ASCII + names + stats."""
        L = self.lib
        L.orc_polish.restype = C.c_void_p
        L.orc_polish.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_uint32,
                                 C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint32]
        t, s = self.reads(targets), self.reads(sequences)
        # names "Utg<i>" / "r<i>" like the product's host shim
        L.orc_reads_set_names.argtypes = [C.c_void_p, C.c_char_p]
        L.orc_reads_set_names(t.h, b"Utg")
        L.orc_reads_set_names(s.h, b"r")
        bag = L.orc_polish(t.h, s.h, q, e, w, int(trim), m, n, g, threads)
        r = self.unbag(bag, dict(sequences=np.uint8, seq_off=np.uint64, names=np.uint8,
                                 stats=np.float64))
        names = r["names"].tobytes().decode().split("\n")[:-1]
        seqs = [r["sequences"][int(r["seq_off"][i]):int(r["seq_off"][i + 1])].tobytes()
                for i in range(len(names))]
        return names, seqs, r["stats"]

    def edit_distance(self, a: bytes, b: bytes) -> int:
        return self.lib.orc_edit_distance(a, len(a), b, len(b))


class Reference(_Flat):
    """The reference's own sources compiled in place (oracle/_ref)."""

    PATH = os.path.join(ORACLE_DIR, "_ref", "libraven_ref.so")

    @classmethod
    def available(cls):
        return os.path.exists(cls.PATH)

    def __init__(self):
        super().__init__(self.PATH, "ref")
        L = self.lib
        L.ref_stage1.restype = C.c_void_p
        L.ref_stage1.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_double,
                                 C.c_uint64, C.c_int, C.c_uint32]
        L.ref_pile_add_layers.restype = C.c_void_p
        L.ref_pile_add_layers.argtypes = [C.c_uint32, C.c_uint32, _U32P, C.c_uint64, C.c_uint32]
        L.ref_overlap_length.restype = C.c_uint32
        L.ref_overlap_length.argtypes = [_U32P]

    def stage1(self, reads, k=15, w=5, freq=0.001, max_overlaps=32, minhash=False,
               threads=1):
        bag = self.lib.ref_stage1(reads.h, k, w, freq, max_overlaps, int(minhash), threads)
        r = self.unbag(bag, _STAGE1)
        r["overlaps"] = r["overlaps"].reshape(-1, 8)
        return r

    def kmer_complexity(self, reads, read_index, positions, k):
        ri = np.ascontiguousarray(read_index, dtype=np.uint32)
        po = np.ascontiguousarray(positions, dtype=np.uint32)
        keep = np.zeros(ri.size, dtype=np.uint8)
        self.lib.ref_kmer_complexity.argtypes = [C.c_void_p, _U32P, _U32P, C.c_uint64,
                                                 C.c_uint32, _U8P]
        self.lib.ref_kmer_complexity(reads.h, _ptr(ri, _U32P), _ptr(po, _U32P), ri.size, k,
                                     _ptr(keep, _U8P))
        return keep

    def pile_add_layers(self, read_id, length, overlaps, rounds=1):
        o = np.ascontiguousarray(overlaps, dtype=np.uint32).reshape(-1, 8)
        bag = self.lib.ref_pile_add_layers(read_id, length, _ptr(o, _U32P), o.shape[0], rounds)
        return self.unbag(bag, dict(pile=np.uint16))["pile"]


class ReferenceStage2(_Flat):
    """The reference's stage 2 over given valid regions (oracle/_ref/libraven_ref_stage2.so)."""

    PATH = os.path.join(ORACLE_DIR, "_ref", "libraven_ref_stage2.so")

    @classmethod
    def available(cls):
        return os.path.exists(cls.PATH)

    def __init__(self):
        super().__init__(self.PATH, "refs2")
        L = self.lib
        L.ref_stage2.restype = C.c_void_p
        L.ref_stage2.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_double, C.c_double,
                                 C.c_uint32, _U32P, _U32P, _U8P]

    def stage2(self, rs, k, w, freq, identity, region_begin, region_end, invalid, threads=1):
        """raven::FindOverlapsAndRepetetiveRegions over fresh piles of the reads of `rs`
        (ids 0..n-1) with the given valid regions (in bins) and invalid flags: valid (the
        sorted valid ids it maps, the first s), s, overlaps (overlaps.back() at the end),
        per pile kmers (Pile::kmers_), touched (kmers_ resized) and contained."""
        rb = np.ascontiguousarray(region_begin, dtype=np.uint32)
        re_ = np.ascontiguousarray(region_end, dtype=np.uint32)
        inv = np.ascontiguousarray(invalid, dtype=np.uint8)
        if not rb.size == re_.size == inv.size == rs.n:
            raise ValueError("one region and flag per read")
        reads = self.reads(rs)
        bag = self.lib.ref_stage2(reads.h, k, w, freq, identity, threads, _ptr(rb, _U32P),
                                  _ptr(re_, _U32P), _ptr(inv, _U8P))
        r = self.unbag(bag, dict(valid=np.uint32, s=np.uint32, overlaps=np.uint32,
                                 kmers=np.uint8, kmer_off=np.uint64, touched=np.uint8,
                                 contained=np.uint8))
        off = r.pop("kmer_off")
        flat = r.pop("kmers").astype(bool)
        r["kmers"] = [flat[int(off[i]):int(off[i + 1])] for i in range(rs.n)]
        r["s"] = int(r["s"][0])
        r["overlaps"] = r["overlaps"].reshape(-1, 8)
        r["touched"] = r["touched"].astype(bool)
        r["contained"] = r["contained"].astype(bool)
        return r


def ref_pile_trim(ref, pile, pile_off, coverage=4):
    """Pile::FindValidRegion(coverage) + FindMedian of the compiled reference (oracle/_ref)
    on the given histograms: begin, end, median, invalid per pile and the trimmed data."""
    d = np.ascontiguousarray(pile, dtype=np.uint16)
    off = np.ascontiguousarray(pile_off, dtype=np.uint64)
    n = off.size - 1
    b, e = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    m, inv = np.zeros(n, np.uint16), np.zeros(n, np.uint8)
    out = np.zeros_like(d)
    ref.lib.ref_pile_trim.restype = None
    ref.lib.ref_pile_trim.argtypes = [_U16P, _U64P, C.c_uint32, C.c_uint32, _U32P, _U32P, _U16P,
                                      _U8P, _U16P]
    ref.lib.ref_pile_trim(_ptr(d, _U16P), _ptr(off, _U64P), n, coverage, _ptr(b, _U32P),
                          _ptr(e, _U32P), _ptr(m, _U16P), _ptr(inv, _U8P), _ptr(out, _U16P))
    return dict(begin=b, end=e, median=m, invalid=inv, data=out)


def ref_assemble(ref, rs, minhash=True, rounds=2, threads=4):
    """RavenTest.Assemble through the compiled reference sources (oracle/_ref)."""
    ref.lib.ref_assemble.restype = C.c_void_p
    ref.lib.ref_assemble.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32]
    reads = ref.reads(rs)
    bag = ref.lib.ref_assemble(reads.h, int(minhash), rounds, threads)
    r = ref.unbag(bag, dict(unitigs=np.uint8, unitig_off=np.uint64, names=np.uint8))
    names = r["names"].tobytes().decode().split("\n")[:-1]
    seqs = [r["unitigs"][int(r["unitig_off"][i]):int(r["unitig_off"][i + 1])].tobytes()
            for i in range(len(names))]
    return names, seqs
