"""ctypes loader of the C ABI (include/raven_b200.h).  The shared library is
built in-tree by __graft_entry__.build(); there is no fallback of any kind:
a missing library or a missing GPU is an error."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# (RVN_LIB: a differently tuned build of the same library, development only)
LIB_PATH = os.environ.get("RVN_LIB") or os.path.join(HERE, "libraven_b200.so")

U64P = C.POINTER(C.c_uint64)
U32P = C.POINTER(C.c_uint32)
U16P = C.POINTER(C.c_uint16)


class Overlap(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in (
        "lhs_id", "lhs_begin", "lhs_end", "rhs_id", "rhs_begin", "rhs_end",
        "score", "strand")]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "index_bases", "index_records", "index_keys", "query_bases",
        "query_records", "hits", "overlaps", "pile_bins", "kernel_launches")] + [
        ("occurrence", C.c_uint32), ("reserved", C.c_uint32)]


OVLP = C.POINTER(Overlap)

# every symbol include/raven_b200.h declares, with its signature
SIGNATURES = {
    "rvn_version": (C.c_int, []),
    "rvn_ctx_create": (C.c_int, [C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "rvn_ctx_destroy": (None, [C.c_void_p]),
    "rvn_last_error": (C.c_char_p, [C.c_void_p]),
    "rvn_engine_configure": (C.c_int, [C.c_void_p] + [C.c_uint32] * 6),
    "rvn_reads_upload": (C.c_int, [C.c_void_p, U64P, U64P, U32P, C.c_uint32]),
    "rvn_reads_upload_range": (C.c_int, [C.c_void_p, U64P, U64P, U32P, C.c_uint32,
                                         C.c_uint32, C.c_uint32]),
    "rvn_reads_upload_ids": (C.c_int, [C.c_void_p, U64P, U64P, U32P, U32P, C.c_uint32]),
    "rvn_reads_upload_files": (C.c_int, [C.c_void_p, C.POINTER(C.c_char_p), C.c_uint32, U64P]),
    "rvn_reads_parsed": (C.c_int, [C.c_void_p, U64P, U64P, U32P, C.POINTER(C.c_uint8), U64P,
                                   C.c_void_p, U64P]),
    "rvn_reads_residency": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), U64P]),
    "rvn_map_external": (C.c_int, [C.c_void_p, U64P, C.c_uint32, C.c_uint32, C.c_int,
                                   C.c_int, C.c_int, C.c_int]),
    "rvn_minimize": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int]),
    "rvn_filter": (C.c_int, [C.c_void_p, C.c_double, U32P]),
    "rvn_map": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_int,
                          C.c_int, C.c_int]),
    "rvn_map_results": (C.c_int, [C.c_void_p, C.POINTER(OVLP), C.POINTER(U64P),
                                  U64P, C.POINTER(U32P), C.POINTER(U64P)]),
    "rvn_pile_add_layers": (C.c_int, [C.c_void_p, U16P, U64P, C.c_uint32, OVLP,
                                      C.c_uint64]),
    "rvn_poa_batch": (C.c_int, [C.c_void_p, C.c_uint32, U32P, U64P, C.c_char_p, C.c_char_p,
                                U32P, U32P, C.c_int8, C.c_int8, C.c_int8, C.c_int, C.c_int,
                                C.c_int]),
    "rvn_poa_results": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(U64P),
                                  C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(U32P), U64P]),
    "rvn_poa_routes": (C.c_int, [C.c_void_p, U32P, U32P]),
    "rvn_polish_windows": (C.c_int, [C.c_void_p, C.c_uint64, U32P, U32P, U32P,
                                     C.POINTER(C.c_uint8), U32P, U64P, U32P, C.c_uint32,
                                     C.c_uint32, C.POINTER(C.c_uint8), U64P,
                                     C.POINTER(C.c_uint8), C.c_double, C.c_int8, C.c_int8,
                                     C.c_int8, C.c_int, C.c_int, U32P]),
    "rvn_kmer_complexity": (C.c_int, [C.c_void_p, U32P, U32P, C.c_uint64, C.c_uint32,
                                      C.POINTER(C.c_uint8)]),
    "rvn_find_overlaps_and_create_piles": (
        C.c_int, [C.c_void_p, C.c_double, C.c_uint64, C.c_int, C.c_uint64,
                  C.c_uint64]),
    "rvn_find_overlaps_and_repetitive_regions": (
        C.c_int, [C.c_void_p, C.c_double, C.c_double, C.c_uint32, U32P, U32P]),
    "rvn_stage2_results": (C.c_int, [C.c_void_p, C.POINTER(OVLP), C.POINTER(U64P),
                                     C.POINTER(U32P), C.POINTER(U64P),
                                     C.POINTER(C.POINTER(C.c_uint8)), U64P]),
    "rvn_stage1_footprint": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64,
                                       U64P, U64P, U64P]),
    "rvn_index_footprint": (C.c_int, [C.c_void_p, C.c_uint64, U64P, U64P]),
    "rvn_minimize_footprint": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, U64P, U64P, U64P]),
    "rvn_stage1_results": (C.c_int, [C.c_void_p, C.POINTER(OVLP), C.POINTER(U64P),
                                     C.POINTER(U16P), C.POINTER(U64P), U64P]),
    "rvn_sketch": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int,
                             C.POINTER(U64P), C.POINTER(U64P), C.POINTER(U64P),
                             U64P]),
    "rvn_index_records": (C.c_int, [C.c_void_p, C.POINTER(U64P), C.POINTER(U64P),
                                    U64P, U64P]),
    "rvn_map_hits": (C.c_int, [C.c_void_p, C.POINTER(U64P), C.POINTER(U64P),
                               C.POINTER(U64P), U64P]),
    "rvn_edit_distance_batch": (C.c_int, [C.c_void_p, C.c_uint64, U32P, U32P, U32P, U32P, U32P,
                                          U32P, C.POINTER(C.c_uint8), C.POINTER(C.c_int32),
                                          C.POINTER(C.c_int32)]),
    "rvn_stage1_pile_regions": (C.c_int, [C.c_void_p, C.c_uint32, U32P, U32P, U16P,
                                          C.POINTER(C.c_uint8)]),
    "rvn_align_breaking_points": (C.c_int, [C.c_void_p, C.c_uint64, U32P, U32P, U32P,
                                            C.POINTER(C.c_uint8), U32P, U32P, U32P, C.c_uint32,
                                            U64P, C.POINTER(C.c_int32), U32P]),
    "rvn_debug_sort_pairs": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_uint64, C.c_int, C.c_int, C.c_int]),
    "rvn_debug_partition_keys": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int,
                                           C.c_int, C.c_void_p]),
    "rvn_debug_exclusive_scan": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "rvn_get_stats": (C.c_int, [C.c_void_p, C.POINTER(Stats)]),
    "rvn_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int64]),
    "rvn_get_timings": (C.c_int, [C.c_void_p, C.POINTER(C.POINTER(C.c_char_p)),
                                  C.POINTER(C.POINTER(C.c_float)), U32P]),
    "rvn_dist_sketch_split": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int,
                                        C.c_uint32, C.POINTER(C.c_void_p),
                                        C.POINTER(C.c_void_p), U64P]),
    "rvn_dist_index_limited": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                         C.c_uint64, C.c_uint64]),
    "rvn_dist_max_threshold": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, U64P]),
    "rvn_dist_index": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                 C.c_uint64]),
    "rvn_dist_histogram": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), U32P, U64P]),
    "rvn_dist_set_occurrence": (C.c_int, [C.c_void_p, U64P, C.c_uint64, C.c_double, U32P]),
    "rvn_dist_hits_split": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64,
                                      C.c_int, C.c_int, C.c_uint32, C.c_uint32,
                                      C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                      C.POINTER(C.c_void_p), U64P]),
    "rvn_dist_chain": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_uint64, C.c_uint32, U64P, C.c_uint32, C.c_uint32,
                                 C.c_uint32, C.POINTER(C.c_void_p), U64P]),
    "rvn_dist_overlaps_split": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32,
                                          C.POINTER(C.c_void_p), U64P]),
    "rvn_dist_stage1_begin": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32]),
    "rvn_dist_stage1_add": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32,
                                      U64P, C.c_uint32, C.c_uint64, C.c_uint64]),
    "rvn_dist_stage1_end": (C.c_int, [C.c_void_p]),
    "rvn_dist_stage1_results": (C.c_int, [C.c_void_p, C.POINTER(OVLP), C.POINTER(U64P),
                                          C.POINTER(U16P), C.POINTER(U64P), U32P, U64P]),
    "rvn_dist_arena_export": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p]),
    "rvn_dist_arena_import": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]),
    "rvn_dist_arena_close_peers": (C.c_int, [C.c_void_p]),
    "rvn_dist_arena": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), U64P]),
    "rvn_dist_put": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64, C.c_void_p,
                               C.c_uint64]),
    "rvn_dist_put_flush": (C.c_int, [C.c_void_p]),
}

_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: run `python __graft_entry__.py` to "
                "build the CUDA extension (there is no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib
