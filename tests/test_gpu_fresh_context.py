"""A context before its first upload is an empty read set: stage 1 (resident, unstreamed and
windowed), the footprint queries and the partitioned stage-1 tail take it as zero reads and
return empty results, as they do after an upload of zero reads."""
import ctypes as C

import numpy as np
import pytest

from raven_b200 import engine

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("options", [{}, {"stage1_stream": 0}, {"stage1_window": 1}])
def test_stage1_before_any_upload(options):
    eng = engine.Engine(device=0)
    try:
        for name, value in options.items():
            eng.set_option(name, value)
        got = eng.find_overlaps_and_create_piles(0.001, 32)
        assert got["overlaps"].shape == (0, 8)
        assert got["ovl_off"].tolist() == [0]
        assert got["pile"].size == 0
        assert got["pile_off"].tolist() == [0]
        assert got["num_mapped"] == 0
    finally:
        eng.close()


def test_footprints_before_any_upload():
    eng = engine.Engine(device=0)
    try:
        fp = eng.stage1_footprint(32, 0, 0)
        assert fp["windowed_host"] == 0
        assert fp["resident"] == fp["windowed_device"] == 0
        assert eng.index_footprint(0) == dict(one_shot=0, chunked=0)
        assert eng.minimize_footprint(0, 0)["one_shot"] == 0
    finally:
        eng.close()


def test_partitioned_stage1_tail_before_any_upload():
    eng = engine.Engine(device=0)
    try:
        eng._check(eng.lib.rvn_dist_stage1_begin(eng.h, 1, 0))
        eng._check(eng.lib.rvn_dist_stage1_end(eng.h))
        n_own, nm = C.c_uint32(7), C.c_uint64(7)
        poff = C.POINTER(C.c_uint64)()
        eng._check(eng.lib.rvn_dist_stage1_results(eng.h, None, None, None, C.byref(poff),
                                                   C.byref(n_own), C.byref(nm)))
        assert n_own.value == 0
        assert np.ctypeslib.as_array(poff, shape=(1,)).tolist() == [0]
    finally:
        eng.close()
