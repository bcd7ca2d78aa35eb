"""No GPU: stage 2's clip (raven::OverlapUpdate) and identity bound, the one
__host__ __device__ definition in include/raven_b200/overlap_clip.hpp that the device
filter and the host IdentityFilter share, against the reference's overlap_utils.cc
(compiled in place into oracle/_ref/overlap_clip_test) and the bound's former host
definition, on seeded random overlaps and regions with their edges."""
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
BIN = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "overlap_clip_test")


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_overlap_clip_and_bound_equal_reference(seed):
    if not os.path.exists(BIN):
        pytest.skip("oracle/_ref/overlap_clip_test not built (needs the reference tree)")
    out = subprocess.run([BIN, str(seed), "200000"], check=True, stdout=subprocess.PIPE,
                         timeout=300).stdout.decode()
    words = out.split()
    assert words[0] == "ok", out
    assert int(words[3]) > 10_000 and int(words[5]) > 10_000, out  # both outcomes reached
