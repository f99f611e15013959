"""Every kernel is launched through gb::launch (csrc/common.cuh), which opts it in to its dynamic shared memory, checks
the launch and counts it.  A launch written by hand anywhere else would skip one of the three."""
import os

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "goliath_b200", "csrc")
SOURCES = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh")))


def _files_with(token):
    found = []
    for f in SOURCES:
        with open(os.path.join(CSRC, f)) as fh:
            if token in fh.read():
                found.append(f)
    return found


@pytest.mark.parametrize("token, allowed", [
    ("<<<", ["common.cuh"]),
    ("cudaFuncSetAttribute", ["common.cuh"]),
    # the counter is added to by gb::launch and read / reset by gb_launch_count*
    ("g_launch_count", ["capi.cu", "common.cuh"]),
    ("count_launches", []),
    ("GB_CHECK_LAUNCH", []),
])
def test_launch_mechanics_only_in_common(token, allowed):
    assert _files_with(token) == allowed
