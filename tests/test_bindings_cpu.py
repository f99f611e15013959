"""CPU: the ctypes signatures derived from include/goliath_b200.h, and the launcher that `_lib.kernels()` wraps around
every entry point ending in `void* stream` (no library, no device: a fake library stands in for the CDLL)."""
import ctypes
import os
import re
import types

import pytest
import torch

from goliath_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _prototypes():
    with open(os.path.join(ROOT, "include", "goliath_b200.h")) as f:
        hdr = re.sub(r"/\*.*?\*/", "", f.read(), flags=re.S)
    return re.findall(r"\b(gb_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", hdr)


def test_one_signature_per_prototype():
    protos = _prototypes()
    names = [n for n, _ in protos]
    assert len(names) == len(set(names)) == len(_lib.SIGNATURES)
    assert set(names) == set(_lib.SIGNATURES)
    for name, params in protos:
        n_params = 0 if params.strip() == "void" else len(params.split(","))
        assert len(_lib.SIGNATURES[name][1]) == n_params, name


def test_representative_types():
    S = _lib.SIGNATURES
    res, args = S["gb_bin_tiles_pack"]
    assert res is ctypes.c_int and args[11] is ctypes.c_int64  # int64_t cap
    assert args[0] is ctypes.c_int and args[1] is ctypes.c_void_p and args[-1] is ctypes.c_void_p
    assert S["gb_sort_workspace_bytes"] == (ctypes.c_size_t, [ctypes.c_int64])
    res, args = S["gb_envmap_prefilter_sg"]
    assert args[8] is ctypes.c_ulonglong  # seed
    assert args[4:7] == [ctypes.c_void_p] * 3  # const float* const*
    assert S["gb_launch_count_reset"] == (None, [])
    assert S["gb_launch_count"] == (ctypes.c_ulonglong, [])
    assert S["gb_version"] == (ctypes.c_int, [])
    assert S["gb_project_gaussians_fwd"][1][3] is ctypes.c_float  # glob_scale
    assert S["gb_conv2d_wnub_fwd"][1][7] is ctypes.c_int64  # long long x_bs


def test_unknown_type_names_the_prototype():
    sigs, launchers = _lib.parse_header("/* ok */ int gb_a(int n, float* x, void* stream);\n"
                                        "size_t gb_b(int64_t n);\n")
    assert sigs == {"gb_a": (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
                    "gb_b": (ctypes.c_size_t, [ctypes.c_int64])}
    assert launchers == {"gb_a"}
    with pytest.raises(_lib.GoliathB200Error, match=r"gb_c\(int n, double x, void\* stream\)"):
        _lib.parse_header("int gb_ok(int n);\nint gb_c(int n, double x, void* stream);\n")
    with pytest.raises(_lib.GoliathB200Error, match="gb_d"):
        _lib.parse_header("unsigned gb_d(int n);\n")


def test_launchers_are_the_prototypes_ending_in_a_stream():
    protos = _prototypes()
    ends_in_stream = {n for n, p in protos if re.search(r"void\s*\*\s*stream\s*$", p)}
    assert _lib.LAUNCHERS == ends_in_stream
    assert len(_lib.LAUNCHERS) >= 112
    # the rest are queries, setters and sizers: none of them takes a stream
    others = set(_lib.SIGNATURES) - _lib.LAUNCHERS
    pattern = (r"gb_version|gb_launch_count\w*|gb_(get|set)_\w+_mode|gb_bin_tiles_supported|gb_tile_schedule_ints"
               r"|gb_lbs_max_joints|gb_optim_\w+|gb_compute_raydirs_bwd|\w+_(workspace|weight)_bytes")
    assert all(re.fullmatch(pattern, n) for n in others), sorted(n for n in others if not re.fullmatch(pattern, n))


class _FakeLib:
    """Stands in for the CDLL: every symbol records its arguments and returns `rc`."""

    def __init__(self):
        self.calls, self.rc = [], 0

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return self.rc

        fn.__name__ = name
        setattr(self, name, fn)
        return fn


@pytest.fixture
def fake(monkeypatch):
    lib = _FakeLib()
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.setattr(_lib, "_kernels", None)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: types.SimpleNamespace(cuda_stream=0xABC))
    return lib


def test_launcher_converts_arguments_and_appends_the_stream(fake):
    K = _lib.kernels()
    t = torch.arange(4, dtype=torch.float32)
    host = (ctypes.c_void_p * 2)(1, 2)
    assert K.gb_head_lights_fwd(3, 4, 3, t, None, host, 1.5, 7, t, t, t, t, t, None) == 0
    name, args = fake.calls[-1]
    assert name == "gb_head_lights_fwd"
    assert args == (3, 4, 3, t.data_ptr(), None, host, 1.5, 7) + (t.data_ptr(),) * 5 + (None, 0xABC)
    assert args[5] is host  # a ctypes array of host pointers passes through unchanged


def test_launcher_raises_naming_the_symbol(fake):
    K = _lib.kernels()
    fake.rc = 700
    with pytest.raises(_lib.GoliathB200Error, match="gb_tile_order failed: CUDA error 700"):
        K.gb_tile_order(1, None, None)


def test_non_launchers_are_the_plain_functions(fake):
    K = _lib.kernels()
    fake.rc = 5
    assert K.gb_version is fake.gb_version
    assert K.gb_bin_tiles_workspace_bytes(1, 2, 3) == 5
    assert fake.calls[-1] == ("gb_bin_tiles_workspace_bytes", (1, 2, 3))  # no stream appended
