"""CPU: the C-ABI library loads and exports every symbol include/goliath_b200.h declares (no compute calls),
and the product package never touches the oracle."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    hdr = open(os.path.join(ROOT, "include", "goliath_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(gb_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as ge

    ge.build()
    from goliath_b200 import _lib

    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = _declared()
    assert len(names) >= 12
    for n in names:
        assert hasattr(lib, n), "missing export %s" % n
        assert n in _lib.SIGNATURES, "no ctypes signature for %s" % n
    assert set(_lib.SIGNATURES) == set(names), set(_lib.SIGNATURES) ^ set(names)
    assert _lib.lib().gb_version() >= 1000


def test_header_cites_reference_for_each_entry_point():
    hdr = open(os.path.join(ROOT, "include", "goliath_b200.h")).read()
    assert hdr.count("replaces") >= 10


def test_product_never_imports_oracle():
    bad = []
    for d, _, files in os.walk(os.path.join(ROOT, "goliath_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(d, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M) or "oracle/" in src.replace("oracle/splat_oracle.c", "").replace("oracle/_ref", "").replace("(oracle:", ""):
                    if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M) or re.search(r"#include\s+\"[^\"]*oracle", src):
                        bad.append(os.path.join(d, f))
    assert not bad, bad


def test_product_fails_loudly_without_library(monkeypatch, tmp_path):
    from goliath_b200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    try:
        _lib.lib()
    except _lib.GoliathB200Error as e:
        assert "no CPU fallback" in str(e) or "not built" in str(e)
    else:
        raise AssertionError("expected GoliathB200Error")


def test_host_side_sizing_functions():
    """Pure host functions of the C ABI (no device work): sizing of the bucket binning, schedule length, blend-mode
    switch.  They decide buffer sizes on the Python side, so their contract is pinned here."""
    from goliath_b200 import _lib

    L = _lib.lib()
    assert L.gb_bin_tiles_supported(1) == 1 and L.gb_bin_tiles_supported(300_000) == 1
    assert L.gb_bin_tiles_supported(1_048_576) == 1          # native RGCA size: 128 KB bitmap
    assert L.gb_bin_tiles_supported(0) == 0 and L.gb_bin_tiles_supported(4_000_000) == 0  # bitmap > shared memory
    T = 42 * 64
    small = L.gb_bin_tiles_workspace_bytes(300_000, T, 1 << 20)
    big = L.gb_bin_tiles_workspace_bytes(300_000, T, 1 << 22)
    assert big - small == ((1 << 22) - (1 << 20)) * 4       # one int32 rank per intersection slot
    assert small >= 300_000 * (6 * 4 + 48)                   # keys/ids ping-pong + rank_of + by-rank records
    assert small % 256 == 0
    assert L.gb_tile_schedule_ints(T) == T + 132 + 1         # one queue per SM of an H100 + the draw counter
    # the stride-2 4x4 layers' weight-gradient partials: at least one [Cin, Cout, 4, 4] per layer, none for no work
    for B, Cin, Cout, H, W in ((1, 16, 125, 64, 48), (2, 264, 40, 8, 8), (1, 256, 256, 16, 16), (1, 3, 5, 17, 33)):
        assert L.gb_deconv4x4s2_wnub_bwd_workspace_bytes(B, Cin, Cout, H, W) >= Cin * Cout * 16 * 4
        assert L.gb_conv4x4s2_wnub_bwd_workspace_bytes(B, Cin, Cout, H, W) >= Cin * Cout * 16 * 4
    assert L.gb_deconv4x4s2_wnub_bwd_workspace_bytes(0, 16, 125, 64, 48) == 0
    assert L.gb_conv4x4s2_wnub_bwd_workspace_bytes(1, 3, 32, 0, 512) == 0
    before = L.gb_get_blend_mode()
    try:
        for m in (0, 1, 2, 3, 4):
            L.gb_set_blend_mode(m)
            assert L.gb_get_blend_mode() == m
        L.gb_set_blend_mode(7)
        assert L.gb_get_blend_mode() == 4
    finally:
        L.gb_set_blend_mode(before)
    assert before in (0, 1, 2, 3, 4)
