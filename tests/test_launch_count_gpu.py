"""gb_launch_count counts exactly the kernels the library puts on the GPU, on the entry points whose launch set
branches on their arguments: the counter's delta over a call equals the kernel activities torch.profiler records for it
(memsets and copies excluded).  Inputs are zeros (and rays that miss every box), allocated before the profiled window,
so the calls take their host-side branches without touching out-of-range memory.  Also: the shared memory opt-in is
made per device, so the same wide launches succeed on a second GPU in one process."""
import json

import pytest
import torch

from goliath_b200 import _lib

ACT = torch.profiler.ProfilerActivity


def _zf(dev, *shape):
    return torch.zeros(*shape, device=dev)


def _zi(dev, *shape, fill=0):
    return torch.full(shape, fill, dtype=torch.int32, device=dev)


def _ws(dev, nbytes):
    return torch.zeros(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def _counted_and_traced(call, trace):
    K = _lib.kernels()
    torch.cuda.synchronize()
    before = K.gb_launch_count()
    with torch.profiler.profile(activities=[ACT.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    delta = K.gb_launch_count() - before
    prof.export_chrome_trace(str(trace))
    kernels = [e["name"] for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") == "kernel"]
    return delta, kernels


def _assert_counted(call, tmp_path):
    # the profiler can drop an activity record now and then; a miscount repeats on every attempt
    for _ in range(3):
        delta, kernels = _counted_and_traced(call, tmp_path / "trace.json")
        if delta == len(kernels):
            break
    assert delta == len(kernels), (delta, sorted(k[:60] for k in kernels))
    assert delta > 0


# ---------------------------------------------------------------- weight-normalised convolutions
@pytest.mark.gpu
@pytest.mark.parametrize("bias_mode", [0, 1, 2])
@pytest.mark.parametrize("apply_act", [0, 1])
@pytest.mark.parametrize("with_gx", [False, True])
def test_conv2d_wnub_bwd(cuda, tmp_path, bias_mode, apply_act, with_gx):
    K = _lib.kernels()
    B, Cin, Cout, H, W, k = 2, 8, 8, 16, 16, 3
    x, out, gout, gz = (_zf(cuda, B, c, H, W) for c in (Cin, Cout, Cout, Cout))
    v, scale, g_bias = _zf(cuda, Cout, Cin, k, k), _zf(cuda, Cout), _zf(cuda, Cout, H, W)
    gx = _zf(cuda, B, Cin, H, W) if with_gx else None
    gw = _zf(cuda, Cout, Cin, k, k)
    ws = _ws(cuda, K.gb_conv2d_wnub_bwd_workspace_bytes(B, Cin, Cout, H, W, k))
    _assert_counted(lambda: K.gb_conv2d_wnub_bwd(B, Cin, Cout, H, W, k, x, Cin * H * W, v, scale, out, gout, 0.2,
                                                 apply_act, bias_mode, gz, g_bias, gx, gw, ws), tmp_path)


# wide: the high-resolution kernels (> 48 KB of shared memory); narrow: the round-1 kernels
DECONV_SHAPES = {"wide": (2, 16, 16, 32, 32), "narrow": (2, 64, 32, 8, 8)}
CONV_SHAPES = {"wide": (5, 16, 64, 64, 64), "narrow": (2, 64, 32, 8, 8)}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["wide", "narrow"])
def test_deconv4x4s2_fwd(cuda, tmp_path, shape):
    K = _lib.kernels()
    B, Cin, Cout, Hi, Wi = DECONV_SHAPES[shape]
    x, v, scale = _zf(cuda, B, Cin, Hi, Wi), _zf(cuda, Cin, Cout, 4, 4), _zf(cuda, Cout)
    bias, out = _zf(cuda, Cout, 2 * Hi, 2 * Wi), _zf(cuda, B, Cout, 2 * Hi, 2 * Wi)
    _assert_counted(lambda: K.gb_deconv4x4s2_wnub_fwd(B, Cin, Cout, Hi, Wi, x, v, scale, bias, 0.2, 1, out), tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["wide", "narrow"])
def test_conv4x4s2_fwd(cuda, tmp_path, shape):
    K = _lib.kernels()
    B, Cin, Cout, Ho, Wo = CONV_SHAPES[shape]
    x, v, scale = _zf(cuda, B, Cin, 2 * Ho, 2 * Wo), _zf(cuda, Cout, Cin, 4, 4), _zf(cuda, Cout)
    bias, out = _zf(cuda, Cout, Ho, Wo), _zf(cuda, B, Cout, Ho, Wo)
    _assert_counted(lambda: K.gb_conv4x4s2_wnub_fwd(B, Cin, Cout, Ho, Wo, x, v, scale, bias, 0.2, 1, out), tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("layer", ["deconv", "conv"])
@pytest.mark.parametrize("shape", ["wide", "narrow"])
@pytest.mark.parametrize("apply_act, with_bias, with_gx, with_gw",
                         [(1, True, True, True), (0, True, False, True), (0, False, True, False), (1, True, False, False)])
def test_4x4s2_bwd(cuda, tmp_path, layer, shape, apply_act, with_bias, with_gx, with_gw):
    K = _lib.kernels()
    if layer == "deconv":
        B, Cin, Cout, Hi, Wi = DECONV_SHAPES[shape]
        xs, ys, wshape = (Hi, Wi), (2 * Hi, 2 * Wi), (Cin, Cout, 4, 4)
        fn, wsb = K.gb_deconv4x4s2_wnub_bwd, K.gb_deconv4x4s2_wnub_bwd_workspace_bytes
    else:
        B, Cin, Cout, Hi, Wi = CONV_SHAPES[shape]  # Hi, Wi: the output's size
        xs, ys, wshape = (2 * Hi, 2 * Wi), (Hi, Wi), (Cout, Cin, 4, 4)
        fn, wsb = K.gb_conv4x4s2_wnub_bwd, K.gb_conv4x4s2_wnub_bwd_workspace_bytes
    x, v, scale = _zf(cuda, B, Cin, *xs), _zf(cuda, *wshape), _zf(cuda, Cout)
    out, gout, gz = (_zf(cuda, B, Cout, *ys) for _ in range(3))
    g_bias = _zf(cuda, Cout, *ys) if with_bias else None
    gx = _zf(cuda, B, Cin, *xs) if with_gx else None
    gw = _zf(cuda, *wshape) if with_gw else None
    ws = _ws(cuda, wsb(B, Cin, Cout, Hi, Wi))
    _assert_counted(lambda: fn(B, Cin, Cout, Hi, Wi, x, v, scale, out, gout, 0.2, apply_act, gz, g_bias, gx, gw, ws),
                    tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("with_gx", [False, True])
def test_upconv_block_bwd(cuda, tmp_path, with_gx):
    K = _lib.kernels()
    B, Cin, Cout, G, Hi, Wi = 2, 16, 8, 2, 8, 8
    H, W = 2 * Hi, 2 * Wi
    x = _zf(cuda, B, Cin, Hi, Wi)
    v1, s1, v2, s2 = _zf(cuda, Cin, Cin // G, 3, 3), _zf(cuda, Cin), _zf(cuda, Cout, Cin // G, 3, 3), _zf(cuda, Cout)
    vr, sr = _zf(cuda, Cout, Cin // G, 1, 1), _zf(cuda, Cout)
    h1, gz1, gu = (_zf(cuda, B, Cin, H, W) for _ in range(3))
    mask = torch.zeros(B, Cout, H, W, dtype=torch.uint8, device=cuda)
    gout, gz2 = _zf(cuda, B, Cout, H, W), _zf(cuda, B, Cout, H, W)
    gb1, gb2, gbr = _zf(cuda, Cin, H, W), _zf(cuda, Cout, H, W), _zf(cuda, Cout)
    gw1, gw2, gwr = _zf(cuda, *v1.shape), _zf(cuda, *v2.shape), _zf(cuda, *vr.shape)
    gx = _zf(cuda, B, Cin, Hi, Wi) if with_gx else None
    ws = _ws(cuda, K.gb_upconv_block_bwd_workspace_bytes(B, Cin, Cout, G, Hi, Wi))
    _assert_counted(lambda: K.gb_upconv_block_bwd(B, Cin, Cout, G, Hi, Wi, x, v1, s1, v2, s2, vr, sr, h1, mask, gout,
                                                  0.2, gz2, gz1, gu, gb1, gb2, gbr, gw1, gw2, gwr, gx, ws), tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("with_gx", [False, True])
def test_downconv_block_bwd(cuda, tmp_path, with_gx):
    K = _lib.kernels()
    B, Cin, Cout, G, H, W = 2, 8, 16, 1, 16, 16
    Ho, Wo = H // 2, W // 2
    x = _zf(cuda, B, Cin, H, W)
    v1, s1, v2, s2 = _zf(cuda, Cin, Cin // G, 3, 3), _zf(cuda, Cin), _zf(cuda, Cout, Cin // G, 3, 3), _zf(cuda, Cout)
    vr, sr = _zf(cuda, Cout, Cin // G, 1, 1), _zf(cuda, Cout)
    h1, gz1 = _zf(cuda, B, Cin, H, W), _zf(cuda, B, Cin, H, W)
    mask = torch.zeros(B, Cout, Ho, Wo, dtype=torch.uint8, device=cuda)
    gout, gz2 = _zf(cuda, B, Cout, Ho, Wo), _zf(cuda, B, Cout, Ho, Wo)
    gb1, gb2, gbr = _zf(cuda, Cin, H, W), _zf(cuda, Cout, Ho, Wo), _zf(cuda, Cout)
    gw1, gw2, gwr = _zf(cuda, *v1.shape), _zf(cuda, *v2.shape), _zf(cuda, *vr.shape)
    gx = _zf(cuda, B, Cin, H, W) if with_gx else None
    ws = _ws(cuda, K.gb_downconv_block_bwd_workspace_bytes(B, Cin, Cout, G, H, W))
    _assert_counted(lambda: K.gb_downconv_block_bwd(B, Cin, Cout, G, H, W, x, Cin * H * W, H * W, W, H, W, None, 1.0,
                                                    v1, s1, v2, s2, vr, sr, h1, mask, gout, 0.2, gz2, gz1, gb1, gb2,
                                                    gbr, gw1, gw2, gwr, gx, ws), tmp_path)


# ---------------------------------------------------------------- mesh rasteriser and normals
@pytest.mark.gpu
@pytest.mark.parametrize("F", [0, 6])
def test_mesh_raster(cuda, tmp_path, F):
    K = _lib.kernels()
    B, V, H, W = 2, 8, 32, 24
    v_pix, vi, index_img = _zf(cuda, B, V, 3), _zi(cuda, max(F, 1), 3), _zi(cuda, B, H, W)
    ws = _ws(cuda, K.gb_mesh_raster_workspace_bytes(B, F, H, W))
    _assert_counted(lambda: K.gb_mesh_raster(B, V, F, H, W, v_pix, vi, index_img, ws), tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("F, C, edge_grad", [(6, 3, 1), (6, 3, 0), (0, 3, 1), (6, 0, 1), (0, 0, 0)])
def test_mesh_render_bwd(cuda, tmp_path, F, C, edge_grad):
    K = _lib.kernels()
    B, V, H, W, Ht, Wt = 2, 8, 32, 24, 16, 16
    v_pix, vi, vti, vt = _zf(cuda, B, V, 3), _zi(cuda, max(F, 1), 3), _zi(cuda, max(F, 1), 3), _zf(cuda, V, 2)
    tex = _zf(cuda, B, max(C, 1), Ht, Wt)
    index_img = _zi(cuda, B, H, W, fill=-1)  # background everywhere
    vt_img, render, g_render = _zf(cuda, B, 2, H, W), _zf(cuda, B, max(C, 1), H, W), _zf(cuda, B, max(C, 1), H, W)
    inc_ptr, inc = _zi(cuda, V + 1), _zi(cuda, 3 * max(F, 1))
    g_v_pix, g_tex = _zf(cuda, B, V, 3), _zf(cuda, B, max(C, 1), Ht, Wt)
    ws = _ws(cuda, K.gb_mesh_render_bwd_workspace_bytes(B, F, H, W, Ht, Wt))
    _assert_counted(lambda: K.gb_mesh_render_bwd(B, V, F, H, W, C, Ht, Wt, v_pix, vi, vti, vt, tex, index_img, vt_img,
                                                 render, g_render, edge_grad, inc_ptr, inc, g_v_pix, g_tex, ws),
                    tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("F", [0, 6])
@pytest.mark.parametrize("direction", ["fwd", "bwd"])
def test_vert_normals(cuda, tmp_path, F, direction):
    K = _lib.kernels()
    B, V = 2, 8
    v, vi, acc, vn, g_acc, g_v = _zf(cuda, B, V, 3), _zi(cuda, max(F, 1), 3), *(_zf(cuda, B, V, 3) for _ in range(4))
    if direction == "fwd":
        _assert_counted(lambda: K.gb_vert_normals_fwd(B, V, F, v, vi, 1e-8, acc, vn), tmp_path)
    else:
        _assert_counted(lambda: K.gb_vert_normals_bwd(B, V, F, v, vi, 1e-8, acc, vn, g_acc, g_v), tmp_path)


# ---------------------------------------------------------------- tile binning
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["pack_ev", "buckets"])
@pytest.mark.parametrize("late_colors", [False, True])
@pytest.mark.parametrize("img", [(256, 192), (2048, 2048)])  # 192 tiles; 16384 tiles (> 48 KB of tile counters)
def test_bin_tiles(cuda, tmp_path, entry, late_colors, img):
    K = _lib.kernels()
    G, (H, W), bw, cap = 1000, img, 16, 4096
    T = ((H + bw - 1) // bw) * ((W + bw - 1) // bw)
    xys, depths, radii, conics = _zf(cuda, G, 2), _zf(cuda, G), _zi(cuda, G), _zf(cuda, G, 3)
    colors3, opacity, comp = _zf(cuda, G, 3), _zf(cuda, G), _zf(cuda, G)
    tile_bins, tile_order, n_out, overflow = _zi(cuda, T, 2), _zi(cuda, T), _zi(cuda, 1), _zi(cuda, 1)
    ws = _ws(cuda, K.gb_bin_tiles_workspace_bytes(G, T, cap))
    ev = torch.cuda.Event()
    ev.record()
    ready = ev.cuda_event if late_colors else None
    if entry == "pack_ev":
        gids, records = _zi(cuda, cap), _zf(cuda, cap, 12)
        call = lambda: K.gb_bin_tiles_pack_ev(G, xys, depths, radii, conics, colors3, opacity, comp, H, W, bw, cap,
                                              tile_bins, tile_order, 0, gids, records, n_out, overflow, ws, ready)
    else:
        keys, bucket, rec, r2g = _zi(cuda, cap), _zi(cuda, cap), _zf(cuda, G, 12), _zi(cuda, G)
        call = lambda: K.gb_bin_tiles_buckets(G, xys, depths, radii, conics, colors3, opacity, comp, H, W, bw, cap,
                                              tile_bins, tile_order, keys, bucket, rec, r2g, n_out, overflow, ws, ready)
    _assert_counted(call, tmp_path)


# ---------------------------------------------------------------- MVP raymarcher
def _march_inputs(dev, N=2, H=16, W=32, K=4, T=4):
    raypos = torch.tensor([100.0, 100.0, -10.0], device=dev).expand(N, H, W, 3).contiguous()  # misses every box
    raydir = torch.tensor([0.0, 0.0, 1.0], device=dev).expand(N, H, W, 3).contiguous()
    tminmax = torch.tensor([0.0, 20.0], device=dev).expand(N, H, W, 2).contiguous()
    prims = dict(nodeaabb=_zf(dev, N, 2 * K - 1, 2, 3), primpos=_zf(dev, N, K, 3), primrot=_zf(dev, N, K, 3, 3),
                 primscale=_zf(dev, N, K, 3), tplate=_zf(dev, N, K, T, T, T, 4), warp=_zf(dev, N, K, T, T, T, 3))
    return raypos, raydir, tminmax, prims


# (10, 32): 10 warps, 60 KB of hit lists (above the 48 KB default); (8, 8): 2 warps
BLOCKS = [(10, 32), (8, 8)]


@pytest.fixture
def raymarch_mode():
    L = _lib.lib()
    saved = L.gb_get_raymarch_mode()
    yield L.gb_set_raymarch_mode
    L.gb_set_raymarch_mode(saved)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", [0, 1])
@pytest.mark.parametrize("mode", [0, 3])
@pytest.mark.parametrize("block", BLOCKS)
@pytest.mark.parametrize("with_shadow", [False, True])
def test_raymarch_fwd(cuda, tmp_path, raymarch_mode, algo, mode, block, with_shadow):
    K_ = _lib.kernels()
    N, H, W, K, T = 2, 16, 32, 4, 4
    raypos, raydir, tminmax, p = _march_inputs(cuda, N, H, W, K, T)
    rayrgba, raysat = _zf(cuda, N, H, W, 4), _zf(cuda, N, H, W, 4)
    shadow = _zf(cuda, N, K, T, T, T, 2) if with_shadow else None
    raymarch_mode(mode)
    _assert_counted(lambda: K_.gb_mvp_raymarch_fwd(N, H, W, K, raypos, raydir, 0.01, tminmax, p["nodeaabb"],
                                                   p["primpos"], p["primrot"], p["primscale"], T, T, T, p["tplate"], T,
                                                   T, T, p["warp"], rayrgba, raysat, shadow, algo, 1.0, 1.0, *block),
                    tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", [0, 1])
@pytest.mark.parametrize("mode", [0, 3])
@pytest.mark.parametrize("block", BLOCKS)
def test_raymarch_bwd(cuda, tmp_path, raymarch_mode, algo, mode, block):
    K_ = _lib.kernels()
    N, H, W, K, T = 2, 16, 32, 4, 4
    raypos, raydir, tminmax, p = _march_inputs(cuda, N, H, W, K, T)
    raysat, g_rgba = _zf(cuda, N, H, W, 4), _zf(cuda, N, H, W, 4)
    g = {k: torch.zeros_like(p[k]) for k in ("primpos", "primrot", "primscale", "tplate", "warp")}
    raymarch_mode(mode)
    _assert_counted(lambda: K_.gb_mvp_raymarch_bwd(N, H, W, K, raypos, raydir, 0.01, tminmax, p["nodeaabb"],
                                                   p["primpos"], p["primrot"], p["primscale"], T, T, T, p["tplate"], T,
                                                   T, T, p["warp"], raysat, g_rgba, g["primpos"], g["primrot"],
                                                   g["primscale"], g["tplate"], g["warp"], algo, 1.0, 1.0, *block),
                    tmp_path)


@pytest.mark.gpu
@pytest.mark.parametrize("block", BLOCKS)
def test_shadow_march(cuda, tmp_path, block):
    K_ = _lib.kernels()
    B, L, H, W, T, U = 2, 2, 16, 32, 4, 8
    N, K = B * L, (U // T) ** 2
    raypos, raydir, tminmax, _ = _march_inputs(cuda, N, H, W, K, T)
    _, _, _, p = _march_inputs(cuda, B, H, W, K, T)
    slab, shadow = _zf(cuda, B, T, U, U), _zf(cuda, N, K, T, T, T, 2)
    _assert_counted(lambda: K_.gb_mvp_shadow_march(N, L, H, W, K, raypos, raydir, 0.01, tminmax, p["nodeaabb"],
                                                   p["primpos"], p["primrot"], p["primscale"], T, T, T, U, slab, None,
                                                   shadow, 1.0, 1.0, *block), tmp_path)


# ---------------------------------------------------------------- the opt-in is per device
@pytest.mark.gpu
def test_wide_launches_on_two_devices(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    K_ = _lib.kernels()
    for dev in (torch.device("cuda:0"), torch.device("cuda:1")):
        B, Cin, Cout, Hi, Wi = DECONV_SHAPES["wide"]
        x, v, scale = _zf(dev, B, Cin, Hi, Wi), _zf(dev, Cin, Cout, 4, 4), _zf(dev, Cout)
        out = _zf(dev, B, Cout, 2 * Hi, 2 * Wi)
        assert K_.gb_deconv4x4s2_wnub_fwd(B, Cin, Cout, Hi, Wi, x, v, scale, None, 0.2, 1, out) == 0
        N, H, W, K, T = 2, 16, 32, 4, 4
        raypos, raydir, tminmax, p = _march_inputs(dev, N, H, W, K, T)
        rayrgba, raysat = _zf(dev, N, H, W, 4), _zf(dev, N, H, W, 4)
        assert K_.gb_mvp_raymarch_fwd(N, H, W, K, raypos, raydir, 0.01, tminmax, p["nodeaabb"], p["primpos"],
                                      p["primrot"], p["primscale"], T, T, T, p["tplate"], T, T, T, p["warp"], rayrgba,
                                      raysat, None, 0, 1.0, 1.0, *BLOCKS[0]) == 0
        torch.cuda.synchronize(dev)
