"""The OLAT (one-light-at-a-time) relighting path against the CPU oracle (oracle/splat_oracle.c), one oracle blend per
lighting condition (its blend takes at most 8 channels):

1. the four-condition blend kernels (gb_records_widen, gb_records_set_colors4, gb_rasterize_multi_fwd/bwd,
   gb_colors12_unpack) through the C ABI, on the oracle's projection and binning, at ragged image sizes, with culled and
   opacity-1 Gaussians, long tile lists, a non-zero background, every group size, and both tile schedules;
2. render_shared / render_views_shared (gsplat/olat.py) against the oracle chain, in every blend mode and OLAT mode;
3. bench.py's OLAT step itself (`OlatWorkload.compute`) at the benchmarked scene and image size.

Bars as for the head path: pixels rtol 1e-4 / atol 2e-5 on 99.95 % of the elements (a borderline alpha < 1/255 or
T <= 1e-4 decision can flip between ex2 and libm's expf), gradients rtol 1e-4 / atol 1e-5 * max on 99.9 %."""
import types

import numpy as np
import pytest
import torch

from fullstep import oracle_olat_step, oracle_shared_view
from util import assert_close, small_scene, t2n

pytestmark = pytest.mark.gpu

PIX = dict(rtol=1e-4, atol=2e-5, frac=0.9995)


def _gtol(want):
    return dict(rtol=1e-4, atol=1e-5 * float(np.abs(want).max()), frac=0.999)


SCENES = {
    # name: (kwargs of small_scene, scale multiplier); block width 16
    "dense96": (dict(G=3000, img_h=96, img_w=80), 12.0),
    "ragged": (dict(G=2500, img_h=70, img_w=93, seed=11, cam=3), 15.0),
    "ties": (dict(G=4000, img_h=96, img_w=80, depth_quant=True), 8.0),
    "tiny_prims": (dict(G=5000, img_h=128, img_w=96, seed=9), 1.0),
    "big": (dict(G=60000, img_h=300, img_w=260, seed=21), 3.0),
    # few tiles with thousands of records each: the backward flushes its entry list many times and carries the rest over
    "long_lists": (dict(G=40000, img_h=48, img_w=40, seed=29), 2.0),
}
GROUPS = (3, 1, 4, 2)  # conditions per pass, back to back on one v_colors12 buffer: every group size, every transition


@pytest.fixture(params=["batch", "pipe", "affine", "mom", "mom-affine"])
def blend_mode(request):
    """the five formulations of the single-condition blend; in modes 2 and 4 the tile order is an SM-affine schedule
    and the four-condition kernels draw their tiles from it too"""
    from goliath_b200 import _lib

    L = _lib.lib()
    before = L.gb_get_blend_mode()
    L.gb_set_blend_mode({"batch": 0, "pipe": 1, "affine": 2, "mom": 3, "mom-affine": 4}[request.param])
    yield request.param
    L.gb_set_blend_mode(before)


@pytest.fixture(params=["multi", "single"])
def olat_mode(request):
    """four conditions per blend pass (default) or one condition per pass"""
    from goliath_b200.gsplat import olat

    before = olat.MODE
    olat.MODE = request.param
    yield request.param
    olat.MODE = before


# ---------------------------------------------------------------------------------- 1. the kernels through the C ABI
@pytest.mark.parametrize("case", list(SCENES))
def test_multi_kernels_match_oracle_per_condition(orc, cuda, case):
    from goliath_b200 import _lib

    kw, mult = SCENES[case]
    s = small_scene(**kw)
    H, W, bw = s["img_h"], s["img_w"], 16
    p = orc.project_fwd(s["means3d"], s["scales"] * np.float32(mult), 1.0, s["quats"], s["viewmat"], s["fx"], s["fy"],
                        s["cx"], s["cy"], H, W, bw, 0.1)
    b = orc.bin_and_sort(p["xys"], p["depths"], p["radii"], p["num_tiles_hit"], H, W, bw)
    gids_o, bins_o = b["gaussian_ids_sorted"], b["tile_bins"]
    G, n, T = len(p["radii"]), int(b["num_intersects"]), len(bins_o)
    rng = np.random.default_rng(13)
    opac = (s["opacity"][:, 0] * p["compensation"]).astype(np.float32)
    if case == "long_lists":
        opac[p["xys"][:, 0] >= 18.0] *= 0.05  # left part saturates early, right part never
    opac[::97] = 0.001  # below 1/255: culled everywhere
    opac[::89] = 1.0    # the 0.999 (forward) / 0.99 (backward) alpha clamps
    C = sum(GROUPS)
    colors = rng.random((C, G, 3)).astype(np.float32)
    bg = rng.uniform(0.2, 1.0, 3).astype(np.float32)
    v_img = rng.standard_normal((C, H, W, 3)).astype(np.float32)

    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    i32 = dict(device=cuda, dtype=torch.int32)
    L = _lib.lib()
    st = _lib.stream_ptr(cuda)
    xys, depths, radii, conics, op, bgd = d(p["xys"]), d(p["depths"]), d(p["radii"]), d(p["conics"]), d(opac), d(bg)
    one = torch.ones(G, device=cuda)  # opac already holds opacity * compensation
    cols = d(colors)
    cap = n + 1000
    bins, order, gids = torch.empty(T, 2, **i32), torch.empty(T, **i32), torch.empty(cap, **i32)
    rec, n_dev, ovf = torch.empty(cap, 12, device=cuda), torch.empty(1, **i32), torch.zeros(1, **i32)
    ws = torch.empty(L.gb_bin_tiles_workspace_bytes(G, T, cap), dtype=torch.uint8, device=cuda)
    _lib.check(L.gb_bin_tiles_pack(G, xys.data_ptr(), depths.data_ptr(), radii.data_ptr(), conics.data_ptr(),
                                   cols.data_ptr(), op.data_ptr(), one.data_ptr(), H, W, bw, cap, bins.data_ptr(),
                                   order.data_ptr(), 0, gids.data_ptr(), rec.data_ptr(), n_dev.data_ptr(), ovf.data_ptr(),
                                   ws.data_ptr(), st), "bin_tiles_pack")
    sched = torch.full((L.gb_tile_schedule_ints(T),), -1, **i32)
    _lib.check(L.gb_tile_schedule(T, bins.data_ptr(), sched.data_ptr(), st), "tile_schedule")
    # the view's final_Ts / final_idx come from the 4-channel single-condition pass (rgb + depth), as in render_shared;
    # the oracle's backward runs on the same ones
    bg4 = d(np.append(bg, bg[0]))
    out4, Ts, fi = torch.empty(H, W, 4, device=cuda), torch.empty(H, W, device=cuda), torch.empty(H, W, **i32)
    _lib.check(L.gb_rasterize_packed_fwd(H, W, 4, bins.data_ptr(), order.data_ptr(), rec.data_ptr(), bg4.data_ptr(),
                                         out4.data_ptr(), Ts.data_ptr(), fi.data_ptr(), st), "rasterize_packed_fwd")
    wide = torch.empty(cap, 20, device=cuda)
    _lib.check(L.gb_records_widen(cap, n_dev.data_ptr(), rec.data_ptr(), wide.data_ptr(), st), "records_widen")
    torch.cuda.synchronize()
    assert int(ovf) == 0 and int(n_dev) == n
    assert np.array_equal(t2n(bins), bins_o) and np.array_equal(t2n(gids[:n]), gids_o), "binning != oracle"
    assert bool((sched[T:] == 0).all()), "draw counters of a fresh schedule"
    if case == "long_lists":
        assert (bins_o[:, 1] - bins_o[:, 0]).max() > 2000
    Ts_n, fi_n = t2n(Ts), t2n(fi)
    assert (Ts_n < 0.9).mean() > 0.02 and (Ts_n > 0.05).mean() > 0.02, "the background must show through in places"

    zero_a = np.zeros((H, W), np.float32)
    ref_img, ref_g, Ts_r = [], [], None
    for c in range(C):
        img, Ts_r, _ = orc.rasterize_fwd(H, W, bw, gids_o, bins_o, p["xys"], p["conics"], colors[c], opac, bg)
        ref_img.append(img)
        ref_g.append(orc.rasterize_bwd(H, W, bw, gids_o, bins_o, p["xys"], p["conics"], colors[c], opac, bg, Ts_n, fi_n,
                                       v_img[c], zero_a))
    runs = {}
    for sv, tile_order in ((0, order), (1, sched)):
        v12 = torch.zeros(G, 12, device=cuda)
        planes, grads = [], []
        c0 = 0
        for nk in GROUPS:
            _lib.check(L.gb_records_set_colors4(cap, n_dev.data_ptr(), gids.data_ptr(), cols[c0].data_ptr(), nk, G,
                                                wide.data_ptr(), st), "records_set_colors4")
            out = torch.full((4, H, W, 3), float("nan"), device=cuda)
            _lib.check(L.gb_rasterize_multi_fwd(H, W, bins.data_ptr(), tile_order.data_ptr(), sv, wide.data_ptr(),
                                                bgd.data_ptr(), out.data_ptr(), st), "rasterize_multi_fwd")
            torch.cuda.synchronize()
            if sv:
                assert bool((sched[T:] == 0).all()), "draw counters must be back to zero after the multi forward"
            vp = torch.zeros(4, H, W, 3, device=cuda)  # a partial group's missing planes carry no gradient (olat.py)
            vp[:nk] = d(v_img[c0:c0 + nk])
            v_xy, v_conic, v_op = (torch.zeros(G, 2, device=cuda), torch.zeros(G, 3, device=cuda),
                                   torch.zeros(G, device=cuda))
            v_col = torch.full((nk, G, 3), float("nan"), device=cuda)
            _lib.check(L.gb_rasterize_multi_bwd(H, W, gids.data_ptr(), bins.data_ptr(), tile_order.data_ptr(), sv,
                                                wide.data_ptr(), bgd.data_ptr(), Ts.data_ptr(), fi.data_ptr(),
                                                vp.data_ptr(), v_xy.data_ptr(), v_conic.data_ptr(), v12.data_ptr(),
                                                v_op.data_ptr(), st), "rasterize_multi_bwd")
            torch.cuda.synchronize()
            if sv:
                assert bool((sched[T:] == 0).all()), "draw counters must be back to zero after the multi backward"
            _lib.check(L.gb_colors12_unpack(G, nk, v12.data_ptr(), v_col.data_ptr(), st), "colors12_unpack")
            torch.cuda.synchronize()
            assert int(torch.count_nonzero(v12)) == 0, "colors12_unpack must clear the group buffer"
            planes.append(out)
            grads.append([t2n(v_xy), t2n(v_conic), t2n(v_col), t2n(v_op)])

            what = "%s sched=%d nk=%d" % (case, sv, nk)
            for k in range(4):
                # a missing condition is blended as black: T * background
                want = ref_img[c0 + k] if k < nk else Ts_r[..., None] * bg
                assert_close(t2n(out[k]), want, what="%s plane %d" % (what, k), **PIX)
            for k in range(nk):
                want = ref_g[c0 + k][2]
                assert_close(grads[-1][2][k], want, what="%s v_colors[%d]" % (what, k), **_gtol(want))
            for name, i in (("v_xy", 0), ("v_conic", 1), ("v_opacity", 3)):
                want = sum(ref_g[c][i] for c in range(c0, c0 + nk)).reshape(grads[-1][i].shape)
                assert_close(grads[-1][i], want, what="%s %s (sum over the group)" % (what, name), **_gtol(want))
            c0 += nk
        runs[sv] = planes, grads
    for g, nk in enumerate(GROUPS):
        assert torch.equal(runs[0][0][g], runs[1][0][g]), "group %d: pixels depend on the tile schedule" % g
        for name, x, y in zip(("v_xy", "v_conic", "v_colors", "v_opacity"), runs[1][1][g], runs[0][1][g]):
            assert_close(x, y, rtol=2e-5, atol=2e-5 * float(np.abs(y).max()),
                         what="group %d %s: schedule vs launch order" % (g, name))


# ---------------------------------------------------------------------------- 2. render_shared / render_views_shared
_RAGGED = (dict(G=2500, img_h=70, img_w=93, seed=11, cam=3), 15.0)
_CHAIN = {}


def _shared_inputs(C):
    s = small_scene(**_RAGGED[0])
    G, H, W = s["means3d"].shape[0], s["img_h"], s["img_w"]
    rng = np.random.default_rng(100 + C)
    opacity = s["opacity"].copy()
    opacity[::97] = 0.001  # culled everywhere
    opacity[::89] = 1.0    # the alpha clamps
    return dict(s=s, scales=(s["scales"] * np.float32(_RAGGED[1])).astype(np.float32), opacity=opacity,
                colors=rng.random((C, G, 3)).astype(np.float32), bg=np.array([0.1, 0.5, 0.9], np.float32),
                w_rgb=rng.standard_normal((C, H, W, 3)).astype(np.float32),
                w_dep=(1e-3 * rng.standard_normal((H, W))).astype(np.float32),
                w_alpha=rng.standard_normal((H, W)).astype(np.float32))


def _shared_oracle(orc, C):
    """the oracle chain does not depend on the capacity, the OLAT mode or the blend mode: once per C"""
    if C not in _CHAIN:
        x = _shared_inputs(C)
        s = x["s"]
        _CHAIN[C] = x, oracle_shared_view(orc, s["means3d"], x["scales"], s["quats"], x["opacity"], x["colors"], x["bg"],
                                          s["viewmat"], (s["fx"], s["fy"], s["cx"], s["cy"]), s["img_h"], s["img_w"],
                                          x["w_rgb"], x["w_dep"], x["w_alpha"])
    return _CHAIN[C]


def _check_shared(got_rgb, got_dep, got_alpha, grads, ref, what):
    C = ref["rgb"].shape[0]
    for c in range(C):
        assert_close(got_rgb[c], ref["rgb"][c], what="%s rgb[%d]" % (what, c), **PIX)
    assert_close(got_alpha, ref["alpha"], rtol=1e-4, atol=2e-6, frac=0.9995, what=what + " alpha")
    assert_close(got_dep, ref["depth_raw"], rtol=1e-4, atol=2e-2, frac=0.9995, what=what + " depth")  # depth ~ 1000 mm
    for name, want in ref["grads"].items():
        got = grads[name].reshape(want.shape)
        assert np.isfinite(got).all(), name
        if name == "colors":
            for c in range(C):
                assert_close(got[c], want[c], what="%s grad colors[%d]" % (what, c), **_gtol(want[c]))
        else:
            assert_close(got, want, what="%s grad %s" % (what, name), **_gtol(want))


@pytest.mark.parametrize("C", [2, 5, 32])
@pytest.mark.parametrize("capacity", [None, 1 << 17])
def test_render_shared_matches_oracle_chain(orc, cuda, C, capacity, olat_mode, blend_mode):
    from goliath_b200.gsplat.fused import check_overflow
    from goliath_b200.gsplat.olat import render_shared

    x, ref = _shared_oracle(orc, C)
    s = x["s"]
    H, W = s["img_h"], s["img_w"]
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    leaves = dict(means3d=d(s["means3d"]), scales=d(x["scales"]), quats=d(s["quats"]), opacity=d(x["opacity"]),
                  colors=d(x["colors"]))
    for v in leaves.values():
        v.requires_grad_()
    rgb, depth_raw, alpha, radii = render_shared(leaves["means3d"], leaves["scales"], 1.0, leaves["quats"],
                                                 d(s["viewmat"]), s["fx"], s["fy"], s["cx"], s["cy"], H, W,
                                                 leaves["opacity"], leaves["colors"], d(x["bg"]), 0.1, capacity)
    ((rgb * d(x["w_rgb"])).sum() + (depth_raw * d(x["w_dep"])).sum() + (alpha * d(x["w_alpha"])).sum()).backward()
    torch.cuda.synchronize()
    assert not check_overflow(cuda)
    assert rgb.shape == (C, H, W, 3) and (ref["alpha"] > 0.1).mean() > 0.02, "the scene must cover pixels"
    _check_shared(t2n(rgb), t2n(depth_raw), t2n(alpha), {k: t2n(v.grad) for k, v in leaves.items()}, ref,
                  "C=%d cap=%s %s %s" % (C, capacity, olat_mode, blend_mode))


def _views_inputs(orc):
    """3 ring cameras around the ragged scene, 6 conditions per view, and the oracle chain of every view (cached)"""
    from goliath_b200 import synthetic

    if "views" not in _CHAIN:
        V, C = 3, 6
        x = _shared_inputs(C)
        s = x["s"]
        G, H, W = s["means3d"].shape[0], s["img_h"], s["img_w"]
        cams = [synthetic.ring_camera(k, img_h=H, img_w=W) for k in (1, 4, 9)]
        for c in cams:
            c.update(fx=s["fx"], fy=s["fy"])  # small_scene's focal length: the head fills the small image
        rng = np.random.default_rng(77)
        cols = rng.random((V, C, G, 3)).astype(np.float32)
        w_rgb = rng.standard_normal((V, C, 3, H, W)).astype(np.float32)
        w_dep = (1e-3 * rng.standard_normal((V, 1, H, W))).astype(np.float32)
        inv_a = lambda a: (1.0 / np.clip(a, 0.05, 1.0)).astype(np.float32)
        refs = []
        for v in range(V):
            ref = oracle_shared_view(orc, s["means3d"], x["scales"], s["quats"], x["opacity"], cols[v], x["bg"],
                                     cams[v]["viewmat"].numpy(), (cams[v]["fx"], cams[v]["fy"], cams[v]["cx"],
                                                                  cams[v]["cy"]), H, W,
                                     np.ascontiguousarray(np.transpose(w_rgb[v], (0, 2, 3, 1))),
                                     v_depth=lambda a, v=v: w_dep[v, 0] * inv_a(a))
            ref["depth_raw"] = ref["depth_raw"] * inv_a(ref["alpha"])  # the depth the views return
            refs.append(ref)
        _CHAIN["views"] = x, cams, cols, w_rgb, w_dep, refs
    return _CHAIN["views"]


def test_render_views_shared_side_streams_match_oracle(orc, cuda, olat_mode, blend_mode):
    """V = 3 views under a capacity run on the side-stream pool, forward and backward; per-view geometry leaves, so
    every view's gradients are checked on their own.  depth = blended depth / alpha.clamp(0.05, 1), alpha detached."""
    from goliath_b200.gsplat.fused import check_overflow
    from goliath_b200.gsplat.olat import render_views_shared

    x, cams, cols, w_rgb, w_dep, refs = _views_inputs(orc)
    s = x["s"]
    V, H, W = len(cams), s["img_h"], s["img_w"]
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    geom = {k: d(np.repeat(a[None], V, 0)).requires_grad_() for k, a in
            (("primpos", s["means3d"]), ("primscale", x["scales"]), ("primqvec", s["quats"]), ("opacity", x["opacity"]))}
    colors = d(cols).requires_grad_()
    Rt = torch.stack([c["viewmat"] for c in cams]).to(cuda)
    intr = [(c["fx"], c["fy"], c["cx"], c["cy"]) for c in cams]
    rgb, alpha, depth = render_views_shared(W, H, Rt, geom, colors, intr, capacity=1 << 17, background=d(x["bg"]))
    ((rgb * d(w_rgb)).sum() + (depth * d(w_dep)).sum()).backward()
    torch.cuda.synchronize()
    assert not check_overflow(cuda) and not alpha.requires_grad
    for v in range(V):
        grads = dict(means3d=t2n(geom["primpos"].grad[v]), scales=t2n(geom["primscale"].grad[v]),
                     quats=t2n(geom["primqvec"].grad[v]), opacity=t2n(geom["opacity"].grad[v]),
                     colors=t2n(colors.grad[v]))
        _check_shared(np.transpose(t2n(rgb[v]), (0, 2, 3, 1)), t2n(depth[v, 0]), t2n(alpha[v, 0]), grads, refs[v],
                      "view %d %s %s" % (v, olat_mode, blend_mode))


@pytest.mark.parametrize("capacity", [None, 1 << 12])
def test_render_shared_without_intersections(cuda, capacity, olat_mode):
    """Every Gaussian behind the camera: the background everywhere, zero gradients, and alpha as render_fused gives it
    (capacity=None: the reference's alpha = 1 quirk, final_Ts = 0; a capacity: alpha = 0)."""
    from goliath_b200.gsplat.fused import render_fused
    from goliath_b200.gsplat.olat import render_shared

    G, H, W, C = 64, 40, 45, 6
    gen = torch.Generator().manual_seed(1)
    V = torch.eye(4, device=cuda)[:3].contiguous()
    means = torch.randn(G, 3, generator=gen).to(cuda)
    means[:, 2] = -5.0 - means[:, 2].abs()
    scales = torch.full((G, 3), 0.1, device=cuda)
    quats = torch.tensor([[1.0, 0, 0, 0]] * G, device=cuda)
    opacity = torch.rand(G, 1, generator=gen).to(cuda)
    cols = torch.rand(C, G, 3, generator=gen).to(cuda)
    bg = torch.tensor([0.25, 0.5, 0.75], device=cuda)
    cam = (V, 50.0, 50.0, 22.0, 20.0, H, W)
    leaves = [t.clone().requires_grad_() for t in (means, scales, quats, opacity, cols)]
    rgb, depth_raw, alpha, radii = render_shared(leaves[0], leaves[1], 1.0, leaves[2], *cam, leaves[3], leaves[4], bg,
                                                 0.1, capacity)
    out4, alpha1, _ = render_fused(means, scales, 1.0, quats, *cam, opacity, cols[0], bg, 0.1, capacity)
    assert int(radii.sum()) == 0
    assert torch.equal(rgb, bg.expand(C, H, W, 3))
    assert torch.equal(depth_raw, out4[..., 3]) and torch.equal(alpha, alpha1)
    assert bool((alpha == (1.0 if capacity is None else 0.0)).all())
    (rgb.sum() + depth_raw.sum() + alpha.sum()).backward()
    for t in leaves:
        assert t.grad is not None and int(torch.count_nonzero(t.grad)) == 0


# ----------------------------------------------------------------------------------------------- 3. the bench step
def test_benchmarked_olat_step_matches_oracle(orc, cuda):
    """bench.py's own OlatWorkload.compute with two views: 300 000 Gaussians x 32 OLAT conditions at 1024x667 (the
    bench's capacity, default binning, default blend mode, four conditions per pass ending in a group of three)."""
    import bench
    from goliath_b200 import synthetic
    from goliath_b200.gsplat.fused import check_overflow

    class TwoViews(bench.OlatWorkload):
        N_VIEWS = 2

    G = 300_000
    wl = TwoViews(types.SimpleNamespace(gaussians=G), 0, 1, cuda)
    packed = bench.packed_scene(G)
    (rgb, alpha, depth), grad = wl.compute(packed.to(cuda))
    torch.cuda.synchronize()
    assert not check_overflow(cuda)
    V, C, H, W = 2, wl.N_COND, bench.H, bench.W
    assert rgb.shape == (V, C, 3, H, W) and alpha.shape == (V, 1, H, W) and depth.shape == (V, 1, H, W)
    got_grads = {k: t2n(v) for k, v in bench.unpack(grad).items()}
    alpha, depth = t2n(alpha), t2n(depth)

    u = {k: np.ascontiguousarray(v) for k, v in bench.unpack(packed.numpy()).items()}
    li = {k: v.numpy() for k, v in synthetic.lights(C).items()}
    cams = [dict(Rt=t2n(wl.Rt[v]), intr=wl.intr[v]) for v in range(V)]
    ref = oracle_olat_step(orc, u, cams, li, H, W)
    for v in range(V):
        assert ref["n_isect"][v] > 2 * G, "the scene must be the dense bench scene"
        for c in range(C):
            assert_close(t2n(rgb[v, c]).transpose(1, 2, 0), ref["rgb"][v, c], what="view %d rgb[%d]" % (v, c), **PIX)
        assert_close(alpha[v, 0], ref["alpha"][v], rtol=1e-4, atol=2e-6, frac=0.9995, what="view %d alpha" % v)
        assert_close(depth[v, 0], ref["depth"][v], rtol=1e-4, atol=2e-2, frac=0.9995, what="view %d depth" % v)
    for k, want in ref["grads"].items():
        got = got_grads[k].reshape(want.shape)
        assert np.isfinite(got).all(), k
        assert_close(got, want, what="grad " + k, **_gtol(want))
