"""The ranked blend pair that hands per-warp hit lists from the forward to the backward
(gb_rasterize_ranked_fwd_lists / gb_rasterize_ranked_bwd_lists, csrc/splat_blend_mom.cu):

- the forward's pixels, final_Ts and final_idx are those of gb_rasterize_ranked_fwd bit for bit;
- each pixel warp's stored list is its footprint hits (a numpy restatement of the cull, records within a rounding
  margin of the cull threshold left out of the comparison) in ascending sorted index, and its count ends at the last
  hit any pixel of the warp blended;
- the backward's gradients are gb_rasterize_ranked_bwd's up to the order of the atomic adds, eagerly, when run twice
  on the same lists, and in a CUDA graph.

Scenes: oracle-style head scenes (tests/util.small_scene), and screen-space scenes that put exactly 1, 127, 128, 129
and 6000 entries in single tiles, saturate pixels in the middle of a 128-record stage, fill the ragged bottom tile row
(warps with no pixel inside the image) and leave most tiles empty."""
import numpy as np
import pytest
import torch

from util import assert_close, small_scene, t2n

pytestmark = pytest.mark.gpu

PIX_WARPS = 8


def _project(s, dev, mult):
    from goliath_b200.gsplat import project_gaussians

    t = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else v) for k, v in s.items()}
    xys, depths, radii, conics, comp, _, _ = project_gaussians(
        t["means3d"], t["scales"] * mult, 1.0, t["quats"], t["viewmat"], s["fx"], s["fy"], s["cx"], s["cy"],
        s["img_h"], s["img_w"], 16, 0.1)
    return dict(xys=xys, depths=depths, radii=radii, conics=conics, comp=comp,
                colors=t["colors"].contiguous(), opacity=t["opacity"].contiguous(), H=s["img_h"], W=s["img_w"])


def _screen_scene(dev):
    """Isotropic screen-space Gaussians: per group (tile column, tile row, count, sigma, opacity range).  sigma 1.3
    with radius 4 around a point at least 4 px inside the tile keeps a Gaussian in its one tile, so those tiles hold
    exactly `count` entries; the wide opaque group saturates its pixels after a few dozen of its 300 hits."""
    rng = np.random.default_rng(5)
    H, W = 70, 93  # 5 x 6 tiles; the bottom row has 6 pixel rows, the right column 13 pixel columns
    groups = [(0, 0, 1, 1.3, (0.2, 0.9)), (1, 0, 127, 1.3, (0.05, 0.9)), (2, 0, 128, 1.3, (0.05, 0.9)),
              (3, 0, 129, 1.3, (0.05, 0.9)), (0, 1, 6000, 1.3, (0.02, 0.6)), (2, 4, 200, 1.3, (0.05, 0.9)),
              (5, 4, 150, 1.3, (0.05, 0.9)), (3, 2, 300, 4.0, (0.4, 0.9))]
    xy, sig, op = [], [], []
    for tx, ty, n, s, (olo, ohi) in groups:
        lo_y, hi_y = ty * 16 + 4, min(ty * 16 + 12, H - 1)
        lo_x, hi_x = tx * 16 + 4, min(tx * 16 + 12, W - 1)
        xy.append(np.stack([rng.uniform(lo_x, hi_x, n), rng.uniform(lo_y, hi_y, n)], 1))
        sig.append(np.full(n, s))
        op.append(rng.uniform(olo, ohi, n))
    xy, sig, op = np.concatenate(xy), np.concatenate(sig), np.concatenate(op)
    G = len(xy)
    f = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
    inv = 1.0 / (sig * sig)
    return dict(xys=f(xy), depths=f(rng.permutation(G) * 0.01 + 1.0),
                radii=f(np.where(sig > 2, 12, 4), torch.int32), conics=f(np.stack([inv, 0 * inv, inv], 1)),
                comp=f(np.ones(G)), colors=f(rng.uniform(0, 1, (G, 3))), opacity=f(op[:, None]), H=H, W=W)


SCENES = {
    "head_dense96": lambda dev: _project(small_scene(G=3000, img_h=96, img_w=80), dev, 12.0),
    "head_ragged": lambda dev: _project(small_scene(G=2500, img_h=70, img_w=93, seed=11, cam=3), dev, 15.0),
    "head_big": lambda dev: _project(small_scene(G=150_000, img_h=512, img_w=384, seed=13), dev, 6.0),
    "screen_tiles": _screen_scene,
}


def _bin(sc, dev):
    from goliath_b200 import _lib
    from goliath_b200.gsplat import utils as gu

    L = _lib.lib()
    H, W = sc["H"], sc["W"]
    G = sc["xys"].shape[0]
    tb = gu._tile_bounds(H, W, 16)
    T = tb[0] * tb[1]
    i32 = dict(dtype=torch.int32, device=dev)
    r = sc["radii"].long()
    cap = int(((2 * r // 16 + 2) ** 2 * (r > 0)).sum()) + 1000  # at least the tiles each bounding square touches
    ws = torch.empty(L.gb_bin_tiles_workspace_bytes(G, T, cap), dtype=torch.uint8, device=dev)
    bins, order = torch.empty(T, 2, **i32), torch.empty(T, **i32)
    ranks, rbr, r2g = torch.empty(cap, **i32), torch.empty(G, 12, device=dev), torch.empty(G, **i32)
    n_out, ovf = torch.zeros(1, **i32), torch.zeros(1, **i32)
    _lib.check(L.gb_bin_tiles_ranked(G, *(_lib.ptr(sc[k]) for k in ("xys", "depths", "radii", "conics", "colors",
                                                                       "opacity", "comp")),
                                     H, W, 16, cap, bins.data_ptr(), order.data_ptr(), 0, ranks.data_ptr(),
                                     rbr.data_ptr(), r2g.data_ptr(), n_out.data_ptr(), ovf.data_ptr(), ws.data_ptr(),
                                     None, _lib.stream_ptr(dev)), "bin_tiles_ranked")
    torch.cuda.synchronize()
    assert int(ovf) == 0
    return dict(bins=bins, order=order, ranks=ranks, rbr=rbr, r2g=r2g, cap=cap, T=T, G=G, n=int(n_out))


class Blend:
    """Both ranked pairs on one binning, through the C ABI."""

    def __init__(self, sc, b, C, dev, seed=0):
        from goliath_b200 import _lib

        self.L, self.st, self.sc, self.b, self.C, self.dev = _lib.lib(), _lib.stream_ptr(dev), sc, b, C, dev
        H, W = sc["H"], sc["W"]
        g = torch.Generator(device="cpu").manual_seed(seed)
        self.bg = torch.rand(C, generator=g).to(dev)
        self.v_out = torch.randn(H, W, C, generator=g).to(dev)
        self.v_alpha = torch.randn(H, W, generator=g).to(dev)
        i32 = dict(dtype=torch.int32, device=dev)
        self.hit_list = torch.full((8 * b["cap"],), -7, **i32)
        self.hit_count = torch.full((16 * b["T"] + 2,), -7, **i32)

    def _outs(self):
        H, W, i32 = self.sc["H"], self.sc["W"], dict(dtype=torch.int32, device=self.dev)
        return torch.empty(H, W, self.C, device=self.dev), torch.empty(H, W, device=self.dev), torch.empty(H, W, **i32)

    def _grads(self):
        G, dev = self.b["G"], self.dev
        return (torch.zeros(G, 2, device=dev), torch.zeros(G, 3, device=dev), torch.zeros(G, self.C, device=dev),
                torch.zeros(G, 1, device=dev))

    def fwd(self, lists):
        b, H, W = self.b, self.sc["H"], self.sc["W"]
        out, Ts, fi = self._outs()
        args = [H, W, self.C, b["bins"].data_ptr(), b["order"].data_ptr(), b["ranks"].data_ptr(), b["rbr"].data_ptr(),
                self.bg.data_ptr(), out.data_ptr(), Ts.data_ptr(), fi.data_ptr()]
        if lists:
            rc = self.L.gb_rasterize_ranked_fwd_lists(*args, self.hit_list.data_ptr(), self.hit_count.data_ptr(),
                                                      self.st)
        else:
            rc = self.L.gb_rasterize_ranked_fwd(*args, self.st)
        assert rc == 0
        return out, Ts, fi

    def bwd(self, lists, Ts, fi, grads=None):
        b, H, W = self.b, self.sc["H"], self.sc["W"]
        grads = self._grads() if grads is None else grads
        tail = [self.bg.data_ptr(), Ts.data_ptr(), fi.data_ptr(), self.v_out.data_ptr(), self.v_alpha.data_ptr()]
        tail += [g.data_ptr() for g in grads]
        if lists:
            rc = self.L.gb_rasterize_ranked_bwd_lists(H, W, self.C, b["ranks"].data_ptr(), b["bins"].data_ptr(),
                                                      self.hit_list.data_ptr(), self.hit_count.data_ptr(),
                                                      b["rbr"].data_ptr(), *tail, self.st)
        else:
            rc = self.L.gb_rasterize_ranked_bwd(H, W, self.C, b["r2g"].data_ptr(), b["ranks"].data_ptr(),
                                                b["bins"].data_ptr(), b["order"].data_ptr(), b["rbr"].data_ptr(), *tail,
                                                self.st)
        assert rc == 0
        return grads


def _cpu_cull(rec, fx0, fx1, fy0, fy1):
    """footprint_hit of csrc/splat_blend_mom.cu in numpy for records `rec` [n,12] and one warp rectangle of pixel
    centres.  Returns (hit, unsure): `unsure` marks records within a rounding margin of the threshold, where the
    kernel's rcp.approx / lg2.approx may decide either way."""
    x, y, ex, ey = rec[:, 0], rec[:, 1], rec[:, 2], rec[:, 3]
    box = (x + ex >= fx0) & (x - ex <= fx1) & (y + ey >= fy0) & (y - ey <= fy1)  # fp32, as the kernel
    never = ex > np.float32(1e30)
    d = rec.astype(np.float64)
    x, y, A, B, Cc, o = d[:, 0], d[:, 1], d[:, 4], d[:, 5], d[:, 6], d[:, 7]
    dxlo, dxhi, dylo, dyhi = x - fx1, x - fx0, y - fy1, y - fy0
    ex0, ey0 = np.clip(0.0, dxlo, dxhi), np.clip(0.0, dylo, dyhi)
    with np.errstate(all="ignore"):
        dy1 = np.clip(-B * ex0 / Cc, dylo, dyhi)
        dx2 = np.clip(-B * ey0 / A, dxlo, dxhi)
        f1 = 0.5 * (A * ex0 * ex0 + Cc * dy1 * dy1) + B * ex0 * dy1
        f2 = 0.5 * (A * dx2 * dx2 + Cc * ey0 * ey0) + B * dx2 * ey0
        s = np.log(255.0 * o)
        thr = s + 2e-3 + 1e-4 * np.abs(s)
        m = np.minimum(f1, f2)
        hit = box & (never | (m <= thr))
        unsure = box & ~never & ~(np.abs(m - thr) > 1e-3 * (1.0 + np.abs(thr)))
    return hit, unsure


def _warp_rect(tile, w, tbx):
    ty, tx = divmod(tile, tbx)
    wx0, wy0 = tx * 16 + (w & 1) * 8, ty * 16 + (w >> 1) * 4
    return wx0, wy0, (np.float32(wx0 + 0.5), np.float32(wx0 + 7.5), np.float32(wy0 + 0.5), np.float32(wy0 + 3.5))


@pytest.fixture(scope="module", params=list(SCENES))
def scene(request, cuda):
    torch.manual_seed(0)
    sc = SCENES[request.param](cuda)
    return request.param, sc, _bin(sc, cuda)


def test_forward_identical_and_lists_match_cpu_cull(cuda, scene):
    name, sc, b = scene
    H, W = sc["H"], sc["W"]
    bl = Blend(sc, b, 4, cuda)
    ref = [t2n(t) for t in bl.fwd(lists=False)]
    got = [t2n(t) for t in bl.fwd(lists=True)]
    torch.cuda.synchronize()
    for r, g, what in zip(ref, got, ("out", "final_Ts", "final_idx")):
        assert np.array_equal(r.view(np.int32), g.view(np.int32)), what
    _, Ts, fi = got
    bins, ranks, rbr = t2n(b["bins"]), t2n(b["ranks"]), t2n(b["rbr"])
    hl, hc = t2n(bl.hit_list), t2n(bl.hit_count)
    tbx = (W + 15) // 16
    assert hc[8 * b["T"]] == 0  # the backward's draw counter
    lens = bins[:, 1] - bins[:, 0]
    checked = saturated_mid_stage = ragged_empty = 0
    for tile in range(b["T"]):
        x0, x1 = bins[tile]
        if x1 <= x0:
            assert (hc[8 * tile:8 * tile + 8] == 0).all()
            continue
        rec = rbr[ranks[x0:x1]]
        for w in range(PIX_WARPS):
            wx0, wy0, rect = _warp_rect(tile, w, tbx)
            cnt = int(hc[8 * tile + w])
            assert 0 <= cnt <= x1 - x0
            pix = fi[wy0:wy0 + 4, wx0:wx0 + 8]
            if pix.size == 0:  # warp entirely below / right of the image
                assert cnt == 0
                ragged_empty += 1
                continue
            wbf = int(pix.max())
            seg = hl[8 * x0 + w * (x1 - x0):][:cnt]
            assert (np.diff(seg) > 0).all() and (cnt == 0 or (seg[0] >= x0 and seg[-1] <= wbf))
            hit, unsure = _cpu_cull(rec, *rect)
            idx = np.arange(x0, x1)
            need = idx <= wbf
            if cnt > 0:
                assert seg[-1] == wbf, (tile, w, cnt)  # the count ends at the last blended hit
            else:
                assert not (need & hit & ~unsure).any(), (tile, w)
            exp = set(idx[need & hit & ~unsure].tolist())
            mine = set(seg.tolist()) - set(idx[unsure].tolist())
            assert mine == exp, (tile, w, sorted(mine ^ exp)[:10])
            checked += 1
            Tw = Ts[wy0:wy0 + 4, wx0:wx0 + 8]
            if (Tw < 1e-3).all() and wbf - x0 < 100 and x1 - x0 > 128:
                saturated_mid_stage += 1
    assert checked > 0
    if name == "screen_tiles":
        assert sorted(set(lens.tolist()) & {1, 127, 128, 129}) == [1, 127, 128, 129] and lens.max() > 5120
        assert saturated_mid_stage > 0 and ragged_empty > 0 and (lens == 0).sum() > 0


@pytest.mark.parametrize("channels", [3, 4])
def test_backward_matches_ranked_backward(cuda, scene, channels):
    _, sc, b = scene
    bl = Blend(sc, b, channels, cuda, seed=channels)
    _, Ts, fi = bl.fwd(lists=True)
    ref = [t2n(g) for g in bl.bwd(False, Ts, fi)]
    got = [t2n(g) for g in bl.bwd(True, Ts, fi)]
    again = [t2n(g) for g in bl.bwd(True, Ts, fi)]  # the draw counter is back at zero: same walk again
    torch.cuda.synchronize()
    hc, T8 = t2n(bl.hit_count), 8 * b["T"]
    assert hc[T8] == 0  # draw counter back at zero
    # the work items: every (tile, warp) with hits once, in descending order of their 16-hit chunk count
    n_work, items = int(hc[T8 + 1]), hc[T8 + 2:T8 + 2 + int(hc[T8 + 1])]
    assert sorted(items.tolist()) == np.nonzero(hc[:T8] > 0)[0].tolist() and n_work > 0
    chunks = np.minimum((hc[items] + 15) // 16, 63)
    assert (np.diff(chunks) <= 0).all()
    for g, g2, r, name in zip(got, again, ref, ("v_xy", "v_conic", "v_colors", "v_opacity")):
        assert np.abs(r).max() > 0, name
        assert_close(g, r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()), frac=0.9999, what=name)
        assert_close(g2, r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()), frac=0.9999, what=name + " (again)")


def test_graph_replay_matches_eager(cuda, scene):
    _, sc, b = scene
    bl = Blend(sc, b, 4, cuda, seed=11)
    out_e, Ts_e, fi_e = bl.fwd(lists=True)
    g_e = [t2n(g) for g in bl.bwd(True, Ts_e, fi_e)]
    out_e, Ts_e, fi_e = t2n(out_e), t2n(Ts_e), t2n(fi_e)
    bl.hit_list.fill_(-7)
    bl.hit_count.fill_(-7)
    grads = bl._grads()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    from goliath_b200 import _lib

    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            bl.st = _lib.stream_ptr(cuda)
            for g in grads:
                g.zero_()
            out, Ts, fi = bl.fwd(lists=True)
            bl.bwd(True, Ts, fi, grads)
    torch.cuda.current_stream().wait_stream(side)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(t2n(out).view(np.int32), out_e.view(np.int32))
        assert np.array_equal(t2n(Ts).view(np.int32), Ts_e.view(np.int32)) and np.array_equal(t2n(fi), fi_e)
        for g, r, name in zip(grads, g_e, ("v_xy", "v_conic", "v_colors", "v_opacity")):
            assert_close(t2n(g), r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()), frac=0.9999, what=name)
