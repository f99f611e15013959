"""The forward that sorts each tile before it blends it (gb_bin_tiles_buckets + gb_rasterize_ranked_fwd_sort_lists,
csrc/splat_blend_mom.cu) against the two-kernel pair it replaces (gb_bin_tiles_ranked + gb_rasterize_ranked_fwd_lists):

- the sorted ids, pixels, final_Ts, final_idx, hit lists and hit counts are identical bit for bit, and so are the bins
  and the by-id records of the binning;
- the backward on its lists gives the same gradients up to the order of the atomic adds;
- a CUDA graph of the pair replays to the eager result.

Scenes: the oracle-style and screen-space scenes of test_blend_hitlists_gpu.py, single tiles of every length around
a warp, the 288-thread CTA, the sort's shared-memory capacity (4320 entries in the forward) and the binning's 5120,
equal-depth runs around the tie fix-up's limit, the benchmarked 300k head from all 16 ring cameras, and the
2^20-Gaussian head whose longest tiles take the chunked path inside the forward."""
import numpy as np
import pytest
import torch

from test_bin_tiles_ties_gpu import TIE_RUN, _runs, _tile_scene
from test_blend_hitlists_gpu import SCENES
from util import assert_close, t2n

pytestmark = pytest.mark.gpu

FWD_THREADS, FWD_CAP = 288, 288 * 15


def _with_records(cuda, xys, depths, radii, H, W, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    G = xys.shape[0]
    f = lambda t: t.to(cuda).contiguous()
    return dict(xys=xys, depths=depths, radii=radii, conics=f(torch.tensor([[0.5, 0.0, 0.5]]).repeat(G, 1)),
                comp=f(torch.ones(G)), colors=f(torch.rand(G, 3, generator=g)),
                opacity=f(torch.rand(G, 1, generator=g) * 0.5 + 0.05), H=H, W=W)


def _run(sc, dev, fused, C=4, seed=0):
    """Binning + hit-list forward, either pair.  Returns every output as a dict of tensors."""
    from goliath_b200 import _lib
    from goliath_b200.gsplat import utils as gu

    L, st = _lib.lib(), _lib.stream_ptr(dev)
    H, W = sc["H"], sc["W"]
    G = sc["xys"].shape[0]
    tb = gu._tile_bounds(H, W, 16)
    T = tb[0] * tb[1]
    i32 = dict(dtype=torch.int32, device=dev)
    r = sc["radii"].long()
    cap = int(((2 * r // 16 + 2) ** 2 * (r > 0)).sum()) + 1000
    ws = torch.empty(L.gb_bin_tiles_workspace_bytes(G, T, cap), dtype=torch.uint8, device=dev)
    o = dict(bins=torch.empty(T, 2, **i32), order=torch.empty(T, **i32), ranks=torch.empty(cap, **i32),
             rbr=torch.empty(G, 12, device=dev), r2g=torch.empty(G, **i32), n=torch.zeros(1, **i32),
             hit_list=torch.full((8 * cap,), -7, **i32), hit_count=torch.full((16 * T + 2,), -7, **i32))
    ovf = torch.zeros(1, **i32)
    ins = [_lib.ptr(sc[k]) for k in ("xys", "depths", "radii", "conics", "colors", "opacity", "comp")]
    head = [G, *ins, H, W, 16, cap, o["bins"].data_ptr(), o["order"].data_ptr()]
    tail = [o["n"].data_ptr(), ovf.data_ptr(), ws.data_ptr(), None, st]
    if fused:
        bucket = torch.empty(cap, **i32)
        _lib.check(L.gb_bin_tiles_buckets(*head, o["ranks"].data_ptr(), bucket.data_ptr(), o["rbr"].data_ptr(),
                                          o["r2g"].data_ptr(), *tail), "bin_tiles_buckets")
    else:
        _lib.check(L.gb_bin_tiles_ranked(*head, 0, o["ranks"].data_ptr(), o["rbr"].data_ptr(), o["r2g"].data_ptr(),
                                         *tail), "bin_tiles_ranked")
    g = torch.Generator(device="cpu").manual_seed(seed)
    bg = torch.rand(C, generator=g).to(dev)
    o.update(out=torch.empty(H, W, C, device=dev), Ts=torch.empty(H, W, device=dev), fi=torch.empty(H, W, **i32))
    px = [o[k].data_ptr() for k in ("out", "Ts", "fi", "hit_list", "hit_count")]
    if fused:
        rc = L.gb_rasterize_ranked_fwd_sort_lists(H, W, C, o["bins"].data_ptr(), o["order"].data_ptr(),
                                                  _lib.ptr(sc["depths"]), bucket.data_ptr(), o["ranks"].data_ptr(),
                                                  o["rbr"].data_ptr(), bg.data_ptr(), *px, st)
    else:
        rc = L.gb_rasterize_ranked_fwd_lists(H, W, C, o["bins"].data_ptr(), o["order"].data_ptr(),
                                             o["ranks"].data_ptr(), o["rbr"].data_ptr(), bg.data_ptr(), *px, st)
    assert rc == 0
    torch.cuda.synchronize()
    assert int(ovf) == 0
    o.update(bg=bg, cap=cap, T=T, G=G, C=C, H=H, W=W)
    return o


def _bwd(o, dev, seed=1):
    from goliath_b200 import _lib

    g = torch.Generator(device="cpu").manual_seed(seed)
    H, W, C, G = o["H"], o["W"], o["C"], o["G"]
    v_out, v_alpha = torch.randn(H, W, C, generator=g).to(dev), torch.randn(H, W, generator=g).to(dev)
    grads = (torch.zeros(G, 2, device=dev), torch.zeros(G, 3, device=dev), torch.zeros(G, C, device=dev),
             torch.zeros(G, 1, device=dev))
    _lib.check(_lib.lib().gb_rasterize_ranked_bwd_lists(
        H, W, C, o["ranks"].data_ptr(), o["bins"].data_ptr(), o["hit_list"].data_ptr(), o["hit_count"].data_ptr(),
        o["rbr"].data_ptr(), o["bg"].data_ptr(), o["Ts"].data_ptr(), o["fi"].data_ptr(), v_out.data_ptr(),
        v_alpha.data_ptr(), *[t.data_ptr() for t in grads], _lib.stream_ptr(dev)), "bwd_lists")
    torch.cuda.synchronize()
    return [t2n(t) for t in grads]


def _check_identical(sc, dev, C=4, seed=0):
    ref = _run(sc, dev, fused=False, C=C, seed=seed)
    got = _run(sc, dev, fused=True, C=C, seed=seed)
    n = int(ref["n"])
    assert int(got["n"]) == n
    for k in ("bins", "r2g", "fi", "hit_list"):
        assert torch.equal(got[k], ref[k]), k
    # the launch order only groups tiles by length: within a group the order may differ from run to run
    assert torch.equal(torch.sort(got["order"])[0], torch.sort(ref["order"])[0]), "order"
    assert torch.equal(got["ranks"][:n], ref["ranks"][:n]), "ranks"
    for k in ("rbr", "out", "Ts"):
        assert torch.equal(got[k].view(torch.int32), ref[k].view(torch.int32)), k
    T8 = 8 * ref["T"]
    assert torch.equal(got["hit_count"][:T8 + 1], ref["hit_count"][:T8 + 1]), "hit_count"
    return ref, got


@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("channels", [3, 4])
def test_scenes_identical_and_same_gradients(cuda, name, channels):
    torch.manual_seed(0)
    sc = SCENES[name](cuda)
    ref, got = _check_identical(sc, cuda, C=channels, seed=channels)
    for g, r, what in zip(_bwd(got, cuda), _bwd(ref, cuda), ("v_xy", "v_conic", "v_colors", "v_opacity")):
        assert np.abs(r).max() > 0, what
        assert_close(g, r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()), frac=0.9999, what=what)


LENGTHS = [1, 31, 32, 33, 255, 256, 257, FWD_THREADS - 1, FWD_THREADS, FWD_THREADS + 1, 511, 512, 513, FWD_CAP - 1,
           FWD_CAP, FWD_CAP + 1, 5119, 5120, 5121]


@pytest.mark.parametrize("depth", ["distinct", "ties"])
def test_tile_lengths(cuda, depth):
    """Tiles of every length around a warp, the forward's CTA, its shared-memory capacity (longer tiles take the
    chunked path) and the binning's 5120."""
    rng = np.random.default_rng(7)
    if depth == "distinct":
        ranks = [rng.permutation(n) for n in LENGTHS]
    else:
        ranks = [rng.integers(0, max(1, n // 2), size=n) for n in LENGTHS]
    xys, depths, radii, _, H, W = _tile_scene(cuda, ranks, seed=17)
    ref, _ = _check_identical(_with_records(cuda, xys, depths, radii, H, W, 3), cuda)
    lengths = t2n(ref["bins"][:, 1] - ref["bins"][:, 0])
    assert sorted(lengths[lengths > 0].tolist()) == sorted(LENGTHS)


def test_equal_depth_runs(cuda):
    """Runs of 2, TIE_RUN and TIE_RUN + 1 equal depths (the last re-sorts on the full key), and whole tiles of one
    depth, in the shared-memory and the chunked path of the forward's sort."""
    R = TIE_RUN
    n = 1700  # 6 items per thread over 288 threads
    tiles = [
        _runs(n, [(0, 2), (30, 2), (63, 2), (191, 2), (287, R), (500, R), (575, 2), (1023, R), (n - 2, 2)]),
        _runs(n, [(0, R), (120, R + 1), (511, 2), (n - R, R)]),
        _runs(FWD_CAP, [(31, R), (4000, 2), (FWD_CAP - R, R)]),
        _runs(FWD_CAP + 1, [(0, R + 1), (FWD_CAP - 2, 3)]),
        _runs(FWD_THREADS + 1, [(FWD_THREADS - 1, 2)]),
        np.zeros(2, np.int64),
        np.zeros(R, np.int64),
        np.zeros(R + 1, np.int64),
        np.zeros(FWD_CAP, np.int64),
        np.zeros(5000, np.int64),
    ]
    xys, depths, radii, _, H, W = _tile_scene(cuda, tiles, seed=23)
    ref, _ = _check_identical(_with_records(cuda, xys, depths, radii, H, W, 4), cuda)
    lengths = t2n(ref["bins"][:, 1] - ref["bins"][:, 0])
    assert lengths[:len(tiles)].tolist() == [len(r) for r in tiles]


def _bench_view(cuda, G, cam):
    import bench
    from goliath_b200 import synthetic
    from goliath_b200.gsplat import project_gaussians

    u = bench.unpack(bench.packed_scene(G).to(cuda))
    c = synthetic.ring_camera(cam, img_h=bench.H, img_w=bench.W)
    xys, depths, radii, conics, comp, _, _ = project_gaussians(
        u["primpos"].contiguous(), u["primscale"].contiguous(), 1.0, u["primqvec"].contiguous(),
        c["viewmat"].to(cuda), c["fx"], c["fy"], c["cx"], c["cy"], bench.H, bench.W, bench.BW, 0.1)
    g = torch.Generator(device="cpu").manual_seed(cam)
    return dict(xys=xys, depths=depths, radii=radii, conics=conics, comp=comp,
                colors=torch.rand(G, 3, generator=g).to(cuda), opacity=torch.rand(G, 1, generator=g).to(cuda),
                H=bench.H, W=bench.W)


def test_bench_ring_cameras(cuda):
    """The benchmarked scene (300k Gaussians, 1024x667) from all 16 ring cameras: every tile in shared memory."""
    for cam in range(16):
        ref, _ = _check_identical(_bench_view(cuda, 300_000, cam), cuda, seed=cam)
        assert int((ref["bins"][:, 1] - ref["bins"][:, 0]).max()) <= FWD_CAP


def test_large_head_long_tiles(cuda):
    """2^20 Gaussians: hundreds of tiles longer than the forward's shared-memory sort, sorted by the chunked path."""
    sc = _bench_view(cuda, 1 << 20, 2)
    ref, got = _check_identical(sc, cuda, seed=5)
    assert int(((ref["bins"][:, 1] - ref["bins"][:, 0]) > FWD_CAP).sum()) > 100
    for g, r, what in zip(_bwd(got, cuda), _bwd(ref, cuda), ("v_xy", "v_conic", "v_colors", "v_opacity")):
        assert_close(g, r, rtol=1e-4, atol=1e-5 * float(np.abs(r).max()), frac=0.9999, what=what)


def test_graph_replay_matches_eager(cuda):
    from goliath_b200 import _lib

    sc = _bench_view(cuda, 300_000, 0)
    eager = _run(sc, cuda, fused=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    L = _lib.lib()
    o, i32 = dict(eager), dict(dtype=torch.int32, device=cuda)
    bucket = torch.empty(o["cap"], **i32)
    for k in ("ranks", "out", "Ts", "fi", "hit_list", "hit_count", "bins", "order", "rbr", "r2g", "n"):
        o[k] = torch.full_like(eager[k], -7)  # -7: the fill of eager's hit_list, whose unwritten slots are compared
    ws = torch.empty(L.gb_bin_tiles_workspace_bytes(o["G"], o["T"], o["cap"]), dtype=torch.uint8, device=cuda)
    ovf = torch.zeros(1, **i32)
    ins = [_lib.ptr(sc[k]) for k in ("xys", "depths", "radii", "conics", "colors", "opacity", "comp")]
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            st = _lib.stream_ptr(cuda)
            _lib.check(L.gb_bin_tiles_buckets(o["G"], *ins, o["H"], o["W"], 16, o["cap"], o["bins"].data_ptr(),
                                              o["order"].data_ptr(), o["ranks"].data_ptr(), bucket.data_ptr(),
                                              o["rbr"].data_ptr(), o["r2g"].data_ptr(), o["n"].data_ptr(),
                                              ovf.data_ptr(), ws.data_ptr(), None, st), "bin_tiles_buckets")
            _lib.check(L.gb_rasterize_ranked_fwd_sort_lists(
                o["H"], o["W"], 4, o["bins"].data_ptr(), o["order"].data_ptr(), _lib.ptr(sc["depths"]),
                bucket.data_ptr(), o["ranks"].data_ptr(), o["rbr"].data_ptr(), eager["bg"].data_ptr(),
                *[o[k].data_ptr() for k in ("out", "Ts", "fi", "hit_list", "hit_count")], st), "fwd_sort_lists")
    torch.cuda.current_stream().wait_stream(side)
    n = int(eager["n"])
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(o["ranks"][:n], eager["ranks"][:n])
        for k in ("fi", "hit_list", "bins"):
            assert torch.equal(o[k], eager[k]), k
        for k in ("out", "Ts"):
            assert torch.equal(o[k].view(torch.int32), eager[k].view(torch.int32)), k
