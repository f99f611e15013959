"""The per-tile sort of the bucket binning (csrc/splat_bin_tiles.cu, tile_sort_kernel) at its edges: the items-per-
thread split of the tile over the CTA's warps, the fix-up of equal-depth runs after the depth-only digit passes, and
the re-sort on the full key when a run is longer than the fix-up takes.  Bins, sorted ids and records must equal the
key sort's (csrc/splat_bin.cu) bit for bit, through gb_bin_tiles_pack and gb_bin_tiles_ranked.

The constructed scenes put every Gaussian at a tile centre with a radius that touches that tile only, so the length
of each tile and the sorted position of every equal-depth run are set exactly."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SORT_THREADS = 512  # threads of one tile sort (kSortThreads)
SORT_CAP = 5120     # entries of one tile sorted in shared memory (kSortCap)
TIE_RUN = 16        # longest equal-depth run sorted in place after the depth passes (kTieRun)
BW = 16
TILES_X = 8


def _check_against_key_sort(cuda, xys, depths, radii, nth, H, W, seed):
    """Bin with the key sort and with both bucket-binning entry points (both tile schedules); all must agree.
    Returns the tile bins."""
    from goliath_b200 import _lib
    from goliath_b200.gsplat import utils as gu

    G = xys.shape[0]
    rng = np.random.default_rng(seed)
    conics = torch.from_numpy(rng.uniform(0.1, 1.0, size=(G, 3)).astype(np.float32)).to(cuda)
    colors = torch.from_numpy(rng.uniform(0.0, 1.0, size=(G, 3)).astype(np.float32)).to(cuda)
    opacity = torch.from_numpy(rng.uniform(0.0, 1.0, size=(G, 1)).astype(np.float32)).to(cuda)
    comp = torch.from_numpy(rng.uniform(0.5, 1.0, size=G).astype(np.float32)).to(cuda)
    L = _lib.lib()
    st = _lib.stream_ptr(cuda)
    tb = gu._tile_bounds(H, W, BW)
    T = tb[0] * tb[1]
    n, cum = gu.compute_cumulative_intersects(nth)
    _, _, _, gids_ref, bins_ref = gu.bin_and_sort_gaussians(G, n, xys, depths, radii, cum, tb, BW)
    rec_ref = torch.empty(n, 12, device=cuda)
    _lib.check(L.gb_pack_records_fused(n, gids_ref.data_ptr(), xys.data_ptr(), conics.data_ptr(), colors.data_ptr(),
                                       depths.data_ptr(), opacity.data_ptr(), comp.data_ptr(), rec_ref.data_ptr(), st),
               "pack")
    i32 = dict(dtype=torch.int32, device=cuda)
    cap = n + 31
    ws = torch.empty(L.gb_bin_tiles_workspace_bytes(G, T, cap), dtype=torch.uint8, device=cuda)
    for tile_sched in (0, 1):
        order_len = L.gb_tile_schedule_ints(T) if tile_sched else T
        bins, order = torch.full((T, 2), -7, **i32), torch.full((order_len,), -7, **i32)
        gids, rec = torch.full((cap,), -7, **i32), torch.full((cap, 12), float("nan"), device=cuda)
        ovf = torch.zeros(1, **i32)
        _lib.check(L.gb_bin_tiles_pack(G, xys.data_ptr(), depths.data_ptr(), radii.data_ptr(), conics.data_ptr(),
                                       colors.data_ptr(), opacity.data_ptr(), comp.data_ptr(), H, W, BW, cap,
                                       bins.data_ptr(), order.data_ptr(), tile_sched, gids.data_ptr(), rec.data_ptr(),
                                       None, ovf.data_ptr(), ws.data_ptr(), st), "bin_tiles_pack")
        bins2, order2 = torch.full((T, 2), -7, **i32), torch.full((order_len,), -7, **i32)
        ids = torch.full((cap,), -7, **i32)
        rbi = torch.full((G, 12), float("nan"), device=cuda)
        r2g = torch.full((G,), -7, **i32)
        _lib.check(L.gb_bin_tiles_ranked(G, xys.data_ptr(), depths.data_ptr(), radii.data_ptr(), conics.data_ptr(),
                                         colors.data_ptr(), opacity.data_ptr(), comp.data_ptr(), H, W, BW, cap,
                                         bins2.data_ptr(), order2.data_ptr(), tile_sched, ids.data_ptr(), rbi.data_ptr(),
                                         r2g.data_ptr(), None, ovf.data_ptr(), ws.data_ptr(), None, st),
                   "bin_tiles_ranked")
        torch.cuda.synchronize()
        assert int(ovf) == 0
        assert torch.equal(bins, bins_ref) and torch.equal(bins2, bins_ref)
        assert torch.equal(gids[:n], gids_ref) and bool((gids[n:] == -7).all())
        assert torch.equal(rec[:n].view(torch.int32), rec_ref.view(torch.int32))
        assert torch.equal(ids[:n], gids_ref) and bool((ids[n:] == -7).all())
        assert torch.equal(r2g, torch.arange(G, **i32))
        assert torch.equal(rbi[ids[:n].long()].view(torch.int32), rec_ref.view(torch.int32))
    return bins_ref


def _tile_scene(cuda, ranks, seed):
    """One tile per entry of `ranks` (row-major over TILES_X tiles per row); ranks[t][i] is the depth rank of the i-th
    Gaussian of tile t in front-to-back order, equal ranks are equal depths.  Gaussian ids are shuffled over all
    tiles, so the id order inside an equal-depth run is random."""
    rng = np.random.default_rng(seed)
    rows = (len(ranks) + TILES_X - 1) // TILES_X
    H, W = rows * BW, TILES_X * BW
    xy, dep = [], []
    for t, r in enumerate(ranks):
        r = np.asarray(r)
        cx, cy = (t % TILES_X) * BW + BW / 2, (t // TILES_X) * BW + BW / 2
        xy.append(np.tile(np.array([[cx, cy]], np.float32), (len(r), 1)))
        dep.append((1.0 + r.astype(np.float64) * 2.0 ** -10).astype(np.float32))  # exact in fp32 below 2^13 ranks
    xy, dep = np.concatenate(xy), np.concatenate(dep)
    perm = rng.permutation(len(dep))
    xys = torch.from_numpy(xy[perm].copy()).to(cuda)
    depths = torch.from_numpy(dep[perm].copy()).to(cuda)
    radii = torch.ones(len(dep), dtype=torch.int32, device=cuda)  # radius 1 at a tile centre: that tile only
    return xys, depths, radii, torch.ones_like(radii), H, W


def _runs(n, runs):
    """Depth ranks of an n-entry tile whose sorted positions [p, p + length) tie for every (p, length) in runs."""
    r = np.arange(n)
    for p, length in runs:
        assert p + length <= n
        r[p:p + length] = p
    return r


LENGTHS = [1, 31, 32, 33, 511, 512, 513, 5119, 5120, 5121]


@pytest.mark.parametrize("depth", ["distinct", "ties"])
def test_tile_lengths_match_key_sort(cuda, depth):
    """Tiles of every length around a warp (32), the CTA (512 = one item per thread) and the shared-memory capacity
    (5120 = ten items per thread; 5121 takes the chunked path)."""
    rng = np.random.default_rng(5)
    if depth == "distinct":
        ranks = [rng.permutation(n) for n in LENGTHS]
    else:  # about two entries per depth: runs of 1 to ~10 at random positions
        ranks = [rng.integers(0, max(1, n // 2), size=n) for n in LENGTHS]
    xys, depths, radii, nth, H, W = _tile_scene(cuda, ranks, seed=11)
    bins = _check_against_key_sort(cuda, xys, depths, radii, nth, H, W, seed=12)
    lengths = (bins[:, 1] - bins[:, 0]).cpu().numpy()
    assert sorted(lengths[lengths > 0].tolist()) == sorted(LENGTHS)


def test_equal_depth_runs_match_key_sort(cuda):
    """Runs of 2, TIE_RUN and TIE_RUN + 1 equal depths at sorted positions across the lane/warp boundaries of the
    tile's layouts (items per thread = ceil(n / 512): a warp holds 32 * ipt consecutive entries in the passes; the
    run fix-up walks entries e, e + 512, ... per thread), at the start and the end of the tile, and whole tiles of one
    depth.  Tiles with a run longer than TIE_RUN re-sort on the full key."""
    R = TIE_RUN
    n = 1700  # 4 items per thread: warps hold 128 entries
    tiles = [
        _runs(n, [(0, 2), (30, 2), (63, 2), (127, 2), (255, R), (500, R), (511, 2), (1023, R), (n - 2, 2)]),
        _runs(n, [(0, R), (120, R + 1), (511, 2), (n - R, R)]),          # one run too long: the full-key passes
        _runs(n, [(n - R - 1, R + 1)]),
        _runs(SORT_CAP, [(31, R), (4607, 2), (5000, R + 1), (SORT_CAP - R, R)]),
        _runs(SORT_CAP, [(s, R) for s in range(0, SORT_CAP - R + 1, R)]),  # runs of R back to back
        _runs(SORT_CAP + 1, [(0, R + 1), (SORT_CAP - 2, 3)]),               # chunked path
        _runs(SORT_THREADS + 1, [(SORT_THREADS - 1, 2)]),
        _runs(33, [(31, 2)]),
        np.zeros(2, np.int64),
        np.zeros(R, np.int64),          # one depth, no digit pass: the fix-up sorts the whole tile
        np.zeros(R + 1, np.int64),      # one depth, too long: the full-key passes
        np.zeros(SORT_CAP, np.int64),
    ]
    xys, depths, radii, nth, H, W = _tile_scene(cuda, tiles, seed=21)
    bins = _check_against_key_sort(cuda, xys, depths, radii, nth, H, W, seed=22)
    lengths = (bins[:, 1] - bins[:, 0]).cpu().numpy()
    assert lengths[:len(tiles)].tolist() == [len(r) for r in tiles]


def test_bench_ring_cameras_match_key_sort(cuda):
    """The benchmarked scene (300k Gaussians, 1024x667) from all 16 ring cameras."""
    import bench
    from goliath_b200 import synthetic
    from goliath_b200.gsplat import project_gaussians

    u = bench.unpack(bench.packed_scene(300_000).to(cuda))
    for cam in range(16):
        c = synthetic.ring_camera(cam, img_h=bench.H, img_w=bench.W)
        xys, depths, radii, conics, comp, nth, cov3d = project_gaussians(
            u["primpos"].contiguous(), u["primscale"].contiguous(), 1.0, u["primqvec"].contiguous(),
            c["viewmat"].to(cuda), c["fx"], c["fy"], c["cx"], c["cy"], bench.H, bench.W, bench.BW, 0.1)
        assert bench.BW == BW
        bins = _check_against_key_sort(cuda, xys, depths, radii, nth, bench.H, bench.W, seed=cam)
        assert int((bins[:, 1] - bins[:, 0]).max()) <= SORT_CAP  # the shared-memory path only
