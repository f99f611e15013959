"""The bucket scatter of the tile binning (csrc/splat_bin_tiles.cu, tile_scatter_kernel) at its edges: Gaussians whose
rectangles cover the whole image or one tile, warps that mix both, Gaussian counts around the warp and CTA sizes (the
scatter spreads the view over one wave of 1024 to 3072 Gaussians per CTA), above the point where the count kernel
takes 4096 Gaussians per CTA, CTAs with more pairs than the staging buffer holds, the tile grids without the staging
buffer and without shared-memory counters, a capacity below the intersection count, late colours, and a tile long
enough for the chunked sort (which reads the bucket whose depth keys the scatter left in the output array).

Every case bins with the key sort (csrc/splat_bin.cu) and with gb_bin_tiles_pack, gb_bin_tiles_pack_ev and
gb_bin_tiles_ranked under both tile schedules; bins, sorted ids, records and the by-id record table must agree bit
for bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BW = 16
STAGE_CAP = 12 * 1024      # pairs one scatter CTA stages in shared memory (kStageCap)
STAGE_MAX_TILES = 10 * 1024  # largest grid with the staging buffer (kStageMaxTiles)
SMEM_TILES = 20 * 1024     # largest grid with shared-memory counters (kMaxSmemTiles)
SCAT_MIN = 1024            # fewest Gaussians per scatter CTA (one per thread); at most 3072, one wave of CTAs between
COUNT_SPLIT = 2048 * 192   # above this the count kernel takes 4096 Gaussians per CTA
SORT_CAP = 5120            # longest tile sorted in shared memory (kSortCap)


def _tiles_hit(xys, radii, H, W):
    """Tiles of each Gaussian's rectangle, with the float32 arithmetic of tile_bbox; 0 when culled."""
    tbx, tby = (W + BW - 1) // BW, (H + BW - 1) // BW
    fb = np.float32(BW)
    tcx, tcy, tr = xys[:, 0] / fb, xys[:, 1] / fb, radii.astype(np.float32) / fb
    x0 = np.clip(np.trunc(tcx - tr), 0, tbx)
    x1 = np.clip(np.trunc((tcx + tr) + np.float32(1)), 0, tbx)
    y0 = np.clip(np.trunc(tcy - tr), 0, tby)
    y1 = np.clip(np.trunc((tcy + tr) + np.float32(1)), 0, tby)
    return np.where(radii > 0, (x1 - x0) * (y1 - y0), 0).astype(np.int32)


def _scene(xy, radii, depth, H, W, cuda):
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    radii = np.asarray(radii, np.int32)
    depth = np.asarray(depth, np.float32)
    nth = _tiles_hit(xy, radii, H, W)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)  # noqa: E731
    return t(xy), t(depth), t(radii), t(nth), H, W


def _random_scene(cuda, G, H, W, seed, r_max=24, culled=0.05):
    """G Gaussians uniform over the image (some past its edges), radii 1..r_max, a few culled; depths on a 2^-12 grid
    so that equal depths occur."""
    rng = np.random.default_rng(seed)
    xy = np.stack([rng.uniform(-20, W + 20, G), rng.uniform(-20, H + 20, G)], 1)
    radii = rng.integers(1, r_max + 1, G)
    radii[rng.random(G) < culled] = 0
    depth = 1.0 + rng.integers(0, 4096, G) / 4096.0
    return _scene(xy, radii, depth, H, W, cuda)


def _tile_centre(t, W):
    tbx = (W + BW - 1) // BW
    return (t % tbx) * BW + BW / 2, (t // tbx) * BW + BW / 2


def _bin_all(cuda, xys, depths, radii, nth, H, W, seed, cap=None, spare=64):
    """Bin with the key sort and every bucket-binning entry point; compare.  cap (default: the intersection count + 31)
    below the count checks the overflow contract instead: the flag, clamped bins, exact tiles below the capacity and
    nothing written past it.  Returns (tile bins of the key sort, intersection count)."""
    from goliath_b200 import _lib
    from goliath_b200.gsplat import utils as gu

    G = xys.shape[0]
    rng = np.random.default_rng(seed)
    f32 = lambda a: torch.from_numpy(a.astype(np.float32)).to(cuda)  # noqa: E731
    conics = f32(rng.uniform(0.1, 1.0, size=(G, 3)))
    colors = f32(rng.uniform(0.0, 1.0, size=(G, 3)))
    opacity = f32(rng.uniform(0.0, 1.0, size=(G, 1)))
    comp = f32(rng.uniform(0.5, 1.0, size=G))
    L = _lib.lib()
    st = _lib.stream_ptr(cuda)
    tb = gu._tile_bounds(H, W, BW)
    T = tb[0] * tb[1]
    n, cum = gu.compute_cumulative_intersects(nth)
    _, _, _, gids_ref, bins_ref = gu.bin_and_sort_gaussians(G, n, xys, depths, radii, cum, tb, BW)
    i32 = dict(dtype=torch.int32, device=cuda)
    rec_ref = torch.empty(max(n, 1), 12, device=cuda)
    _lib.check(L.gb_pack_records_fused(n, gids_ref.data_ptr(), xys.data_ptr(), conics.data_ptr(), colors.data_ptr(),
                                       depths.data_ptr(), opacity.data_ptr(), comp.data_ptr(), rec_ref.data_ptr(), st),
               "pack")
    all_ids = torch.arange(G, **i32)
    rec_by_id_ref = torch.empty(G, 12, device=cuda)
    _lib.check(L.gb_pack_records_fused(G, all_ids.data_ptr(), xys.data_ptr(), conics.data_ptr(), colors.data_ptr(),
                                       depths.data_ptr(), opacity.data_ptr(), comp.data_ptr(), rec_by_id_ref.data_ptr(),
                                       st), "pack by id")
    overflow = cap is not None and cap < n
    if cap is None:
        cap = n + 31
    # positions below cap whose tile lies wholly below cap: exact even with an overflow
    lens = (bins_ref[:, 1] - bins_ref[:, 0]).long()
    tile_of = torch.repeat_interleave(torch.arange(T, device=cuda), lens)
    exact = (bins_ref[tile_of, 1] <= cap)[:min(n, cap)]
    m = int(exact.sum())
    assert bool(exact[:m].all())  # a prefix
    bins_exp = bins_ref.clone()
    bins_exp[:, 1] = bins_exp[:, 1].clamp(max=cap)
    bins_exp[(bins_exp[:, 1] <= bins_exp[:, 0]) | (lens == 0)] = 0
    vis = (radii > 0)
    ws = torch.empty(L.gb_bin_tiles_workspace_bytes(G, T, cap), dtype=torch.uint8, device=cuda)
    for tile_sched in (0, 1):
        order_len = L.gb_tile_schedule_ints(T) if tile_sched else T
        for entry in ("pack", "pack_ev", "ranked"):
            bins, order = torch.full((T, 2), -7, **i32), torch.full((order_len,), -7, **i32)
            ids = torch.full((cap + spare,), -7, **i32)
            n_out, ovf = torch.full((1,), -7, **i32), torch.zeros(1, **i32)
            common = (G, xys.data_ptr(), depths.data_ptr(), radii.data_ptr(), conics.data_ptr(), colors.data_ptr(),
                      opacity.data_ptr(), comp.data_ptr(), H, W, BW, cap, bins.data_ptr(), order.data_ptr(), tile_sched,
                      ids.data_ptr())
            if entry == "ranked":
                rbi = torch.full((G, 12), float("nan"), device=cuda)
                r2g = torch.full((G,), -7, **i32)
                _lib.check(L.gb_bin_tiles_ranked(*common, rbi.data_ptr(), r2g.data_ptr(), n_out.data_ptr(),
                                                 ovf.data_ptr(), ws.data_ptr(), None, st), "bin_tiles_ranked")
            else:
                rec = torch.full((cap + spare, 12), float("nan"), device=cuda)
                if entry == "pack":
                    _lib.check(L.gb_bin_tiles_pack(*common, rec.data_ptr(), n_out.data_ptr(), ovf.data_ptr(),
                                                   ws.data_ptr(), st), "bin_tiles_pack")
                else:  # late colours: the colour quarter waits for an event recorded after the colours are written
                    late = torch.full_like(colors, float("nan"))
                    _lib.check(L.gb_bin_tiles_pack_ev(*common[:5], late.data_ptr(), *common[6:], rec.data_ptr(),
                                                      n_out.data_ptr(), ovf.data_ptr(), ws.data_ptr(), _ev(cuda, late,
                                                                                                           colors),
                                                      st), "bin_tiles_pack_ev")
            torch.cuda.synchronize()
            what = "%s, tile_sched %d" % (entry, tile_sched)
            assert int(n_out) == n, what
            assert int(ovf) == int(overflow), what
            assert torch.equal(bins, bins_exp), what
            assert bool((ids[cap:] == -7).all()), what + ": write past cap"
            assert torch.equal(ids[:m], gids_ref[:m]), what
            if not overflow:
                assert bool((ids[n:] == -7).all()), what
            if entry == "ranked":
                assert torch.equal(r2g, all_ids), what
                assert torch.equal(rbi[vis].view(torch.int32), rec_by_id_ref[vis].view(torch.int32)), what
                assert bool(rbi[~vis].isnan().all()), what + ": record of a culled Gaussian"
            else:
                assert torch.equal(rec[:m].view(torch.int32), rec_ref[:m].view(torch.int32)), what
                assert bool(rec[cap:].isnan().all()), what + ": record past cap"
    return bins_ref, n


def _ev(cuda, late, colors):
    """Copy the colours into `late` on a side stream and return the raw event recorded after it."""
    side = torch.cuda.Stream(device=cuda)
    side.wait_stream(torch.cuda.current_stream(cuda))
    torch.cuda._sleep(1_000_000)  # the binning's first kernels are queued while the colours are still missing
    with torch.cuda.stream(side):
        torch.cuda._sleep(2_000_000)
        late.copy_(colors)
        ev = torch.cuda.Event()
        ev.record(side)
    _ev.keep = (side, ev)  # alive until the caller synchronises
    return ev.cuda_event


def test_one_gaussian_covers_every_tile(cuda):
    """G = 1 whose rectangle is the whole 40 x 30 tile grid: one thread owns every pair of the CTA."""
    H, W = 480, 640
    _, n = _bin_all(cuda, *_scene([[W / 2, H / 2]], [2000], [1.5], H, W, cuda), seed=1)
    assert n == (W // BW) * (H // BW)


def test_one_gaussian_over_the_image_among_others(cuda):
    """A whole-image rectangle in the middle of 3000 small Gaussians, and one past the edges that is clipped."""
    H, W = 480, 640
    xys, depths, radii, nth, _, _ = _random_scene(cuda, 3000, H, W, seed=2)
    xy, r, d = xys.cpu().numpy(), radii.cpu().numpy(), depths.cpu().numpy()
    xy[1500], r[1500], d[1500] = (W / 2, H / 2), 5000, 1.25
    xy[77], r[77] = (-100.0, -100.0), 300
    _bin_all(cuda, *_scene(xy, r, d, H, W, cuda), seed=3)


def test_consecutive_ids_in_one_tile(cuda):
    """32 consecutive ids (one whole warp) in one tile, 33 (one past a warp) in another, around random Gaussians;
    then 2053 in one tile (three scatter CTAs, each claiming its run of the tile)."""
    H, W = 256, 256
    rng = np.random.default_rng(4)
    G = 200
    xy = np.stack([rng.uniform(0, W, G), rng.uniform(0, H, G)], 1)
    radii = rng.integers(1, 20, G)
    depth = 1.0 + rng.integers(0, 64, G) / 64.0
    xy[32:64], radii[32:64] = _tile_centre(5, W), 1
    xy[96:129], radii[96:129] = _tile_centre(40, W), 1
    bins, _ = _bin_all(cuda, *_scene(xy, radii, depth, H, W, cuda), seed=5)
    assert int(bins[5, 1] - bins[5, 0]) >= 32 and int(bins[40, 1] - bins[40, 0]) >= 33
    G = 2 * SCAT_MIN + 5
    xy = np.tile(np.array([_tile_centre(17, W)], np.float32), (G, 1))
    depth = 1.0 + rng.integers(0, 300, G) / 512.0
    bins, _ = _bin_all(cuda, *_scene(xy, np.ones(G), depth, H, W, cuda), seed=6)
    assert int(bins[17, 1] - bins[17, 0]) == G


def test_warps_mix_one_huge_rectangle_with_single_tiles(cuda):
    """Every warp holds one Gaussian that covers most of the image (at a different lane per warp) and 31 that each
    touch one tile."""
    H, W = 512, 512
    rng = np.random.default_rng(7)
    G = 4 * SCAT_MIN + 37
    tiles = rng.integers(0, (W // BW) * (H // BW), G)
    xy = np.array([_tile_centre(t, W) for t in tiles], np.float32)
    radii = np.ones(G, np.int64)
    depth = 1.0 + rng.integers(0, 4096, G) / 4096.0
    for w in range((G + 31) // 32):
        g = w * 32 + (w % 32)
        if g < G:
            xy[g] = rng.uniform(100, 400, 2)
            radii[g] = rng.integers(150, 260)
    _bin_all(cuda, *_scene(xy, radii, depth, H, W, cuda), seed=8)


@pytest.mark.parametrize("G", [1, 31, 33, 1000, 1023, 1025, 2047, 2049, 5000, 30001, 200003])
def test_gaussian_counts_around_warp_and_cta(cuda, G):
    H, W = 667, 1024
    _bin_all(cuda, *_random_scene(cuda, G, H, W, seed=G), seed=G + 1)


def test_count_and_scatter_partitions_differ(cuda):
    """Above 393,216 Gaussians the count kernel takes 4096 Gaussians per CTA; the scatter takes about 3000 (three per
    thread, the last item partly filled)."""
    G = COUNT_SPLIT + 3001
    _bin_all(cuda, *_random_scene(cuda, G, 667, 1024, seed=9, r_max=12), seed=10)


def test_cta_with_more_pairs_than_the_staging_buffer(cuda):
    """Large rectangles: every scatter CTA has far more than STAGE_CAP pairs and writes them directly."""
    H, W = 667, 1024
    G = 4 * SCAT_MIN + 100
    xys, depths, radii, nth, _, _ = _random_scene(cuda, G, H, W, seed=11, r_max=60)
    assert int(nth[:SCAT_MIN].sum()) > STAGE_CAP
    _bin_all(cuda, xys, depths, radii, nth, H, W, seed=12)


def test_grid_without_the_staging_buffer(cuda):
    """128 x 100 tiles: shared-memory counters, no room for the staging buffer."""
    H, W = 1600, 2048
    assert STAGE_MAX_TILES < (H // BW) * (W // BW) <= SMEM_TILES
    _bin_all(cuda, *_random_scene(cuda, 20000, H, W, seed=13), seed=14)


def test_grid_with_global_atomics(cuda):
    """160 x 144 tiles: more than the shared-memory counters hold, one global atomic per pair."""
    H, W = 2304, 2560
    assert (H // BW) * (W // BW) > SMEM_TILES
    _bin_all(cuda, *_random_scene(cuda, 20000, H, W, seed=15), seed=16)


@pytest.mark.parametrize("frac", [0.0, 0.37, 0.999])
def test_capacity_below_the_intersection_count(cuda, frac):
    """cap < intersections: the overflow flag, bins clamped to cap, every tile below cap exact, nothing past cap."""
    H, W = 667, 1024
    scene = _random_scene(cuda, 6000, H, W, seed=17)
    n = int(scene[3].sum())
    _bin_all(cuda, *scene, seed=18, cap=int(n * frac))


def test_tile_longer_than_the_shared_memory_sort(cuda):
    """A tile of SORT_CAP + 900 entries (the chunked sort, whose first pass overwrites the keys in the output array)
    among ordinary tiles, with equal depths in it."""
    H, W = 256, 256
    rng = np.random.default_rng(19)
    G = SORT_CAP + 900 + 3000
    xy = np.stack([rng.uniform(0, W, G), rng.uniform(0, H, G)], 1)
    radii = rng.integers(1, 12, G)
    hot = rng.permutation(G)[:SORT_CAP + 900]
    xy[hot], radii[hot] = _tile_centre(33, W), 1
    depth = 1.0 + rng.integers(0, 2048, G) / 2048.0
    bins, _ = _bin_all(cuda, *_scene(xy, radii, depth, H, W, cuda), seed=20)
    assert int(bins[33, 1] - bins[33, 0]) > SORT_CAP
