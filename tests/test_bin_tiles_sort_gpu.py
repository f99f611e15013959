"""The per-tile sort of the bucket binning (csrc/splat_bin_tiles.cu, tile_sort_kernel) on the inputs that take its
rare paths: tiles longer than the shared-memory capacity (sorted chunk by chunk through global memory) and tiles
full of equal depth keys (order decided by the Gaussian id alone).  Bins, sorted ids and records must equal the key
sort's (csrc/splat_bin.cu) bit for bit, through gb_bin_tiles_pack and gb_bin_tiles_ranked."""
import numpy as np
import pytest
import torch

from util import small_scene, t2n

pytestmark = pytest.mark.gpu

SORT_CAP = 5120  # entries of one tile sorted in shared memory (kSortCap)

CASES = {
    # name: (kwargs of small_scene, scale multiplier, depth levels (None: the scene's own depths), longest tile >)
    "long_tiles": (dict(G=40_000, img_h=96, img_w=80, seed=41), 14.0, None, SORT_CAP),
    "long_equal_depths": (dict(G=30_000, img_h=96, img_w=80, seed=43, cam=0), 14.0, 1, SORT_CAP),
    "depth_levels": (dict(G=6000, img_h=96, img_w=80, seed=47, cam=0), 8.0, 3, 0),
    "long_depth_levels": (dict(G=30_000, img_h=96, img_w=80, seed=53, cam=0), 14.0, 5, SORT_CAP),
}


def _scene(case):
    kw, mult, levels, _ = CASES[case]
    s = small_scene(**kw)
    if levels is not None:  # camera 0 looks down the world z axis: depth = 1000 - z, so z picks the depth key
        rng = np.random.default_rng(kw["seed"])
        s["means3d"][:, 2] = (rng.integers(0, levels, size=len(s["means3d"])) * 4.0).astype(np.float32)
    return s, mult


@pytest.mark.parametrize("tile_sched", [0, 1])
@pytest.mark.parametrize("case", list(CASES))
def test_tile_sort_rare_paths_match_key_sort(cuda, case, tile_sched):
    from goliath_b200 import _lib
    from goliath_b200.gsplat import project_gaussians
    from goliath_b200.gsplat import utils as gu

    s, mult = _scene(case)
    H, W, bw = s["img_h"], s["img_w"], 16
    t = {k: (torch.from_numpy(v).to(cuda) if isinstance(v, np.ndarray) else v) for k, v in s.items()}
    xys, depths, radii, conics, comp, nth, cov3d = project_gaussians(
        t["means3d"], t["scales"] * mult, 1.0, t["quats"], t["viewmat"], s["fx"], s["fy"], s["cx"], s["cy"], H, W, bw, 0.1)
    colors, opacity = t["colors"].contiguous(), t["opacity"].contiguous()
    G = xys.shape[0]
    L = _lib.lib()
    st = _lib.stream_ptr(cuda)
    n, cum = gu.compute_cumulative_intersects(nth)
    tb = gu._tile_bounds(H, W, bw)
    T = tb[0] * tb[1]
    _, _, _, gids_ref, bins_ref = gu.bin_and_sort_gaussians(G, n, xys, depths, radii, cum, tb, bw)
    lengths = t2n(bins_ref[:, 1] - bins_ref[:, 0])
    assert lengths.max() > CASES[case][3], "the scene must reach the path it is meant to test"
    if CASES[case][2] is not None:
        d = t2n(depths)[t2n(radii) > 0]
        assert len(np.unique(d)) <= CASES[case][2]
    rec_ref = torch.empty(n, 12, device=cuda)
    _lib.check(L.gb_pack_records_fused(n, gids_ref.data_ptr(), xys.data_ptr(), conics.data_ptr(), colors.data_ptr(),
                                       depths.data_ptr(), opacity.data_ptr(), comp.data_ptr(), rec_ref.data_ptr(), st),
               "pack")
    i32 = dict(dtype=torch.int32, device=cuda)
    cap = n + 55
    ws = torch.empty(L.gb_bin_tiles_workspace_bytes(G, T, cap), dtype=torch.uint8, device=cuda)
    order_len = L.gb_tile_schedule_ints(T) if tile_sched else T
    # packed
    bins, order = torch.full((T, 2), -7, **i32), torch.full((order_len,), -7, **i32)
    gids, rec = torch.full((cap,), -7, **i32), torch.full((cap, 12), float("nan"), device=cuda)
    ovf = torch.zeros(1, **i32)
    _lib.check(L.gb_bin_tiles_pack(G, xys.data_ptr(), depths.data_ptr(), radii.data_ptr(), conics.data_ptr(),
                                   colors.data_ptr(), opacity.data_ptr(), comp.data_ptr(), H, W, bw, cap, bins.data_ptr(),
                                   order.data_ptr(), tile_sched, gids.data_ptr(), rec.data_ptr(), None, ovf.data_ptr(),
                                   ws.data_ptr(), st), "bin_tiles_pack")
    # ranked: sorted ids, by-id records, identity rank_to_gid
    bins2, order2 = torch.full((T, 2), -7, **i32), torch.full((order_len,), -7, **i32)
    ids = torch.full((cap,), -7, **i32)
    rbi = torch.full((G, 12), float("nan"), device=cuda)
    r2g = torch.full((G,), -7, **i32)
    _lib.check(L.gb_bin_tiles_ranked(G, xys.data_ptr(), depths.data_ptr(), radii.data_ptr(), conics.data_ptr(),
                                     colors.data_ptr(), opacity.data_ptr(), comp.data_ptr(), H, W, bw, cap,
                                     bins2.data_ptr(), order2.data_ptr(), tile_sched, ids.data_ptr(), rbi.data_ptr(),
                                     r2g.data_ptr(), None, ovf.data_ptr(), ws.data_ptr(), None, st), "bin_tiles_ranked")
    torch.cuda.synchronize()
    assert int(ovf) == 0
    assert torch.equal(bins, bins_ref) and torch.equal(bins2, bins_ref)
    assert torch.equal(gids[:n], gids_ref) and bool((gids[n:] == -7).all())
    assert torch.equal(rec[:n].view(torch.int32), rec_ref.view(torch.int32))
    assert torch.equal(ids[:n], gids_ref) and bool((ids[n:] == -7).all())
    assert torch.equal(r2g, torch.arange(G, **i32))
    assert torch.equal(rbi[ids[:n].long()].view(torch.int32), rec_ref.view(torch.int32))
