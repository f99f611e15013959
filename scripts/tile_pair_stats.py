"""(Gaussian, tile) pair statistics of the bench head view, computed on the CPU (oracle/splat_oracle.c projects): how
many tiles each Gaussian touches, and how the pairs of one warp of the bucket scatter (32 consecutive Gaussian ids)
spread over tiles.  These bound the work of tile_scatter_kernel (csrc/splat_bin_tiles.cu) without a GPU.

  python scripts/tile_pair_stats.py [--camera 0] [--gaussians 300000]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def tile_rects(xys, radii, tbx, tby, bw):
    """Tile rectangle [x0, x1) x [y0, y1) of every Gaussian, with the float32 arithmetic of tile_bbox."""
    fb = np.float32(bw)
    cx, cy, r = xys[:, 0].astype(np.float32), xys[:, 1].astype(np.float32), radii.astype(np.float32)
    tcx, tcy, tr = cx / fb, cy / fb, r / fb
    x0 = np.clip(np.trunc(tcx - tr), 0, tbx).astype(np.int64)
    x1 = np.clip(np.trunc((tcx + tr) + np.float32(1)), 0, tbx).astype(np.int64)
    y0 = np.clip(np.trunc(tcy - tr), 0, tby).astype(np.int64)
    y1 = np.clip(np.trunc((tcy + tr) + np.float32(1)), 0, tby).astype(np.int64)
    vis = radii > 0
    n = np.where(vis, (x1 - x0) * (y1 - y0), 0)
    return x0, y0, x1, y1, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--camera", type=int, default=0)
    ap.add_argument("--gaussians", type=int, default=300_000)
    a = ap.parse_args()
    import bench
    import oracle
    from goliath_b200 import synthetic

    u = bench.unpack(bench.packed_scene(a.gaussians))
    c = synthetic.ring_camera(a.camera, img_h=bench.H, img_w=bench.W)
    p = oracle.project_fwd(u["primpos"].numpy(), u["primscale"].numpy(), 1.0, u["primqvec"].numpy(),
                           c["viewmat"].numpy(), c["fx"], c["fy"], c["cx"], c["cy"], bench.H, bench.W, bench.BW, 0.1)
    tbx, tby = oracle.tile_bounds(bench.H, bench.W, bench.BW)
    x0, y0, x1, y1, n = tile_rects(p["xys"], p["radii"], tbx, tby, bench.BW)
    assert np.array_equal(n, p["num_tiles_hit"]), "tile rectangles disagree with the oracle's tile counts"
    G = len(n)
    vis = n > 0
    nv = n[vis]
    print("camera %d: %d Gaussians, %d visible, %d tiles (%d x %d), %d pairs" % (a.camera, G, vis.sum(), tbx * tby, tbx,
                                                                              tby, n.sum()))
    print("tiles per visible Gaussian: mean %.2f, p50 %d, p90 %d, p99 %d, max %d"
          % (nv.mean(), np.percentile(nv, 50), np.percentile(nv, 90), np.percentile(nv, 99), nv.max()))
    # warps of 32 consecutive ids: the serial walk lasts as long as the largest rectangle of the warp
    Gp = (G + 31) // 32 * 32
    nw = np.zeros(Gp, np.int64)
    nw[:G] = n
    nw = nw.reshape(-1, 32)
    wmax, wsum = nw.max(1), nw.sum(1)
    busy = wsum[wmax > 0] / (32.0 * wmax[wmax > 0])
    print("per warp: sum of lane maxima %d (serial walk steps), sum of ceil(pairs / 32) %d (cooperative steps); "
          "lane utilisation of the serial walk %.1f %%" % (wmax.sum(), ((wsum + 31) // 32).sum(), 100.0 * busy.mean()))
    # tile of every pair in the warp's flattened list, 32 at a time: distinct tiles per step and the largest group
    distinct, largest, steps = [], [], 0
    for w in range(Gp // 32):
        ids = np.arange(w * 32, min(w * 32 + 32, G))
        ids = ids[n[ids] > 0]
        if len(ids) == 0:
            continue
        lst = np.concatenate([(np.arange(y0[i], y1[i])[:, None] * tbx + np.arange(x0[i], x1[i])[None, :]).ravel()
                              for i in ids])
        for s in range(0, len(lst), 32):
            _, cnt = np.unique(lst[s:s + 32], return_counts=True)
            distinct.append(len(cnt))
            largest.append(cnt.max())
            steps += 1
    distinct, largest = np.array(distinct), np.array(largest)
    print("cooperative steps of 32 pairs: %d; distinct tiles per step mean %.1f (p10 %d, p90 %d); largest same-tile "
          "group per step mean %.1f (p90 %d, max %d)" % (steps, distinct.mean(), np.percentile(distinct, 10),
                                                         np.percentile(distinct, 90), largest.mean(),
                                                         np.percentile(largest, 90), largest.max()))


if __name__ == "__main__":
    main()
