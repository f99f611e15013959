"""Time `GeometryModule.from_topology(impaint=True)` (csrc/uv_layout.cu) on the synthetic avatar-size UV layout
(goliath_b200.synthetic.uv_layout: 32769 faces) at 1024^2 and 2048^2.

  * end to end: CUDA events around from_topology, warmed up, median of --reps calls, with the topology on the host
    (the buffers then come back to the host, as the reference's do: the device-to-host copies and the module's dtype
    conversions are included) and with the topology on the device (the buffers stay there); both include the one
    host read of the empty-image check and the Python glue;
  * per stage: kernel times from torch.profiler in a separate run (raster = init + per-face + per-large-face kernels,
    per-texel pass, distance transform = column + row passes, source selection, gather), with the bytes each stage
    must move computed from the shapes and their share of the H100 SXM's 3.35 TB/s HBM3;
  * baseline: the reference's impaint formulation on the host, sklearn's KDTree built over the valid texels and
    queried with the invalid ones, as index_image_impaint runs it.  pytorch3d's rasteriser is not available here, so
    the raster has no baseline.

The card's name, power limit and max SM clock are read in the same run.  Prints one JSON line and writes it, with the
two profiler traces, to --out.   Usage: python scripts/profile_uv_images.py [--reps 20] [--out DIR]
(writes DIR/uv_images.json)
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from goliath_b200 import geom, synthetic  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
STAGES = {"raster": ("uv_raster_init", "uv_raster_small", "uv_raster_large"), "texel": ("uv_texel",),
          "distance transform": ("edt_cols", "edt_rows"), "source selection": ("impaint_select",),
          "gather": ("impaint_gather",)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def stage_bytes(U, F):
    """the bytes each stage must read and write, from the shapes (a lower bound: no re-reads)"""
    T = U * U
    return {"raster": 4 * T + F * (12 + 3 * 8),                        # the int32 image set, faces and their corners
            "texel": T * (4 + 8 + 24 + 12 + 1),                        # image in; face, vi[face], bary, valid out
            "distance transform": T * (24 + 4) + T * (4 + 4),          # index in, g out; g in, d2 out
            "source selection": T * (4 + 4),                           # d2 in, src out
            "gather": T * (4 + 2 * (24 + 12 + 8))}                     # src in; index, bary, face in and out


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def stage_times(fn, reps, trace):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    ev = [e for e in json.load(open(trace))["traceEvents"] if e.get("cat") == "kernel"]
    out = {}
    for stage, names in STAGES.items():
        out[stage] = sum(e["dur"] for e in ev if any(n in e["name"] for n in names)) / reps / 1e3  # ms per call
    return out


def kdtree_baseline(index_image):
    from sklearn.neighbors import KDTree

    valid = (index_image != -1).any(-1)
    vij, iij = np.argwhere(valid), np.argwhere(~valid)
    t0 = time.perf_counter()
    tree = KDTree(vij)
    t1 = time.perf_counter()
    tree.query(iij)
    t2 = time.perf_counter()
    return {"build_ms": 1e3 * (t1 - t0), "query_ms": 1e3 * (t2 - t1), "n_valid": len(vij), "n_invalid": len(iij)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--sizes", default="1024,2048")
    ap.add_argument("--out", default="uv_images_profile")
    ap.add_argument("--no-baseline", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_uv_images: needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    L = synthetic.uv_layout()
    F = L["vti"].shape[0]
    res = {"card": card(), "faces": F, "sizes": {}}
    for U in (int(s) for s in args.sizes.split(",")):
        fn = lambda: geom.GeometryModule.from_topology(L["vi"], L["vt"], L["vti"], L["v2uv"], U, impaint=True)
        med, best = timed(fn, args.reps)
        Lc = {k: v.cuda() for k, v in L.items()}
        fn_dev = lambda: geom.GeometryModule.from_topology(Lc["vi"], Lc["vt"], Lc["vti"], Lc["v2uv"], U, impaint=True)
        med_dev, best_dev = timed(fn_dev, args.reps)
        st = stage_times(fn, args.reps, os.path.join(args.out, "uv_images_trace_%d.json" % U))
        by = stage_bytes(U, F)
        r = {"from_topology_ms_median": med, "from_topology_ms_min": best,
             "from_topology_cuda_topology_ms_median": med_dev, "from_topology_cuda_topology_ms_min": best_dev,
             "stages_ms": st,
             "kernels_ms": sum(st.values()),
             "stage_hbm_share": {k: by[k] / (st[k] * 1e-3) / HBM_BYTES_PER_S if st[k] > 0 else None for k in st},
             "stage_bytes": by}
        if not args.no_baseline:
            index = geom._index_images(L["vt"], L["vti"], L["vi"], U, False, face=False, vert=True)[1]
            r["kdtree_host"] = kdtree_baseline(index.cpu().numpy())
        res["sizes"][U] = r
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    with open(os.path.join(args.out, "uv_images.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
