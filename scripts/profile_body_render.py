"""Time the body avatar's render (DESIGN.md row R9'': csrc/mesh_raster.cu behind goliath_b200.mesh_render.RenderLayer)
at the configuration's size: B = 4, 2048 x 1334, a 4-channel 2048^2 texture, on the closed synthetic multi-part mesh of
goliath_b200.synthetic.body_mesh at two face counts (the body template's own face count is not known here).

Reports, per face count: the raster, render forward and backward (with and without edge_grad) kernel-entry times from
CUDA events; the end-to-end forward and forward + backward times and their peak memory; the render forward's share
of the HBM roof from the byte count below; and torch's grid_sample forward and backward on our vt_img (fp32 with TF32
off, and torch's defaults).  drtk is not available, so there is no end-to-end baseline; the output says so.

Usage: python scripts/profile_body_render.py [--reps 10] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_GBS = 3350.0      # H100 SXM HBM3 peak
B, H, W, C, T = 4, 2048, 1334, 4, 2048


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "unknown (%s)" % e
    return q


def timed(fn, reps):
    for _ in range(3):
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
    return float(np.median(ts))


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def fwd_bytes(n_pix, n_cov):
    """least traffic of the render forward: read the index image, write depth, 3 bary, 2 vt, mask and C render
    floats per pixel; per covered pixel read 3 vertices (9 floats), 3 vt (6 floats) and 4 taps per channel"""
    return n_pix * 4 * (1 + 1 + 3 + 2 + 1 + C) + n_cov * 4 * (9 + 6 + 4 * C)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    from goliath_b200 import _lib, synthetic
    from goliath_b200.mesh_render import RenderLayer, _MeshRender, transform

    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    dev = torch.device("cuda:0")
    L = _lib.lib()
    res = {"card": card(), "torch": torch.__version__, "reps": args.reps, "B": B, "H": H, "W": W, "C": C, "tex": T,
           "baseline": "no drtk on this machine: no end-to-end baseline; torch comparison is grid_sample only"}
    gen = torch.Generator(device=dev).manual_seed(0)
    tex = torch.rand(B, C, T, T, device=dev, generator=gen)
    g_out = torch.randn(B, C, H, W, device=dev, generator=gen)
    for n_faces in (100_000, 400_000):
        s = synthetic.body_mesh(n_faces, H, W, B)
        layer = RenderLayer(H, W, s["vi"], s["vt"], s["vti"]).to(dev)
        verts = s["verts"][None].expand(B, -1, -1).contiguous().to(dev)
        K, Rt = s["K"].to(dev), s["Rt"].to(dev)
        v_pix = transform(verts, K, Rt).contiguous()
        vi, vti, vt, inc = layer._device_tables(dev)
        F, V = vi.shape[0], v_pix.shape[1]
        r = {"faces": F, "verts": V}
        st = _lib.stream_ptr(dev)
        idx = torch.empty(B, H, W, device=dev, dtype=torch.int32)
        ws = torch.empty(L.gb_mesh_raster_workspace_bytes(B, F, H, W), device=dev, dtype=torch.uint8)
        raster = lambda: L.gb_mesh_raster(B, V, F, H, W, v_pix.data_ptr(), vi.data_ptr(), idx.data_ptr(),
                                          ws.data_ptr(), st)
        r["raster_ms"] = timed(raster, args.reps)
        outs = [torch.empty(B, H, W, device=dev), torch.empty(B, 3, H, W, device=dev),
                torch.empty(B, 2, H, W, device=dev), torch.empty(B, 1, H, W, device=dev),
                torch.empty(B, C, H, W, device=dev)]
        fwd = lambda: L.gb_mesh_render_fwd(B, V, F, H, W, C, T, T, v_pix.data_ptr(), vi.data_ptr(), vti.data_ptr(),
                                           vt.data_ptr(), tex.data_ptr(), idx.data_ptr(),
                                           *[o.data_ptr() for o in outs], st)
        r["render_fwd_ms"] = timed(fwd, args.reps)
        n_cov = int((idx >= 0).sum())
        r["coverage"] = n_cov / (B * H * W)
        r["render_fwd_hbm_roof"] = fwd_bytes(B * H * W, n_cov) / (r["render_fwd_ms"] * 1e-3) / (HBM_GBS * 1e9)
        g_v, g_t = torch.empty_like(v_pix), torch.empty_like(tex)
        bws = torch.empty(L.gb_mesh_render_bwd_workspace_bytes(B, F, H, W, T, T), device=dev, dtype=torch.uint8)
        r["bwd_workspace_mib"] = bws.numel() / 2 ** 20
        inc_ptr = inc.ptr
        for eg in (0, 1):
            bwd = lambda: L.gb_mesh_render_bwd(
                B, V, F, H, W, C, T, T, v_pix.data_ptr(), vi.data_ptr(), vti.data_ptr(), vt.data_ptr(),
                tex.data_ptr(), idx.data_ptr(), outs[2].data_ptr(), outs[4].data_ptr(), g_out.data_ptr(), eg,
                inc_ptr.data_ptr(), inc.inc.data_ptr(), g_v.data_ptr(), g_t.data_ptr(), bws.data_ptr(), st)
            r["render_bwd_edge%d_ms" % eg] = timed(bwd, args.reps)
        del bws

        vv = verts.clone().requires_grad_()
        tt = tex.clone().requires_grad_()
        e2e_f = lambda: layer(verts, tex, K, Rt)
        r["e2e_fwd_ms"] = timed(lambda: torch.no_grad()(e2e_f)(), args.reps)
        r["e2e_fwd_peak_mib"] = peak(lambda: torch.no_grad()(e2e_f)())

        def fb():
            out = layer(vv, tt, K, Rt)
            torch.autograd.grad((out["render"] * g_out).sum(), [vv, tt])
        r["e2e_fwd_bwd_ms"] = timed(fb, args.reps)
        r["e2e_fwd_bwd_peak_mib"] = peak(fb)

        # torch grid_sample on our vt_img (the one stage torch can express)
        grid = outs[2].permute(0, 2, 3, 1).contiguous()
        for tag, tf32 in (("torch_tf32_off", False), ("torch_defaults", None)):
            saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
            gs = lambda: torch.nn.functional.grid_sample(tex, grid, mode="bilinear", align_corners=False) * outs[3]
            r[tag + "_grid_sample_fwd_ms"] = timed(gs, args.reps)

            def gsb():
                o = torch.nn.functional.grid_sample(tt, grid, mode="bilinear", align_corners=False) * outs[3]
                torch.autograd.grad((o * g_out).sum(), [tt])
            r[tag + "_grid_sample_fwd_bwd_ms"] = timed(gsb, args.reps)
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
        res["faces_%d" % n_faces] = r
        del layer, s
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
