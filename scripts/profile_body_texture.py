"""Time the body avatar's texture branch (DESIGN.md row R9') on the GPU: UNetViewDecoder -> ShadowUNet ->
TextureComposer, forward at B = 1 and forward + backward at B = 4, against the torch restatement
(tests/body_texture_restate.py with the seam sampler restated in torch) in fp32 with TF32 off and with torch's
defaults; the composite kernel's forward and backward with CUDA events against their shape-derived byte counts and the
HBM roof; peak memory; the card name and power limit.

Usage: python scripts/profile_body_texture.py [--reps 10] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_GBS = 3350.0      # H100 SXM HBM3 peak


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    import body_texture_restate as bt
    from test_body_texture_gpu import _our_branch, restated_branch
    from goliath_b200.mesh_vae import _TexCompose

    dev = torch.device("cuda:0")
    res = {"card": card(), "torch": torch.__version__, "reps": args.reps}
    inp, (view, shadow, comp) = _our_branch(dev)
    _, shadow_r, view_r, comp_r = restated_branch(device=dev, dtype=torch.float32)

    def branch(v, s, c):
        def f(tmr, geom, cam, ao):
            tvr = v(geom, tmr, cam)["tex_view_rec"]
            return c(tmr, tvr, s(ao)["shadow_map"])
        return f

    for B in (1, 4):
        bi = {k: (t if k in ("ao_mean", "tex_mean") else t[:1].expand(B, *t.shape[1:]).contiguous())
              for k, t in inp.items()}
        for name, f, mods in (("ours", branch(view, shadow, comp), (view, shadow, comp)),
                              ("torch_fp32_notf32", branch(view_r, shadow_r, comp_r), (view_r, shadow_r, comp_r)),
                              ("torch_default", branch(view_r, shadow_r, comp_r), (view_r, shadow_r, comp_r))):
            tf32 = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = name == "torch_default"
            try:
                def fwd():
                    with torch.no_grad():
                        return f(bi["tex_mean_rec"], bi["geom_rec"], bi["camera_pos"], bi["ao_map"])

                def fwd_bwd():
                    tmr = bi["tex_mean_rec"].clone().requires_grad_()
                    f(tmr, bi["geom_rec"], bi["camera_pos"], bi["ao_map"]).sum().backward()

                if B == 1:
                    res["fwd_B1_ms_" + name] = timed(fwd, args.reps)
                    res["fwd_B1_peak_MiB_" + name] = peak(fwd)
                else:
                    res["fwd_bwd_B4_ms_" + name] = timed(fwd_bwd, args.reps)
                    res["fwd_bwd_B4_peak_MiB_" + name] = peak(fwd_bwd)
            finally:
                torch.backends.cudnn.allow_tf32 = tf32
            for m in mods:
                m.zero_grad(set_to_none=True)

    # the composite kernel alone, against its bytes and the torch formula (fp32)
    ob = comp.upscale_net.out_block
    rows = []
    for B in (1, 4):
        H = 1024
        g = torch.Generator(device=dev).manual_seed(B)
        t1 = torch.randn(B, 3, H, H, device=dev, generator=g)
        h = torch.randn(B, 4, H, H, device=dev, generator=g)
        s3 = torch.rand(B, 1, 2 * H, 2 * H, device=dev, generator=g)
        tm = comp.tex_mean
        gp = torch.randn(B, 3, 2 * H, 2 * H, device=dev, generator=g)
        px, px2 = H * H, 4 * H * H
        # forward: T1, h, 12 untied biases, tex_mean, S3 read; P written
        by_fwd = 4.0 * (B * 3 * px + B * 4 * px + 12 * px + 3 * px2 + B * px2 + B * 3 * px2)
        # backward: T1, h, biases, tex_mean, S3, g_P read; g_T1, g_h, g_bias, g_S3 written
        by_bwd = 4.0 * (B * 3 * px + B * 4 * px + 12 * px + 3 * px2 + B * px2 + B * 3 * px2
                        + B * 3 * px + B * 4 * px + 12 * px + B * px2)
        leaves = [t.requires_grad_() for t in (t1, h, s3)]
        row = {"B": B, "fwd_bytes": by_fwd, "bwd_bytes": by_bwd}

        def ours_f():
            with torch.no_grad():
                _TexCompose.apply(t1, h, ob.weight_v, ob.weight_g, ob.bias, tm, s3, bt.TEX_STD)

        def ours_fb():
            out = _TexCompose.apply(leaves[0], leaves[1], ob.weight_v, ob.weight_g, ob.bias, tm, leaves[2], bt.TEX_STD)
            torch.autograd.grad(out, leaves + [ob.weight_v, ob.bias], gp)

        def torch_f():
            with torch.no_grad():
                bt.compose(t1, h, ob.weight_v, ob.weight_g, ob.bias, bt.TEX_STD, tm, s3)

        def torch_fb():
            out = bt.compose(leaves[0], leaves[1], ob.weight_v, ob.weight_g, ob.bias, bt.TEX_STD, tm, leaves[2])
            torch.autograd.grad(out, leaves + [ob.weight_v, ob.bias], gp)

        torch.backends.cudnn.allow_tf32 = False
        for name, f, fb in (("ours", ours_f, ours_fb), ("torch", torch_f, torch_fb)):
            row["fwd_ms_" + name] = timed(f, args.reps * 5)
            row["fwd_bwd_ms_" + name] = timed(fb, args.reps * 5)
            row["fwd_bwd_peak_MiB_" + name] = peak(fb)
        row["bwd_ms_ours"] = row["fwd_bwd_ms_ours"] - row["fwd_ms_ours"]
        row["fwd_share_of_bw_roof"] = by_fwd / (row["fwd_ms_ours"] * 1e-3) / 1e9 / HBM_GBS
        row["bwd_share_of_bw_roof"] = by_bwd / (row["bwd_ms_ours"] * 1e-3) / 1e9 / HBM_GBS
        rows.append(row)
    res["compose"] = rows
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
