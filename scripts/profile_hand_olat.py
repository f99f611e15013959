"""Per-stage time and peak memory of the relightable hand teacher's `OLATRGBDecoder` at the config's shapes (B = 1,
4096 primitives of 8 x 16 x 16 voxels, 1024^2 shadow images, uv 1024), L = 5 and L = 10, against the reference's
formulation built from this repository's own pieces: the expanded [B*L, K, 8, 16, 16, 4] template through
`mvpraymarch(with_shadow=True)`, the feature block as torch ops, the same U-Net layers and the compose in torch.

    python scripts/profile_hand_olat.py [--reps 5] [--out hand_olat.json]

Times are CUDA events over `--reps` calls after a warm-up, per chunk of 5 lights except `step` (forward + backward of
the whole decoder over all L lights).  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    from goliath_b200.hand_teacher import light_cameras, olat_compose
    from goliath_b200.mvpraymarch import mvpraymarch
    from goliath_b200.utils import compute_raydirs
    from test_hand_olat_gpu import _features_torch, _full_decoder, _hand_scene

    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "reps": args.reps, "runs": []}
    dec = _full_decoder(dev).train()
    B, K, Z, U = 1, 4096, 8, 1024
    for L in (5, 10):
        s = _hand_scene(dev, B=B, L=L)
        joint = torch.randn(B, 64, 64, 64, device=dev, requires_grad=True)
        lp5, li5 = s["light_pos"][:, :5].contiguous(), s["light_intensity"][:, :5]
        r = {"L": L}
        with torch.no_grad():
            prims = dec._prims(s["primpos"], s["primrot"], s["primscale"], s["primalpha"], s["valid_prims"])
            r["prims_ms"] = timed(lambda: dec._prims(s["primpos"], s["primrot"], s["primscale"], s["primalpha"],
                                                     s["valid_prims"]), args.reps)
            r["shadow_march_ms"] = timed(lambda: dec.shadow_march(prims, lp5), args.reps)
            r["shadow_march_peak_mib"] = peak(lambda: dec.shadow_march(prims, lp5))
            shadow = dec.shadow_march(prims, lp5)
            r["features_ms"] = timed(lambda: dec.features(prims, s["campos"], lp5, shadow), args.reps)
            x = dec.features(prims, s["campos"], lp5, shadow)[0]
        tex = dec.unet(x, joint, 5)
        g = torch.randn_like(tex)
        r["unet_fwd_ms"] = timed(lambda: dec.unet(x, joint, 5), args.reps)
        r["unet_bwd_ms"] = timed(lambda: tex.backward(g, retain_graph=True), args.reps)
        texd = tex.detach().requires_grad_()
        rgb, texolat = olat_compose(texd, li5, Z, want_texolat=True)
        g_rgb, g_tol = torch.randn_like(rgb), torch.randn_like(texolat)
        r["compose_fwd_ms"] = timed(lambda: olat_compose(texd, li5, Z, want_texolat=True), args.reps)
        r["compose_bwd_ms"] = timed(lambda: torch.autograd.backward([rgb, texolat], [g_rgb, g_tol], retain_graph=True),
                                    args.reps)
        del tex, g, texd, rgb, texolat, g_rgb, g_tol, shadow, x

        def step():
            out = dec(s["campos"], None, None, s["primpos"], s["primrot"], s["primscale"], s["primalpha"],
                      s["valid_prims"], joint, s["light_pos"], s["light_intensity"], 5000)
            (out["primrgb"].sum() + out["texolat"].sum()).backward()

        r["step_ms"] = timed(step, args.reps)
        r["step_peak_mib"] = peak(step)

        # the reference's formulation, per chunk of 5 lights, on this repository's kernels and torch
        def ref_march():
            alpha = s["primalpha"].reshape(B, 8, 1, 64, 16, 64, 16).permute(0, 3, 5, 1, 4, 6, 2)
            alpha = alpha[:, None].expand(-1, 5, -1, -1, -1, -1, -1, -1).reshape(B * 5, K, 8, 16, 16, 1)
            alpha = s["valid_prims"][None, :, None, None, None, None] * alpha
            tpl = torch.cat([torch.ones(B * 5, K, 8, 16, 16, 3, device=dev) * 255.0, alpha], -1)
            lpos, lrot, focal, princpt = light_cameras(s["primpos"], s["valid_prims"], lp5, 1024, 1024)
            pix = torch.cat(B * 5 * [dec.pixel_coords[None]], 0)
            raypos, raydir, tminmax = compute_raydirs(lpos, lrot, focal, princpt, pix, 2000.0)
            ex = lambda t: t[:, None].expand(B, 5, *t.shape[1:]).reshape(B * 5, *t.shape[1:]).contiguous()
            return mvpraymarch(raypos, raydir, 1.0 / 2000.0, tminmax,
                               (ex(s["primpos"] / 2000.0), ex(s["primrot"]), ex(s["primscale"])), tpl, None,
                               with_shadow=True)[1]

        with torch.no_grad():
            r["ref_shadow_march_ms"] = timed(ref_march, args.reps)
            r["ref_shadow_march_peak_mib"] = peak(ref_march)
            raw = torch.cat([ref_march(), torch.ones(B * 5, K, 8, 16, 16, 1, device=dev)], -1)
            r["ref_features_ms"] = timed(lambda: _features_torch(
                s["primpos"], s["primrot"], s["primscale"], s["valid_prims"], lp5, s["campos"], raw, 2000.0, 16, 16,
                8, 64, 64), args.reps)
            del raw

        def ref_compose():
            t = texd2.view(B, 5, Z, 4, U, U)
            rgb = (torch.sigmoid(t[:, :, :, :1]) * F.relu(25.0 * t[:, :, :, 1:] + 100.0)
                   * li5[:, :, None, :, None, None]).sum(1)
            rgb.sum().backward()

        texd2 = torch.randn(B * 5, 4 * Z, U, U, device=dev, requires_grad=True)
        r["ref_compose_fwd_bwd_ms"] = timed(ref_compose, args.reps)
        del texd2
        res["runs"].append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps({"gpu": gpu}))


if __name__ == "__main__":
    main()
