"""Time the environment-map relighting frame on the GPU against the reference's torch formulation.

* compose_envmap (csrc/envmap_compose.cu: bicubic lookup + two 101-tap blur passes + composite) against the reference's
  formulation on the same device (bicubic grid_sample, dense 101x101 depthwise conv2d in fp32, elementwise composite),
  B = 2 at 1024x667 and 2048x1334;
* render_views_envmap (three colour sets against one projection and one binning per view + compose) against three
  render_views calls + the torch compose, on bench.py's head scene (300k Gaussians, two ring cameras, 1024x667).

Prints the device name and power limit, per-call times from CUDA events (median of the timed calls after a warm-up)
and max |diff| for each pair.  Usage: python scripts/profile_envmap.py [--reps N]
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from goliath_b200 import synthetic  # noqa: E402
from goliath_b200.envmap import compose_envmap  # noqa: E402
from goliath_b200.render import render_views, render_views_envmap  # noqa: E402
from test_envmap_compose_gpu import golden, torch_compose  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), out


def maxdiff(a, b):
    return float((a - b).abs().max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    print("device: %s" % card())
    rng = np.random.default_rng(0)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    for H, W in ((1024, 667), (2048, 1334)):
        f = 3300.0 * W / 1334.0
        cams = [golden._camera(golden._random_rot(rng), f, f, W / 2.0, H / 2.0) for _ in range(2)]
        x = [d(golden._smooth(rng, (2, 3, H, W), 0.0, 1.0)), d(golden._smooth(rng, (2, 1, H, W), 0.0, 1.0)),
             d(golden._smooth(rng, (2, 3, 256, 512), 0.0, 2.5)), d(np.stack([c[0] for c in cams])),
             d(np.stack([c[1] for c in cams]))]
        with torch.no_grad():
            t_ours, ours = timed(lambda: compose_envmap(*x), args.reps)
            t_ref, ref = timed(lambda: torch_compose(*x), max(2, args.reps // 5), warmup=1)
        print("compose_envmap B=2 %dx%d: ours %.3f ms, torch formulation %.3f ms (x%.1f), max|diff| %.2e"
              % (H, W, t_ours, t_ref, t_ref / t_ours, maxdiff(ours, ref)))

    H, W, G = 1024, 667, 300_000
    sc = {k: v.to(dev) for k, v in synthetic.head_gaussians(G).items()}
    cams = [synthetic.ring_camera(k, img_h=H, img_w=W) for k in (0, 5)]
    intr = [(c["fx"], c["fy"], c["cx"], c["cy"]) for c in cams]
    K = d(np.stack([np.array([[c["fx"], 0, c["cx"]], [0, c["fy"], c["cy"]], [0, 0, 1]], np.float32) for c in cams]))
    Rt = torch.stack([c["viewmat"] for c in cams]).to(dev)
    rep = lambda t: t[None].expand(2, *t.shape).contiguous()
    gen = torch.Generator(device="cpu").manual_seed(1)
    preds = dict(primpos=rep(sc["means3d"]), primscale=rep(sc["scales"]), primqvec=rep(sc["quats"]),
                 opacity=rep(sc["opacity"]), color=rep(sc["colors"]),
                 diff_color=rep(torch.randn(G, 3, generator=gen).to(dev)),
                 spec_color=rep(0.2 * torch.randn(G, 3, generator=gen).to(dev)))
    envbg = d(golden._smooth(rng, (2, 3, 256, 512), 0.0, 2.5))
    cap = 8 * G

    def three_renders():
        out = []
        for k, col in (("color", preds["color"]), ("diff_color", preds["diff_color"].clamp(min=0.0)),
                       ("spec_color", preds["spec_color"].clamp(min=0.0))):
            p = dict(preds, color=col)
            rgb, alpha, depth = render_views(W, H, K, Rt, p, intrinsics_host=intr, capacity=cap)
            out.append(torch_compose(rgb, alpha, envbg, K, Rt) if k == "color" else rgb)
        return torch.cat(out, -1), alpha, depth

    with torch.no_grad():
        t_ours, ours = timed(lambda: render_views_envmap(W, H, K, Rt, Rt, preds, envbg, intrinsics_host=intr,
                                                         capacity=cap), args.reps)
        t_ref, ref = timed(three_renders, max(2, args.reps // 5), warmup=1)
    print("render_views_envmap B=2 %dx%d G=%d: ours %.3f ms, 3x render_views + torch compose %.3f ms (x%.1f); "
          "max|diff| rgb %.2e alpha %.2e depth %.2e"
          % (H, W, G, t_ours, t_ref, t_ref / t_ours, maxdiff(ours[0], ref[0]), maxdiff(ours[1], ref[1]),
             maxdiff(ours[2], ref[2])))


if __name__ == "__main__":
    main()
