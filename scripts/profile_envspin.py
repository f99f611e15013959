"""Time the environment-spin lighting (goliath_b200.light_decorator.EnvSpinDecorator, csrc/envmap_prefilter.cu) on the
GPU against the reference's formulation, in one run:

* the per-frame decorator work (light table, envbg, the scaled mip chain, the dict) at B = 1 and B = 4: ours against
  the reference's formulation with the probe on the host, as run_vis_relight.py has it (per item: rotate_envmap_mat on
  the CPU, np.percentile of the probe, the antialiased resize, the sin-weighted normalisation; then the host-to-device
  copies).  Wall time per frame around work that ends in a device synchronise, median of the timed frames;
* the SG prefilter at the decorator's sizes (256x512, 128x256, 64x128 at sigma 0.2, 0.4, 0.6) with 4096 samples: our
  one launch against the torch restatement of tests/test_envspin_gpu.py run one sample per pass, as prefilterEnvmapSG
  does;
* decorator + render_views_envmap on bench.py's head scene (300k Gaussians, 1024x667, B = 2 ring cameras), with our
  decorator and with the reference formulation.

Prints the device name and power limit beside the numbers.  Usage: python scripts/profile_envspin.py [--reps N]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from goliath_b200 import synthetic  # noqa: E402
from goliath_b200.envmap import _prefilter_levels, rotate_envmap_mat  # noqa: E402
from goliath_b200.light_decorator import EnvSpinDecorator  # noqa: E402
from goliath_b200.render import render_views_envmap  # noqa: E402
from test_envspin_gpu import _decorator_levels, golden, torch_prefilter  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def wall(fn, reps, warmup=2):
    """median wall time (ms) of fn() followed by a device synchronise"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts)), out


def reference_frame(dec, device, index):
    """EnvSpinDecorator.forward's per-frame work as the reference formulates it: the probe on the host, one item at a
    time, then the copies to the device"""
    B = len(index)
    image = dec.image_host
    rots, envbg, envmaps, li, ns = [], [], [], [], []
    for i in range(B):
        a = torch.tensor(2.0 * np.pi * index[i] / dec.cycle, dtype=torch.float32)
        R = torch.eye(3)
        n = a.abs().clamp(min=1e-6)
        N = torch.zeros(3, 3)
        N[0, 2], N[2, 0] = a / n, -a / n
        R = R + torch.sin(n) * N + ((1 - torch.cos(n)) * N) @ N
        rot = rotate_envmap_cpu(image, R)
        perc90 = np.percentile(image.numpy(), 90)
        envbg.append(rot / perc90 * 255)
        down = F.interpolate(rot[None], (16, 32), mode="bilinear", antialias=True)[0]
        s = (down * torch.sin((torch.arange(16) + 0.5) * np.pi / 16)[None, :, None]).sum()
        env = dec.env_scale * down / s
        ns.append(dec.env_scale / s)
        rots.append(R)
        envmaps.append(env)
        li.append(env.view(3, -1).t())
    data = dict(lightrot=torch.stack(rots).to(device), envmap=torch.stack(envmaps).to(device),
                light_intensity=torch.stack(li).to(device), envbg=torch.stack(envbg).to(device) / 255.0)
    data["preconv_envmap"] = dec.mipmap(B, device, 2.0 * np.pi * ns[0])
    data["light_pos"] = dec.envmap_dist * dec.sphvec.view(3, -1).t()[None].expand(B, -1, -1).to(device)
    data["n_lights"] = 512 * torch.ones(B, 1, device=device)
    return data


def rotate_envmap_cpu(image, R):
    """rotate_envmap_mat (ca_code/utils/envmap.py:141-166) in torch on the host"""
    H, W = image.shape[1:]
    theta, phi = torch.meshgrid((torch.arange(H, dtype=torch.float32) + 0.5) * 3.1415926 / H,
                                (torch.arange(-W // 2, W // 2, dtype=torch.float32) + 0.5) * 3.1415926 * 2 / W,
                                indexing="ij")
    vec = torch.stack([torch.sin(theta) * torch.sin(phi), torch.cos(theta), torch.sin(theta) * torch.cos(phi)], -1)
    vec = torch.clamp(vec @ R.T.contiguous()[None], -1, 1)
    uv = torch.stack([(1 / np.pi) * torch.atan2(vec[..., 0], vec[..., 2]),
                      2 * ((1 / np.pi) * torch.acos(vec[..., 1])) - 1.0], -1)
    return F.grid_sample(image[None], uv[None], padding_mode="border", align_corners=False)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    print("device: %s" % card())

    dec = EnvSpinDecorator(lambda **d: d, golden.probe(), **golden.DECORATOR)
    dec.image_host = dec.image.cpu()
    for B in (1, 4):
        index = [37 + 50 * i for i in range(B)]
        data = dict(campos=torch.zeros(B, 3, device=dev), index=index)
        with torch.no_grad():
            t_ours, ours = wall(lambda: dec(**dict(data)), args.reps)
            t_ref, ref = wall(lambda: reference_frame(dec, dev, index), max(3, args.reps // 4), warmup=1)
        diff = max(float((ours[k] - ref[k]).abs().max()) for k in ("lightrot", "envmap", "light_intensity", "envbg"))
        print("decorator frame B=%d: ours %.3f ms, reference formulation (host probe) %.3f ms (x%.1f), max|diff| %.2e"
              % (B, t_ours, t_ref, t_ref / t_ours, diff))

    S = 4096
    levels = _decorator_levels(dev)
    t_ours, ours = wall(lambda: _prefilter_levels([lv + (None,) for lv in levels], S, seed=1), args.reps)
    t_ref, ref = wall(lambda: [torch_prefilter(s, v, e, S, chunk=1)[0] for s, v, e in levels], 1, warmup=0)
    print("prefilter 256x512 + 128x256 + 64x128, %d samples: ours %.3f ms, torch restatement one sample per pass "
          "%.1f ms (x%.0f), max|diff| (Monte-Carlo) %.2e"
          % (S, t_ours, t_ref, t_ref / t_ours, max(float((a - b).abs().max()) for a, b in zip(ours, ref))))

    H, W, G = 1024, 667, 300_000
    sc = {k: v.to(dev) for k, v in synthetic.head_gaussians(G).items()}
    cams = [synthetic.ring_camera(k, img_h=H, img_w=W) for k in (0, 5)]
    intr = [(c["fx"], c["fy"], c["cx"], c["cy"]) for c in cams]
    K = torch.tensor(np.stack([np.array([[c["fx"], 0, c["cx"]], [0, c["fy"], c["cy"]], [0, 0, 1]], np.float32)
                               for c in cams])).to(dev)
    Rt = torch.stack([c["viewmat"] for c in cams]).to(dev)
    rep = lambda t: t[None].expand(2, *t.shape).contiguous()
    gen = torch.Generator(device="cpu").manual_seed(1)
    preds = dict(primpos=rep(sc["means3d"]), primscale=rep(sc["scales"]), primqvec=rep(sc["quats"]),
                 opacity=rep(sc["opacity"]), color=rep(sc["colors"]),
                 diff_color=rep(torch.randn(G, 3, generator=gen).to(dev)),
                 spec_color=rep(0.2 * torch.randn(G, 3, generator=gen).to(dev)))
    render = lambda d: render_views_envmap(W, H, K, Rt, Rt, preds, d["envbg"], intrinsics_host=intr, capacity=8 * G)
    dec.mod = lambda **d: render(d)
    data = dict(campos=torch.zeros(2, 3, device=dev), index=[37, 129])
    with torch.no_grad():
        t_ours, _ = wall(lambda: dec(**dict(data)), args.reps)
        t_ref, _ = wall(lambda: render(reference_frame(dec, dev, data["index"])), max(3, args.reps // 4), warmup=1)
    print("decorator + render_views_envmap B=2 %dx%d G=%d: ours %.3f ms, reference decorator formulation + "
          "render_views_envmap %.3f ms (x%.1f)" % (H, W, G, t_ours, t_ref, t_ref / t_ours))


if __name__ == "__main__":
    main()
