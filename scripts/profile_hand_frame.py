"""Time the hand avatar's frame `hand_mvp.AutoEncoder` on the GPU at hand_mvp_example.yml's configuration with
B = 8 cameras at 1024 x 667 (the example's 2048 x 1334 at the data loader's downsample of 2), synthetic assets of
tests/hand_frame_restate.py and seeded parameters: forward + backward in eval and in training (with the background),
CUDA events, medians; the launches of this library per step, peak memory, and the two kernels of csrc/hand_frame.cu
(valid gather, render finish) forward + backward on the frame's tensors.  The card name and power limit are read in
the same run.  No reference baseline is timed.  Needs a GPU: without one it fails.

Usage: python scripts/profile_hand_frame.py [--reps 10] [--out DIR]   (writes DIR/hand_frame.json)"""
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

B, H, W = 8, 667, 1024


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def timed(fn, reps):
    for _ in range(2):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="hand_frame_profile")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_hand_frame needs a GPU")
    import hand_frame_restate as hf
    from goliath_b200 import _lib
    from goliath_b200.hand_mvp import AutoEncoder, hand_finish, valid_gather

    dev = torch.device("cuda")
    m = hf.seeded_fill(AutoEncoder(**hf.config(H, W), assets=hf.assets())).to(dev)
    g = torch.Generator().manual_seed(7)
    pose = 0.05 * torch.randn(B, 12, generator=g)
    with torch.no_grad():
        posed = m.lbs_fn.pose(torch.zeros_like(m.lbs_fn.lbs_template_verts), pose.to(dev)).cpu().double()
    K, Rt, campos = hf.side_cameras(posed, H, W)
    inp = {"pose": pose.to(dev), "campos": campos.float().to(dev), "K": K.float().to(dev), "Rt": Rt.float().to(dev),
           "ambient_occlusion": torch.rand(B, 1, 128, 128, generator=g).to(dev),
           "camera_id": (hf.BATCH_CAMERAS * B)[:B], "background": hf.background(B, H, W).to(dev)}
    params = [p for p in m.parameters() if p.requires_grad]

    def step():
        p = m(**inp, iteration=5000)
        torch.autograd.grad(p["rgb"].sum() + p["alpha"].sum(), params, allow_unused=True)

    res = {"card": card(), "B": B, "H": H, "W": W, "n_valid": m.n_valid}
    for mode in ("eval", "train"):
        m.train(mode == "train")
        torch.cuda.reset_peak_memory_stats()
        res["%s_fwd_bwd_ms" % mode] = timed(step, args.reps)
        res["%s_peak_gib" % mode] = torch.cuda.max_memory_allocated() / 2 ** 30
        L = _lib.lib()
        torch.cuda.synchronize()
        L.gb_launch_count_reset()
        step()
        torch.cuda.synchronize()
        res["%s_launches_per_step" % mode] = int(L.gb_launch_count())
    m.eval()

    # the two kernels on the frame's shapes
    tpl = torch.rand(B, m.n_prims, 8, 16, 16, 4, device=dev, requires_grad=True)
    tr = [torch.rand(B, m.n_prims, *s, device=dev, requires_grad=True) for s in ((3,), (3, 3), (3,))]
    outs = valid_gather(tpl, *tr, m.valid_slot, m.n_valid, 2000.0)
    cots = [torch.rand_like(o) for o in outs]
    res["gather_fwd_ms"] = timed(lambda: valid_gather(tpl, *tr, m.valid_slot, m.n_valid, 2000.0), args.reps)
    res["gather_fwd_bwd_ms"] = timed(lambda: torch.autograd.grad(
        valid_gather(tpl, *tr, m.valid_slot, m.n_valid, 2000.0), [tpl] + tr, cots), args.reps)
    del tpl, tr, outs, cots
    ray = torch.rand(B, H, W, 4, device=dev, requires_grad=True)
    w = torch.rand(B, 3, device=dev, requires_grad=True)
    b = torch.rand(B, 3, device=dev, requires_grad=True)
    grey = (torch.arange(B, device=dev) % 2).to(torch.int32)
    bg = inp["background"]
    res["finish_fwd_ms"] = timed(lambda: hand_finish(ray, w, b, grey, bg), args.reps)
    res["finish_fwd_bwd_ms"] = timed(lambda: torch.autograd.grad(
        sum(t.sum() for t in hand_finish(ray, w, b, grey, bg)), [ray, w, b]), args.reps)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "hand_frame.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
