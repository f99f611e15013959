"""Time the head avatar's frame `rgca.AutoEncoder` on the GPU at the rgca_example.yml configuration (slab 1024, so
1,048,576 Gaussians, 2048 x 1334 render; synthetic assets of tests/head_frame_restate.py, the constructor's
initial parameters):

  * eval point-light frame, B = 4, L = 460, with a per-stage breakdown (lights, encode, geometry decode, Gaussian
    decode, render, finish);
  * training forward + backward, B = 4, with a background;
  * the environment-map frame under EnvSpinDecorator, B = 2;
  * the light kernel alone (B = 4, L = 460) against its torch formula (fp32, sh.dir2sh), alternated in one loop.

Each case reports CUDA-event medians, this library's launch count per call and the peak memory.  The card name and
power limit are read in the same run.  Needs a GPU: without one it fails.

Usage: python scripts/profile_head_frame.py [--reps 10] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

H, W, SLAB = 2048, 1334, 1024


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def timed(fns, reps):
    """median ms of each callable, the callables alternated inside one timing loop"""
    for f in fns.values():
        for _ in range(2):
            f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ts[k].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in ts.items()}


def launches(fn):
    from goliath_b200 import _lib

    torch.cuda.synchronize()
    _lib.lib().gb_launch_count_reset()
    fn()
    torch.cuda.synchronize()
    return int(_lib.lib().gb_launch_count())


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import head_frame_restate as hr
    from goliath_b200.light_decorator import EnvSpinDecorator
    from goliath_b200.photo_loss import post_render
    from goliath_b200.rgca import AutoEncoder, head_lights
    from goliath_b200.sh import dir2sh

    dev = torch.device("cuda")
    out = {"card": card()}
    print("card: %s" % out["card"])
    torch.manual_seed(0)
    m = AutoEncoder(**hr.config(h=H, w=W, slab=SLAB), assets=hr.assets(slab=SLAB)).to(dev)
    todev = lambda d: {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in d.items()}
    B = 4
    inp = todev(hr.inputs(batch=B, h=H, w=W, slab=SLAB, n_active=(300, 460, 460, 200)))
    inp["camera_id"] = [hr.BATCH_CAMERAS[b % 2] for b in range(B)]

    # ---- eval point-light frame
    m.eval()

    def eval_frame():
        with torch.no_grad():
            return m(**inp)

    def stages():
        with torch.no_grad():
            lights = head_lights(inp["head_pose"], inp["campos"], inp["Rt"], inp["light_pos"], inp["light_intensity"])
            enc = m.encoder(inp["registration_vertices"], inp["color"])
            geom = m.geomdecoder(enc["embs"])["face_geom"]
            dec = m.decoder(enc["embs"], geom, lights["headrel_campos"], inp["light_intensity"].expand(-1, -1, 3),
                            lights["headrel_light_pos"], lights["headrel_light_sh"], inp["n_lights"])
            rgb, alpha, _ = m.render(inp["K"], lights["headrel_Rt"], dec)
            w, b, grey = m.cal.rows(m.cal.name_to_idx(inp["camera_id"]))
            post_render(rgb, None, None, w, b, grey, m.learn_blur.weights(inp["camera_id"]))
            return lights, enc, geom, dec, rgb

    lights, enc, geom, dec, rgb = stages()
    with torch.no_grad():
        st = timed({
            "frame": eval_frame,
            "lights": lambda: head_lights(inp["head_pose"], inp["campos"], inp["Rt"], inp["light_pos"],
                                          inp["light_intensity"]),
            "encode": lambda: m.encoder(inp["registration_vertices"], inp["color"]),
            "geom_decode": lambda: m.geomdecoder(enc["embs"]),
            "prim_decode": lambda: m.decoder(enc["embs"], geom, lights["headrel_campos"],
                                             inp["light_intensity"].expand(-1, -1, 3), lights["headrel_light_pos"],
                                             lights["headrel_light_sh"], inp["n_lights"]),
            "render": lambda: m.render(inp["K"], lights["headrel_Rt"], dec),
            "finish": lambda: post_render(rgb, None, None, *m.cal.rows(m.cal.name_to_idx(inp["camera_id"])),
                                          m.learn_blur.weights(inp["camera_id"])),
        }, args.reps)
    out["eval_point_light_B4"] = {"ms": st, "launches": launches(eval_frame), "peak_gib": peak(eval_frame)}
    print("eval point-light frame, B = 4, L = 460: %s" % json.dumps(out["eval_point_light_B4"]))

    # ---- training forward + backward
    m.train()
    tin = dict(inp)
    tin["background"] = torch.rand(B, 3, H, W, device=dev)
    tin["is_fully_lit_frame"] = torch.tensor([True, False, True, False], device=dev)

    def train_step():
        m.zero_grad(set_to_none=True)
        p = m(**tin)
        p["rgb"].square().mean().backward()

    t = timed({"fwd_bwd": train_step}, args.reps)
    out["train_B4"] = {"ms": t, "launches": launches(train_step), "peak_gib": peak(train_step)}
    print("training forward + backward, B = 4: %s" % json.dumps(out["train_B4"]))
    m.zero_grad(set_to_none=True)
    del tin

    # ---- environment-map frame under EnvSpinDecorator
    m.eval()
    m.cal_enabled, m.learn_blur_enabled = False, False   # as run_vis_relight.py sets them
    probe = np.random.default_rng(2).uniform(0.0, 4.0, (512, 1024, 3)).astype(np.float32)
    env = EnvSpinDecorator(m, probe).to(dev)
    ein = {k: (v[:2] if torch.is_tensor(v) else v) for k, v in inp.items()}
    ein["camera_id"] = ein["camera_id"][:2]
    ein["index"] = [0, 64]

    def env_frame():
        with torch.no_grad():
            return env(**dict(ein))

    t = timed({"frame": env_frame}, args.reps)
    out["envmap_B2"] = {"ms": t, "launches": launches(env_frame), "peak_gib": peak(env_frame)}
    print("environment-map frame under EnvSpinDecorator, B = 2: %s" % json.dumps(out["envmap_B2"]))
    m.cal_enabled, m.learn_blur_enabled = True, True

    # ---- the light kernel against its torch formula
    def torch_lights():
        hp = inp["head_pose"]
        hp4 = torch.cat([hp, torch.zeros_like(hp[:, :1, :])], 1)
        hp4[:, 3, 3] = 1.0
        hrt = inp["Rt"] @ hp4
        hc = ((inp["campos"] - hp[:, :3, 3])[:, None] @ hp[:, :3, :3])[:, 0]
        hl = (inp["light_pos"] - hp[:, None, :3, 3]) @ hp[:, :3, :3]
        sh = dir2sh(8, F.normalize(hl, p=2, dim=-1))
        return hrt, hc, hl, (sh[:, :, None] * inp["light_intensity"].expand(-1, -1, 3)[..., None]).sum(1)

    kern = lambda: head_lights(inp["head_pose"], inp["campos"], inp["Rt"], inp["light_pos"], inp["light_intensity"])
    t = timed({"kernel": kern, "torch": torch_lights}, max(args.reps, 50))
    out["light_kernel_B4_L460"] = {"ms": t, "launches_kernel": launches(kern)}
    print("light kernel alone, B = 4, L = 460: %s" % json.dumps(out["light_kernel_B4_L460"]))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
