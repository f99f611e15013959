"""Time the relightable hand teacher's frame `hand_teacher.AutoEncoder` on the GPU at hand_teacher_mvp_example.yml's
configuration (B = 1, the example's batch size, at 1024 x 667: 2048 x 1334 at the data loader's downsample of 2;
1024^2 shadow images, chunks of 5 lights), synthetic assets of tests/hand_frame_restate.py and seeded parameters:

  * point: the eval frame of run_vis_relight's point-light cycle (SingleLightCycleDecorator, one light), forward;
  * train: one training step with L = 6 lights (a chunk of 5 and one of 1) and the background, forward + backward;
  * env:   the eval frame of the environment spin (EnvSpinDecorator: 512 lights, 103 chunks, and the `envbg`
           composite), forward.

Whole frames are timed with CUDA events (medians).  Each configuration's forward is also split into stages by CUDA
events recorded between them on one stream: per chunk of lights the decoder's shadow march, features, U-Net and OLAT
compose (summed over the chunks), then the template, the march, the finish and the environment composite; the
encoders and the geometry decoder are `front`.  The card name and power limit are read in the same run.  Needs a GPU:
without one it fails.

Usage: python scripts/profile_hand_teacher_frame.py [--reps 5] [--out DIR]   (writes DIR/hand_teacher_frame.json)"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

B, H, W = 1, 667, 1024


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


class _Marks:
    """CUDA events between stages; `split()` sums the time of each stage name"""

    def __init__(self):
        self.ev = [("start", torch.cuda.Event(enable_timing=True))]
        self.ev[0][1].record()

    def mark(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.ev.append((name, e))

    def split(self):
        torch.cuda.synchronize()
        out = {}
        for (_, a), (name, b) in zip(self.ev, self.ev[1:]):
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
        return out


def staged_forward(m, d):
    """hand_teacher.AutoEncoder.forward on the same stages, with an event after each"""
    from goliath_b200.envmap import compose_envmap
    from goliath_b200.hand_mvp import slabs_to_primrgba
    from goliath_b200.hand_teacher import _colour_intensity, olat_compose

    t = _Marks()
    joint = m.poseencoder(d["pose"])
    geo = m.geomdecoder(d["pose"], joint, 5000)
    joint2 = m.poseencoder2(d["pose"])
    t.mark("front")
    dec = m.relightdecoder
    prims = dec._prims(geo["primpos"], geo["primrot"], geo["primscale"], geo["primalpha"], m.valid_prims)
    t.mark("decoder_prims")
    lpos, lint = d["light_pos"], _colour_intensity(d["light_intensity"])
    rgb = primshadow = None
    L = lpos.shape[1]
    n = (L - 1) // dec.chunksize + 1
    for i in range(n):
        sl = slice(i * dec.chunksize, (i + 1) * dec.chunksize)
        shadow = dec.shadow_march(prims, lpos[:, sl])
        t.mark("decoder_shadow_march")
        x, primshadow, _ = dec.features(prims, d["campos"], lpos[:, sl], shadow, primshadow)
        del shadow
        t.mark("decoder_features")
        tex = dec.unet(x, joint2, lpos[:, sl].shape[1])
        t.mark("decoder_unet")
        rgb, _ = olat_compose(tex, lint[:, sl], dec.primsize[2], None, rgb, want_texolat=m.training and i == n - 1)
        t.mark("decoder_compose")
    preds = {"primrgb": rgb, "primalpha": geo["primalpha"], "primpos": geo["primpos"], "primrot": geo["primrot"],
             "primscale": geo["primscale"]}
    preds["primrgba"] = slabs_to_primrgba(rgb, geo["primalpha"], m.primsize)
    t.mark("template")
    ray = m._march(d["K"], d["Rt"], preds)
    t.mark("march")
    out, alpha = m._finish(ray, d.get("camera_id"), d.get("background"))
    t.mark("finish")
    if "envbg" in d:
        out = compose_envmap(out / 255.0, alpha, d["envbg"], d["K"], d["Rt"])
        t.mark("envmap_compose")
    if m.learn_blur_enabled:
        out = m.learn_blur(out, d.get("camera_id"))
        t.mark("blur")
    return t.split()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="hand_teacher_frame_profile")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_hand_teacher_frame needs a GPU")
    import hand_frame_restate as hf
    import hand_teacher_frame_restate as ht
    from goliath_b200.hand_teacher import AutoEncoder
    from goliath_b200.light_decorator import EnvSpinDecorator, single_light_position

    spec = importlib.util.spec_from_file_location("make_envspin_golden",
                                                  os.path.join(ROOT, "tests", "golden", "make_envspin_golden.py"))
    envspin = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(envspin)

    dev = torch.device("cuda")
    m = hf.seeded_fill(AutoEncoder(**hf.config(H, W), assets=hf.assets())).to(dev)
    pose = 0.05 * torch.randn(B, 12, generator=torch.Generator().manual_seed(7))
    with torch.no_grad():
        posed = m.lbs_fn.pose(torch.zeros_like(m.lbs_fn.lbs_template_verts), pose.to(dev)).cpu().double()
    K, Rt, campos = hf.side_cameras(posed, H, W)
    base = {"pose": pose.to(dev), "campos": campos.float().to(dev), "K": K.float().to(dev), "Rt": Rt.float().to(dev),
            "camera_id": hf.BATCH_CAMERAS[:B]}
    res = {"card": card(), "B": B, "H": H, "W": W, "n_valid": m.n_valid}

    # point-light eval frame: SingleLightCycleDecorator's light (axis 1) at frame 180
    lp = single_light_position(180, 256, 1, pose[0, :3].numpy())
    point = dict(base, light_pos=torch.from_numpy(lp).float().to(dev)[None, None].expand(B, 1, 3).contiguous(),
                 light_intensity=torch.ones(B, 1, 1, device=dev))
    m.eval()
    with torch.no_grad():
        res["point_eval_fwd_ms"] = timed(lambda: m(**point, iteration=5000), args.reps)
        res["point_eval_stages_ms"] = staged_forward(m, point)

    # training step, L = 6
    light_pos, light_int = ht.lights(posed, n=6, batch=B)
    train = dict(base, light_pos=light_pos.to(dev), light_intensity=light_int.to(dev),
                 background=hf.background(B, H, W).to(dev))
    params = [p for p in m.parameters() if p.requires_grad]

    def step():
        p = m(**train, iteration=5000)
        loss = ((p["rgb"] - 128.0) ** 2).mean() + p["texolat"].clamp(max=0.0).pow(2).mean()
        torch.autograd.grad(loss, params, allow_unused=True)

    m.train()
    torch.cuda.reset_peak_memory_stats()
    res["train_L6_fwd_bwd_ms"] = timed(step, args.reps)
    res["train_L6_peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    res["train_L6_fwd_stages_ms"] = staged_forward(m, train)
    m.eval()

    # env-lit eval frame, 512 lights
    env = dict(base)
    got = {}
    EnvSpinDecorator(lambda **d: got.update(d), envspin.probe(), **envspin.DECORATOR)(**env, index=[5])
    env = {k: got[k] for k in ("pose", "campos", "K", "Rt", "camera_id", "light_pos", "light_intensity", "envbg")}
    with torch.no_grad():
        res["env_eval_fwd_ms"] = timed(lambda: m(**env, iteration=5000), max(1, args.reps // 2))
        res["env_eval_stages_ms"] = staged_forward(m, env)
    res["env_lights"] = int(env["light_pos"].shape[1])
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "hand_teacher_frame.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
