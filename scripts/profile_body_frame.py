"""Time the body avatar's frame `mesh_vae.AutoEncoder` on the GPU at the mesh_vae_example.yml configuration with its
2048 x 1334 render (synthetic assets of tests/body_frame_restate.py, seeded parameters, eval mode): the forward at
B = 1 and forward + backward at B = 4 (CUDA events, medians), a per-stage breakdown of the B = 1 forward (encode,
decode, pose, view, shadow, texture, cal, render, finish = depth mask + blur + pixel bias), peak memory, this
library's launch counts, and the two kernels of csrc/body_frame.cu against their torch formulation, alternated in one
loop.  The card name and power limit are read in the same run.  There is no end-to-end reference baseline: the
reference renders through drtk, which is not available.  Needs a GPU: without one it fails.

Usage: python scripts/profile_body_frame.py [--reps 10] [--json out.json]"""
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

H, W, DS = 2048, 1334, 8


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


def frame_inputs(m, B, dev, seed=7):
    import body_frame_restate as bf

    g = torch.Generator().manual_seed(seed)
    P = m.lbs_fn.lbs_fn.param_transform.transform.shape[1] - m.lbs_fn.lbs_scale.shape[-1]
    V = m.lbs_fn.lbs_template_verts.shape[0]
    pose = (0.3 * torch.randn(B, P, generator=g)).to(dev)
    with torch.no_grad():
        posed = m.lbs_fn.pose(torch.zeros(B, V, 3, device=dev), pose)
    K, Rt, campos = bf.look_at(posed.cpu(), H, W)
    return {"pose": pose, "campos": campos.to(dev), "registration_vertices": posed + 0.5 * torch.randn_like(posed),
            "ambient_occlusion": bf.ambient_occlusion(B).to(dev), "K": K.to(dev), "Rt": Rt.to(dev),
            "camera_id": (bf.BATCH_CAMERAS * B)[:B]}


def staged(m, inp):
    """AutoEncoder.forward with an event after each stage; returns ms per stage"""
    from goliath_b200.geom import depth_discontuity_mask
    from goliath_b200.mesh_vae import encode

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(10)]
    ev[0].record()
    enc = encode(m.lbs_fn, m.geo_fn, m.encoder, m.encoder_face, inp["registration_vertices"], inp["pose"])
    ev[1].record()
    dec = m.decoder(pose=inp["pose"], embs=enc["embs"], face_embs=enc["face_embs"])
    ev[2].record()
    geom = m.lbs_fn.pose(dec["geom_delta_rec"], inp["pose"])
    ev[3].record()
    view = m.decoder_view(geom_rec=geom, tex_mean_rec=dec["tex_mean_rec"], camera_pos=inp["campos"])
    ev[4].record()
    shadow = m.shadow_net(ao_map=inp["ambient_occlusion"])
    ev[5].record()
    tex = m.forward_tex(dec["tex_mean_rec"], view["tex_view_rec"], shadow["shadow_map"])
    ev[6].record()
    idx = m.cal.name_to_idx(inp["camera_id"])
    tex = m.cal(tex, idx)
    ev[7].record()
    r = m.renderer(geom, tex=torch.cat([tex, torch.ones_like(tex[:, :1])], 1), K=inp["K"], Rt=inp["Rt"])
    ev[8].record()
    depth_discontuity_mask(r["depth_img"][:, None].detach())
    rgb = m.learn_blur(r["render"][:, :3], inp["camera_id"])
    m.learn_blur.reg(inp["camera_id"])
    m.pixel_cal(idx, rgb)
    ev[9].record()
    torch.cuda.synchronize()
    names = ["encode", "decode", "pose", "view", "shadow", "texture", "cal", "render", "finish"]
    return {n: ev[i].elapsed_time(ev[i + 1]) for i, n in enumerate(names)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_body_frame.py needs a CUDA device")
    import body_frame_restate as bf
    from goliath_b200 import _lib
    from goliath_b200.geom import depth_discontuity_mask
    from goliath_b200.mesh_vae import AutoEncoder, CameraPixelBias

    dev = torch.device("cuda:0")
    res = {"card": card(), "torch": torch.__version__, "render": [H, W], "ds_rate": DS}
    m = bf.seeded_fill(AutoEncoder(**bf.config(H, W, DS), assets=bf.assets())).to(dev).eval()
    L = _lib.lib()

    inp1 = frame_inputs(m, 1, dev)
    with torch.no_grad():
        res["forward_B1_ms"] = timed({"ours": lambda: m(**inp1)}, args.reps)["ours"]
        L.gb_launch_count_reset()
        m(**inp1)
        torch.cuda.synchronize()
        res["forward_B1_launches"] = int(L.gb_launch_count())
        st = [staged(m, inp1) for _ in range(args.reps)]
    res["forward_B1_stages_ms"] = {k: float(np.median([s[k] for s in st])) for k in st[0]}

    inp4 = frame_inputs(m, 4, dev)
    params = [p for p in m.parameters() if p.requires_grad]

    def step():
        p = m(**inp4)
        torch.autograd.grad(p["rgb"].sum() + p["alpha"].sum(), params, allow_unused=True)

    res["fwd_bwd_B4_ms"] = timed({"ours": step}, args.reps)["ours"]
    L.gb_launch_count_reset()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step()
    torch.cuda.synchronize()
    res["fwd_bwd_B4_launches"] = int(L.gb_launch_count())
    res["fwd_bwd_B4_peak_MiB"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20

    # the two new kernels against their torch formulation, B = 4 at 2048 x 1334
    g = torch.Generator(device=dev).manual_seed(1)
    depth = 1000 + 3000 * (torch.rand(4, 1, H, W, device=dev, generator=g) > 0.999).float()
    res["depth_mask_ms"] = timed({"ours": lambda: depth_discontuity_mask(depth),
                                  "torch": lambda: bf.depth_disc_mask(depth)[0]}, 50)
    pb = CameraPixelBias(H, W, bf.CAMERAS, DS).to(dev)
    torch.nn.init.normal_(pb.bias)
    bias = pb.bias
    rgb = torch.randn(4, 3, H, W, device=dev, requires_grad=True)
    idx = torch.tensor([0, 1, 0, 2], device=dev)

    def ours_pb():
        out = pb(idx, rgb)
        torch.autograd.grad(out.sum(), [bias, rgb])

    def torch_pb():
        out = rgb + F.interpolate(bias[idx], size=(H, W), mode="bilinear")
        torch.autograd.grad(out.sum(), [bias, rgb])

    res["pixel_bias_fwd_bwd_ms"] = timed({"ours": ours_pb, "torch": torch_pb}, 50)
    res["not_measured"] = ["an end-to-end reference baseline (the reference renders through drtk, not available)",
                           "kernel-only times of the stages", "CUDA-graph replay of the frame"]
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
