"""Time the drivable body avatar `mesh_vae_drivable.AutoEncoder` on the GPU at B = 4 with a 2048 x 1334 render and the
real face model's 7306-vertex (21 918-value) face geometry (synthetic assets of tests/body_drive_restate.py, seeded
parameters): the eval forward (pose-driven shadow, no AO map) and the training forward + backward, each with a
per-stage breakdown (CUDA events, medians); the three kernels of csrc/body_drive.cu against their torch formulas; and
the face decoder's texture tower on the tensor cores against the SIMT layer kernels, alternated in one loop.  The card
name and power limit are read in the same run.  Needs a GPU: without one it fails.

Usage: python scripts/profile_body_drive.py [--reps 10] [--json out.json]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from profile_body_frame import card, timed  # noqa: E402

H, W, DS, B, N_FACE_VERTS = 2048, 1334, 8, 4, 7306


def frame_inputs(m, dev, seed=7):
    import body_frame_restate as bf

    g = torch.Generator().manual_seed(seed)
    P = m.lbs_fn.lbs_fn.param_transform.transform.shape[1] - m.lbs_fn.lbs_scale.shape[-1]
    V = m.lbs_fn.lbs_template_verts.shape[0]
    motion = (0.3 * torch.randn(B, P, generator=g)).to(dev)
    with torch.no_grad():
        posed = m.lbs_fn.pose(torch.zeros(B, V, 3, device=dev), motion)
    K, Rt, campos = bf.look_at(posed.cpu(), H, W)
    return {"lbs_motion": motion, "campos": campos.to(dev), "geom": posed + 0.5 * torch.randn_like(posed),
            "ao": bf.ambient_occlusion(B).to(dev), "K": K.to(dev), "Rt": Rt.to(dev),
            "_index": {"camera": (bf.BATCH_CAMERAS * B)[:B]}, "face_embs": torch.randn(B, 256, device=dev)}


def staged(m, inp, train):
    """the drivable forward with an event after each stage (and the backward in training); ms per stage"""
    names = ["encode", "decode", "pose", "view", "shadow", "texture", "cal", "render", "finish"] + (
        ["backward"] if train else [])
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
    ev[0].record()
    enc = m.encode(inp["geom"], inp["lbs_motion"], inp["face_embs"])
    ev[1].record()
    dec = m.decoder(motion=inp["lbs_motion"], embs=enc["embs"], face_embs=enc["face_embs"])
    ev[2].record()
    geom = m.lbs_fn.pose(dec["geom_delta_rec"], inp["lbs_motion"])
    ev[3].record()
    view = m.decoder_view(geom_rec=geom, tex_mean_rec=dec["tex_mean_rec"], camera_pos=inp["campos"])
    ev[4].record()
    if train:
        shadow = m.shadow_net(ao_map=inp["ao"])
        pose_shadow = m.pose_to_shadow(inp["lbs_motion"])["shadow_map"]
    else:
        shadow = m.pose_to_shadow(inp["lbs_motion"])
    ev[5].record()
    tex = m.forward_tex(dec["tex_mean_rec"], view["tex_view_rec"], shadow["shadow_map"])
    ev[6].record()
    idx = m.cal.name_to_idx(inp["_index"]["camera"])
    tex = m.cal(tex, idx)
    ev[7].record()
    rgb = m.renderer(geom, tex, K=inp["K"], Rt=inp["Rt"], edge_grad=False)["render"]
    ev[8].record()
    rgb = m.pixel_cal(idx, m.learn_blur(rgb, inp["_index"]["camera"]))
    ev[9].record()
    if train:
        params = [p for p in m.parameters() if p.requires_grad]
        torch.autograd.grad(rgb.sum() + pose_shadow.sum(), params, allow_unused=True)
        ev[10].record()
    torch.cuda.synchronize()
    return {n: ev[i].elapsed_time(ev[i + 1]) for i, n in enumerate(names)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_body_drive.py needs a CUDA device")
    import torch.nn.functional as F

    import body_drive_restate as bd
    from goliath_b200 import _lib
    from goliath_b200.face import face_tex_tail
    from goliath_b200.mesh_vae_drivable import AutoEncoder, face_tex_cond
    from goliath_b200.nn import tower_forward_tc
    from goliath_b200.shadow import pose_shadow

    dev = torch.device("cuda:0")
    res = {"card": card(), "torch": torch.__version__, "render": [H, W], "batch": B, "face_verts": N_FACE_VERTS}
    cfg = bd.config(H, W, DS, n_face_verts=N_FACE_VERTS)
    m = bd.seeded_fill(AutoEncoder(**cfg, assets=bd.assets())).to(dev).eval()
    L = _lib.lib()
    inp = frame_inputs(m, dev)
    eval_inp = {**inp, "ao": None}
    params = [p for p in m.parameters() if p.requires_grad]

    def train_step():
        p = m(**inp)
        torch.autograd.grad(p["rgb"].sum() + p["pose_shadow_map"].sum(), params, allow_unused=True)

    with torch.no_grad():
        res["eval_forward_ms"] = timed({"ours": lambda: m(**eval_inp)}, args.reps)["ours"]
        L.gb_launch_count_reset()
        m(**eval_inp)
        torch.cuda.synchronize()
        res["eval_forward_launches"] = int(L.gb_launch_count())
        st = [staged(m, inp, False) for _ in range(args.reps)]
    res["eval_forward_stages_ms"] = {k: float(np.median([s[k] for s in st])) for k in st[0]}
    m.train()
    m.encoder.noise_std = m.encoder_face.noise_std = 0.0
    res["train_fwd_bwd_ms"] = timed({"ours": train_step}, args.reps)["ours"]
    st = [staged(m, inp, True) for _ in range(args.reps)]
    res["train_fwd_bwd_stages_ms"] = {k: float(np.median([s[k] for s in st])) for k in st[0]}
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    L.gb_launch_count_reset()
    train_step()
    torch.cuda.synchronize()
    res["train_fwd_bwd_launches"] = int(L.gb_launch_count())
    res["train_fwd_bwd_peak_MiB"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    m.eval()

    # the three kernels against their torch formulas at the frame's sizes, B = 4 (TF32 off for torch's convolution)
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device=dev).manual_seed(1)
    last = m.decoder_face.texmod[-1]
    x = F.leaky_relu(torch.randn(B, 8, 512, 512, device=dev, generator=g), 0.2)
    fb = m.decoder_face.bias
    face_tex = 255 * torch.rand(B, 3, 1024, 1024, device=dev, generator=g)
    mask = m.encoder_face.tex_cond_mask
    lowres = torch.randn(B, 1, 128, 128, device=dev, generator=g, requires_grad=True)
    with torch.no_grad():
        res["face_tex_tail_ms"] = timed({
            "ours": lambda: face_tex_tail(x, last, fb),
            "torch": lambda: bd.face_tex_tail(x, last.weight_v, last.weight_g, last.bias, fb)}, 50)
        res["face_tex_cond_ms"] = timed({"ours": lambda: face_tex_cond(face_tex, mask),
                                         "torch": lambda: bd.face_tex_cond(face_tex, mask)}, 50)

    def ours_ps():
        torch.autograd.grad(pose_shadow(lowres, 1.0, 2048).sum(), [lowres])

    def torch_ps():
        torch.autograd.grad(bd.pose_shadow(lowres, 1.0, 2048).sum(), [lowres])

    res["pose_shadow_fwd_bwd_ms"] = timed({"ours": ours_ps, "torch": torch_ps}, 50)

    # the face decoder's texture tower (first seven layers): tensor cores against the SIMT layer kernels
    tower = m.decoder_face.texmod[:-1]
    z = torch.randn(B, 256, 4, 4, device=dev, generator=g)
    with torch.no_grad():
        res["face_tower_ms"] = timed({"tensor_cores": lambda: tower_forward_tc(tower, z), "simt": lambda: tower(z)},
                                     args.reps * 2)
    res["not_measured"] = ["an end-to-end reference baseline (the reference renders through pytorch3d, not available)",
                           "kernel-only times of the stages", "CUDA-graph replay of the frame"]
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
