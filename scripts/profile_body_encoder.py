"""Time the body encoders on the GPU: `mesh_vae.encode` (LBSModule.unpose -> to_uv -> Encoder + FaceEncoder) forward at
B = 1 and forward + backward at B = 4 against the torch formulation on the same GPU (the restated modules of
tests/body_encoder_restate.py in fp32, TF32 off and torch's defaults, on the same to_uv, with the reference-style
unpose: a [B,V,4,4] matrix and inverse() in a loop over the batch), the two alternated in one call; unpose alone; per
ConvDownBlock, CUDA-event times with the block's bytes and FLOPs computed from shapes; launch counts of this library;
peak memory; the card name and power limit.  Needs a GPU: without one it fails.

Usage: python scripts/profile_body_encoder.py [--reps 20] [--json out.json]"""
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
FP32_TFLOPS = 67.0    # H100 SXM fp32 SIMT peak
V_BODY = 7306         # vertices of the body mesh the unpose timing uses


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "unknown (%s)" % e
    return q


def timed_pair(fns, reps):
    """median ms of each callable, the callables alternated inside one timing loop"""
    for f in fns.values():
        for _ in range(3):
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


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def launches(fn):
    from goliath_b200 import _lib

    L = _lib.lib()
    torch.cuda.synchronize()
    L.gb_launch_count_reset()
    fn()
    torch.cuda.synchronize()
    return int(L.gb_launch_count())


def looped_unpose(lbs, verts, motion):
    """LBSModule.unpose the way the reference computes it: blended [B,V,4,4], then inverse() item by item"""
    f = lbs.lbs_fn
    B = motion.shape[0]
    mats = f.skeleton(motion, lbs.lbs_scale.reshape(1, -1).expand(B, -1))
    m = (mats[:, f.skin_indices] * f.skin_weights[None, :, :, None, None]).sum(2)
    m4 = torch.cat([m, torch.zeros_like(m[:, :, :1])], 2)
    m4[:, :, 3, 3] = 1.0
    v4 = torch.cat([verts / lbs.global_scaling, torch.ones_like(verts[:, :, :1])], 2)[..., None]
    out = torch.cat([(m4[i].contiguous().inverse() @ v4[i])[None] for i in range(B)])
    return out[..., :3, 0].contiguous() - lbs.lbs_template_verts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_body_encoder needs a CUDA device (there is no CPU path to time)")
    import body_encoder_restate as br
    import lbs_recipe as R
    from goliath_b200 import mesh_vae
    from goliath_b200.geom import GeometryModule
    from goliath_b200.lbs import LBSModule
    from goliath_b200.nn import ConvDownBlock

    dev = torch.device("cuda:0")
    mask = br.synthetic_mask()
    enc, face = mesh_vae.Encoder(n_embs=1024, mask=mask).to(dev), mesh_vae.FaceEncoder(mask=mask, n_embs=256).to(dev)
    t_enc, t_face = br.Encoder(n_embs=1024, mask=mask).to(dev), br.FaceEncoder(mask=mask, n_embs=256).to(dev)
    t_enc.load_state_dict(enc.state_dict())
    t_face.load_state_dict(face.state_dict())
    # a V_BODY-vertex skinned model on the tree24 skeleton, with a random UV layout of the right size
    model, cfg, template, scales = R.skinned_model("tree24", 100, n_verts=V_BODY)
    lbs = LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0]).to(dev)
    rng = np.random.default_rng(0)
    index = torch.as_tensor(rng.integers(0, V_BODY, (1024, 1024, 3)), dtype=torch.int32)
    index[rng.random((1024, 1024)) < 0.2] = -1
    bary = torch.as_tensor(rng.dirichlet(np.ones(3), (1024, 1024)), dtype=torch.float32)
    geo = GeometryModule(torch.zeros(1, 3, dtype=torch.int32), index, bary).to(dev)

    def torch_encode(reg, mo):
        with torch.no_grad():
            uv = geo.to_uv(looped_unpose(lbs, reg, mo))
        return {**t_enc(uv), **t_face(uv)}

    res = {"card": card(), "torch": torch.__version__, "reps": args.reps, "V": V_BODY}
    params = list(enc.parameters()) + list(face.parameters())
    t_params = list(t_enc.parameters()) + list(t_face.parameters())
    for B in (1, 4):
        mo = R.motion(B, 5).to(dev)
        reg = lbs.pose(0.1 * torch.randn(B, V_BODY, 3, device=dev), mo)
        for m in (enc, face, t_enc, t_face):
            m.train(B == 4)

        def ours_fwd():
            with torch.no_grad():
                return mesh_vae.encode(lbs, geo, enc, face, reg, mo)

        def torch_fwd():
            with torch.no_grad():
                return torch_encode(reg, mo)

        def ours_fb():
            out = mesh_vae.encode(lbs, geo, enc, face, reg, mo)
            torch.autograd.grad(sum(v.sum() for v in out.values()), params)

        def torch_fb():
            out = torch_encode(reg, mo)
            torch.autograd.grad(sum(v.sum() for v in out.values()), t_params)

        ours, tch, tag = (ours_fwd, torch_fwd, "fwd_B1") if B == 1 else (ours_fb, torch_fb, "fwd_bwd_B4")
        for name, tf32 in (("torch_fp32_notf32", False), ("torch_default", None)):
            old = torch.backends.cudnn.allow_tf32
            if tf32 is not None:
                torch.backends.cudnn.allow_tf32 = tf32
            try:
                t = timed_pair({"ours": ours, name: tch}, args.reps)
            finally:
                torch.backends.cudnn.allow_tf32 = old
            res["%s_ms_%s" % (tag, name)] = t[name]
            res["%s_ms_ours_beside_%s" % (tag, name)] = t["ours"]
        res[tag + "_peak_MiB_ours"], res[tag + "_peak_MiB_torch"] = peak(ours), peak(tch)
        res[tag + "_launches_ours"] = launches(ours)
        t = timed_pair({"ours": lambda: lbs.unpose(reg, mo), "torch_looped_inverse": lambda: looped_unpose(lbs, reg, mo)},
                       args.reps)
        res["unpose_B%d_ms" % B] = t
        res["unpose_B%d_launches_ours" % B] = launches(lambda: lbs.unpose(reg, mo))

    # per block: the fused kernels against the torch block (fp32, TF32 off)
    blocks = []
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    for cin, cout, size in br.ENCODER_BLOCKS:
        for B in (1, 4):
            ours = ConvDownBlock(cin, cout, size).to(dev)
            tb = br.ConvDownBlock(cin, cout, size).to(dev)
            tb.load_state_dict(ours.state_dict())
            x = torch.randn(B, cin, size, size, device=dev, requires_grad=True)
            H, Ho = size, size // 2
            fl_fwd = 2.0 * B * (H * H * 9 * cin * cin + Ho * Ho * (9 * cin * cout + cin * cout))
            # x (conv1, plus a quarter for the skip), both untied biases, h1 written and read back, out
            by_fwd = 4.0 * (1.25 * B * cin * H * H + cin * H * H + cout * Ho * Ho + 2 * B * cin * H * H
                            + B * cout * Ho * Ho)
            row = {"cin": cin, "cout": cout, "size": size, "B": B, "fwd_bytes": by_fwd, "fwd_flops": fl_fwd}

            def runners(m):
                def f():
                    with torch.no_grad():
                        m(x)

                def fb():
                    torch.autograd.grad(m(x).sum(), [x] + list(m.parameters()))

                return f, fb

            (fo, fbo), (ft, fbt) = runners(ours), runners(tb)
            t = timed_pair({"ours": fo, "torch": ft}, args.reps)
            tb_ = timed_pair({"ours": fbo, "torch": fbt}, args.reps)
            row.update(fwd_ms_ours=t["ours"], fwd_ms_torch=t["torch"], fwd_bwd_ms_ours=tb_["ours"],
                       fwd_bwd_ms_torch=tb_["torch"], fwd_launches_ours=launches(fo), fwd_bwd_launches_ours=launches(fbo),
                       fwd_bwd_peak_MiB_ours=peak(fbo), fwd_bwd_peak_MiB_torch=peak(fbt))
            sec = row["fwd_ms_ours"] * 1e-3
            row["fwd_GBs_ours"] = by_fwd / sec / 1e9
            row["fwd_share_of_bw_roof"] = row["fwd_GBs_ours"] / HBM_GBS
            row["fwd_share_of_fp32_roof"] = fl_fwd / sec / 1e12 / FP32_TFLOPS
            blocks.append(row)
    torch.backends.cudnn.allow_tf32 = old
    res["blocks"] = blocks
    print(json.dumps(res, indent=1))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
