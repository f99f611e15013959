"""Time the body decoder (DESIGN.md row R9) on the GPU: forward at B = 1 and forward + backward at B = 4 of
goliath_b200.mesh_vae.ConvDecoder (with this library's SeamSampler and GeometryModule.from_uv on synthetic seam data)
against the torch formulation on the same GPU (oracle.mesh_vae_oracle.ConvDecoder in fp32, TF32 off and torch's
defaults, with the seam sampler and sample_uv restated in torch); per trunk block, CUDA-event kernel times with the
block's bytes and FLOPs computed from shapes; peak memory; the card name and power limit.

Usage: python scripts/profile_body_decoder.py [--reps 10] [--json out.json]"""
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

CFG = dict(uv_size=1024, init_uv_size=64, n_pose_dims=98, n_pose_enc_channels=16, n_embs=1024, n_embs_enc_channels=32,
           n_face_embs=256, n_init_channels=64, n_min_channels=4)
HBM_GBS = 3350.0      # H100 SXM HBM3 peak
FP32_TFLOPS = 67.0    # H100 SXM fp32 SIMT peak


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
    import seams_restate as sr
    from goliath_b200.geom import GeometryModule
    from goliath_b200.mesh_vae import ConvDecoder
    from goliath_b200.nn import UpConvBlockDeep
    from goliath_b200.seams import SeamSampler
    from oracle import mesh_vae_oracle as mo

    dev = torch.device("cuda:0")
    seams = sr.synthetic_seams(1024)
    rng = np.random.default_rng(2)
    vt = torch.as_tensor(rng.random((9000, 2)), dtype=torch.float32)
    v2uv = torch.as_tensor(rng.integers(0, 9000, (7306, 4)), dtype=torch.int32)
    geo = GeometryModule(torch.zeros(1, 3, dtype=torch.int32), torch.zeros(1, 1, 3), torch.zeros(1, 1, 3), vt=vt,
                         v2uv=v2uv).to(dev)
    dec = ConvDecoder(geo, seam_sampler=SeamSampler(seams).to(dev), assets=mo.synthetic_masks(), **CFG).to(dev)
    ts = sr.TorchSeamSampler(*(seams[k].to(dev) for k in ("dst_ij", "src_ij", "uvs", "weights")))
    ref = mo.ConvDecoder(mo.synthetic_masks(), None, lambda t: sr.sample_uv(t, vt.to(dev), v2uv.to(dev))).to(dev)
    ref.load_state_dict({k: v for k, v in dec.state_dict().items() if not k.startswith("seam_sampler")
                         and not k.startswith("geo_fn")})

    def oracle_call(*inp):
        calls = iter((ts.impaint, ts.resample, ts.resample))
        ref.resample = lambda x: next(calls)(x)
        return ref(*inp)

    res = {"card": card(), "torch": torch.__version__, "reps": args.reps}
    for B in (1, 4):
        inp = [t.to(dev) for t in mo.seeded_inputs(batch=B)]
        for name, f in (("ours", dec), ("torch_fp32_notf32", oracle_call), ("torch_default", oracle_call)):
            tf32 = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = name == "torch_default"
            try:
                def fwd():
                    with torch.no_grad():
                        return f(*inp)

                def fwd_bwd():
                    out = f(*inp)
                    sum(v.float().sum() for v in out.values()).backward()

                if B == 1:
                    res["fwd_B1_ms_" + name] = timed(fwd, args.reps)
                    res["fwd_B1_peak_MiB_" + name] = peak(fwd)
                else:
                    res["fwd_bwd_B4_ms_" + name] = timed(fwd_bwd, args.reps)
                    res["fwd_bwd_B4_peak_MiB_" + name] = peak(fwd_bwd)
            finally:
                torch.backends.cudnn.allow_tf32 = tf32
            dec.zero_grad(set_to_none=True)
            ref.zero_grad(set_to_none=True)

    # per trunk block: fused kernels vs the torch block (fp32, TF32 off)
    blocks = []
    torch.backends.cudnn.allow_tf32 = False
    for cin, cout, size in ((128, 64, 128), (64, 32, 256), (32, 16, 512), (16, 8, 1024)):
        for B in (1, 4):
            ours = UpConvBlockDeep(cin, cout, size, groups=2).to(dev)
            tb = mo.UpConvBlockDeep(cin, cout, size, groups=2).to(dev)
            tb.load_state_dict(ours.state_dict())
            x = torch.randn(B, cin, size // 2, size // 2, device=dev, requires_grad=True)
            H = size
            cg = cin // 2
            fl_fwd = 2.0 * B * H * H * (9 * cin * cg + 9 * cout * cg + cout * cg)
            # x, both untied biases, h1 written and read back, out (the inference forward writes no mask)
            by_fwd = 4.0 * (B * cin * H * H / 4 + (cin + cout) * H * H + 2 * B * cin * H * H + B * cout * H * H)
            row = {"cin": cin, "cout": cout, "size": size, "B": B, "fwd_bytes": by_fwd, "fwd_flops": fl_fwd}
            for name, m in (("ours", ours), ("torch", tb)):
                def f():
                    with torch.no_grad():
                        m(x)

                def fb():
                    m(x).sum().backward()

                row["fwd_ms_" + name] = timed(f, args.reps)
                row["fwd_bwd_ms_" + name] = timed(fb, args.reps)
                row["fwd_bwd_peak_MiB_" + name] = peak(fb)
            t = row["fwd_ms_ours"] * 1e-3
            row["fwd_GBs_ours"] = by_fwd / t / 1e9
            row["fwd_share_of_bw_roof"] = row["fwd_GBs_ours"] / HBM_GBS
            row["fwd_share_of_fp32_roof"] = fl_fwd / t / 1e12 / FP32_TFLOPS
            blocks.append(row)
    res["blocks"] = blocks
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
