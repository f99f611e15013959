"""Time the RGCA encoder's texture stack (`texmod`, rgca.py:281-298: eight Conv2dWNUB(.., 4, 2, 1) + LeakyReLU(0.2),
1024^2 -> 4^2) per layer and in total, forward and forward + backward, at B = 1 and B = 4, for three variants:

  ours      goliath_b200.nn.Conv2dWNUB (fused sm_90a kernels: conv + weight-norm scale + untied bias + LeakyReLU);
  lib_tf32  the reference's composition F.conv2d + bias[None] + leaky_relu with torch's default (cuDNN TF32 allowed);
  lib_fp32  the same composition with TF32 disallowed (the precision class of ours).

CUDA events after warm-up, median of the reps, L2 flushed (256 MiB write) before each rep.  The library variants run
in child processes under `timeout` (the first cuDNN call can spend minutes compiling engines); the fp32 child also
compares our outputs with the library's at every timed size.  Prints one JSON document with the algorithmic FLOP and
bytes per layer, the share of the FP32 peak, and the GPU's name and power limit read in the same run.

Usage: python scripts/profile_encoder.py [--reps 20] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

LAYERS = [(3, 32, 512), (32, 32, 256), (32, 64, 128), (64, 64, 64), (64, 128, 32), (128, 128, 16), (128, 256, 8),
          (256, 256, 4)]  # (Cin, Cout, output size)
BATCHES = (1, 4)
FP32_PEAK = 67e12   # H100 SXM data sheet, dense FP32
HBM_BW = 3.35e12    # H100 SXM data sheet, HBM3


def layer_work(B, cin, cout, s):
    """algorithmic FLOP and bytes of one layer: forward (read x, weights, bias; write out) and backward (read gout,
    out, x, weights; write gx unless first layer, gw, g_bias)"""
    mac = B * cout * s * s * cin * 16
    x, out, bias, w = 4 * B * cin * 4 * s * s, 4 * B * cout * s * s, 4 * cout * s * s, 4 * cout * cin * 16
    fwd_bytes = x + w + bias + out
    bwd_bytes = 2 * out + x + w + bias + w + (x if cin != 3 else 0)
    bwd_flop = 2 * mac * (1 if cin == 3 else 2)  # weight gradient (+ data gradient)
    return {"fwd_flop": 2 * mac, "fwd_bytes": fwd_bytes, "fwd_bwd_flop": 2 * mac + bwd_flop, "fwd_bwd_bytes": fwd_bytes + bwd_bytes}


def make_params(dev):
    gen = torch.Generator().manual_seed(2024)
    ps = []
    for cin, cout, s in LAYERS:
        v = torch.randn(cout, cin, 4, 4, generator=gen) / np.sqrt(cin * 16)
        g = v.norm() * (0.8 + 0.4 * torch.rand(cout, 1, 1, 1, generator=gen))
        b = 0.05 * torch.randn(cout, s, s, generator=gen)
        ps.append((v.to(dev), g.to(dev), b.to(dev)))
    return ps


def make_input(B, dev):
    gen = torch.Generator().manual_seed(100 + B)
    return (255.0 * torch.rand(B, 3, 1024, 1024, generator=gen) / 255.0 - 0.5).to(dev)


class Timer:
    def __init__(self, dev, reps):
        self.flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        self.reps = reps

    def __call__(self, fn, warm=3):
        for _ in range(warm):
            fn()
        ts = []
        for _ in range(self.reps):
            self.flush_buf.fill_(1)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))


def ours_layers(params, dev):
    from goliath_b200 import nn as gnn

    mods = []
    for (cin, cout, s), (v, g, b) in zip(LAYERS, params):
        m = gnn.Conv2dWNUB(cin, cout, s, s, 4, 2, 1).to(dev)
        m.fused_slope = 0.2
        with torch.no_grad():
            m.weight_v.copy_(v)
            m.weight_g.copy_(g)
            m.bias.copy_(b)
        mods.append(m)
    return [lambda h, m=m: m(h) for m in mods], [p for m in mods for p in m.parameters()]


def lib_layers(params):
    ts = [(v.clone().requires_grad_(), g.clone().requires_grad_(), b.clone().requires_grad_()) for v, g, b in params]

    def layer(h, v, g, b):  # layers.py:200-204,303-327 + the LeakyReLU that follows (rgca.py:282-297)
        return F.leaky_relu(F.conv2d(h, g * v / v.norm(), None, 2, 1) + b[None], 0.2)

    return [lambda h, t=t: layer(h, *t) for t in ts], [p for t in ts for p in t]


def run_variant(name, reps):
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    if name == "lib_fp32":
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
    elif name == "lib_tf32":
        torch.backends.cudnn.allow_tf32 = True
    params = make_params(dev)
    fns, leaves = ours_layers(params, dev) if name == "ours" else lib_layers(params)
    timer = Timer(dev, reps)
    res = {"variant": name, "tf32_allowed": bool(torch.backends.cudnn.allow_tf32) if name != "ours" else False}
    cmp = {}
    ours_fns = ours_layers(params, dev)[0] if name == "lib_fp32" else None
    for B in BATCHES:
        x0 = make_input(B, dev)
        # per-layer inputs: the stack's own activations
        acts = [x0]
        with torch.no_grad():
            for f in fns:
                acts.append(f(acts[-1]))
            if ours_fns is not None:  # our outputs against the fp32 library's, layer by layer, from the same inputs
                for i, f in enumerate(ours_fns):
                    r, o = acts[i + 1].double(), f(acts[i]).double()
                    cmp["B%d_layer%d" % (B, i + 1)] = float((o - r).norm() / r.norm())
                h = x0
                for f in ours_fns:
                    h = f(h)
                cmp["B%d_stack" % B] = float((h.double() - acts[-1].double()).norm() / acts[-1].double().norm())
        per = []
        for i, f in enumerate(fns):
            xin = acts[i]
            xg = xin.clone().requires_grad_(i > 0)
            go = torch.ones_like(acts[i + 1])
            with torch.no_grad():
                t_f = timer(lambda: f(xin))

            def fb():
                f(xg).backward(go)
                for p in leaves:
                    p.grad = None
                xg.grad = None

            t_fb = timer(fb)
            per.append({"fwd_ms": t_f, "fwd_bwd_ms": t_fb})

        def stack(h):
            for f in fns:
                h = f(h)
            return h

        with torch.no_grad():
            t_sf = timer(lambda: stack(x0))
        go = torch.ones_like(acts[-1])

        def stack_fb():
            stack(x0).backward(go)
            for p in leaves:
                p.grad = None

        t_sfb = timer(stack_fb)
        res["B%d" % B] = {"layers": per, "stack_fwd_ms": t_sf, "stack_fwd_bwd_ms": t_sfb}
        del acts, x0
        torch.cuda.empty_cache()
    if cmp:
        res["ours_vs_lib_fp32_rel_err"] = cmp
    return res


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clk = [c.strip() for c in q.split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clk}
    except Exception as e:  # the query is informative only; the timings stand without it
        return {"name": torch.cuda.get_device_name(0), "power_limit": "unavailable (%s)" % e}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--variant", choices=["ours", "lib_tf32", "lib_fp32"])
    ap.add_argument("--timeout", type=int, default=1200, help="seconds allowed to each library child process")
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("profile_encoder.py needs a CUDA device")
    if args.variant:  # child process: one variant, JSON on stdout
        print(json.dumps(run_variant(args.variant, args.reps)))
        return
    doc = {"gpu": gpu_info(), "method": "CUDA events, median of %d reps after 3 warm-up calls, L2 flushed (256 MiB "
           "write) before each rep; library variants in child processes" % args.reps,
           "peaks": {"fp32_flops": FP32_PEAK, "hbm_bytes_per_s": HBM_BW, "source": "H100 SXM data sheet"},
           "work": {"B%d" % B: [dict(layer="%d->%d @%d^2" % (c, o, s), **layer_work(B, c, o, s)) for c, o, s in LAYERS]
                    for B in BATCHES}}
    doc["ours"] = run_variant("ours", args.reps)
    for name in ("lib_tf32", "lib_fp32"):
        cmd = ["timeout", str(args.timeout), sys.executable, os.path.abspath(__file__), "--variant", name, "--reps",
               str(args.reps)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
        doc[name] = json.loads(lines[-1]) if r.returncode == 0 and lines else {
            "error": "exit %d" % r.returncode, "stderr_tail": r.stderr[-2000:]}
    # shares of the FP32 peak and of the roofline (larger of FLOP / peak and bytes / bandwidth) for ours
    for B in BATCHES:
        key = "B%d" % B
        for w, t in zip(doc["work"][key], doc["ours"][key]["layers"]):
            for ph in ("fwd", "fwd_bwd"):
                sec = t[ph + "_ms"] * 1e-3
                t[ph + "_fp32_peak_share"] = w[ph + "_flop"] / FP32_PEAK / sec
                lo_c, lo_m = w[ph + "_flop"] / FP32_PEAK, w[ph + "_bytes"] / HBM_BW
                t[ph + "_roofline_share"] = max(lo_c, lo_m) / sec
                t[ph + "_bound"] = "fp32" if lo_c >= lo_m else "hbm"
        tot = sum(w["fwd_flop"] for w in doc["work"][key])
        doc["ours"][key]["stack_fwd_fp32_peak_share"] = tot / FP32_PEAK / (doc["ours"][key]["stack_fwd_ms"] * 1e-3)
    text = json.dumps(doc)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
