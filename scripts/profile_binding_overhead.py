"""Host cost of one library launch from Python: the `_lib.kernels()` launcher against the explicit pattern it replaced,
`with torch.cuda.device(dev): _lib.check(lib().gb_x(.., _lib.ptr(t), .., _lib.stream_ptr(dev)), "x")`.

Both call the same entry points with sizes that make them return 0 before launching anything (gb_conv2d_wnub_fwd with
B = 0, 5 pointers; gb_head_lights_fwd with B = 0, 10 pointers), so the time is the Python and ctypes work of a call.
The library's launch counter is checked to stay unchanged.  Each pattern makes 10^5 calls per entry point, in
alternating blocks on cuda:0; the card name and power limit are read in the same run.  Needs a GPU: without one it
fails.

Usage: python scripts/profile_binding_overhead.py [--calls 100000] [--blocks 10] [--out DIR]
(writes DIR/binding_overhead.json when --out is given)"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from goliath_b200 import _lib  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def cases(dev):
    L, K = _lib.lib(), _lib.kernels()
    t = [torch.empty(16, device=dev) for _ in range(10)]
    x, v, scale, bias, out = t[:5]
    ptr, check, stream_ptr = _lib.ptr, _lib.check, _lib.stream_ptr

    def conv_old():
        with torch.cuda.device(dev):
            check(L.gb_conv2d_wnub_fwd(0, 8, 8, 4, 4, 3, ptr(x), 128, ptr(v), ptr(scale), ptr(bias), 0, 1.0, 0,
                                       ptr(out), stream_ptr(dev)), "conv2d_wnub_fwd")

    def conv_new():
        K.gb_conv2d_wnub_fwd(0, 8, 8, 4, 4, 3, x, 128, v, scale, bias, 0, 1.0, 0, out)

    def lights_old():
        with torch.cuda.device(dev):
            check(L.gb_head_lights_fwd(0, 4, 3, ptr(t[0]), ptr(t[1]), ptr(t[2]), ptr(t[3]), ptr(t[4]), ptr(t[5]),
                                       ptr(t[6]), ptr(t[7]), ptr(t[8]), ptr(t[9]), ptr(t[5]), stream_ptr(dev)),
                  "head_lights_fwd")

    def lights_new():
        K.gb_head_lights_fwd(0, 4, 3, t[0], t[1], t[2], t[3], t[4], t[5], t[6], t[7], t[8], t[9], t[5])

    return {"gb_conv2d_wnub_fwd (5 pointers)": (conv_old, conv_new),
            "gb_head_lights_fwd (10 pointers)": (lights_old, lights_new)}


def run(fn, n):
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100_000, help="calls per pattern and entry point")
    ap.add_argument("--blocks", type=int, default=10, help="alternating blocks the calls are split into")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_binding_overhead.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    L = _lib.lib()
    per_block = args.calls // args.blocks
    res = {"card": card(), "calls": per_block * args.blocks, "blocks": args.blocks, "entry_points": {}}
    for name, (old, new) in cases(dev).items():
        run(old, 1000)
        run(new, 1000)
        launches = L.gb_launch_count()
        blocks = {"old": [], "new": []}
        for _ in range(args.blocks):
            blocks["old"].append(run(old, per_block) / per_block * 1e6)
            blocks["new"].append(run(new, per_block) / per_block * 1e6)
        assert L.gb_launch_count() == launches, "a zero-size call launched a kernel"
        entry = {}
        for k, us in blocks.items():
            us = sorted(us)
            entry[k] = {"median_us": us[len(us) // 2], "min_us": us[0], "max_us": us[-1]}
        entry["new_minus_old_median_us"] = entry["new"]["median_us"] - entry["old"]["median_us"]
        res["entry_points"][name] = entry
        print("%-34s old %.2f us  new %.2f us per call (medians of %d blocks; old %.2f-%.2f, new %.2f-%.2f)" % (
            name, entry["old"]["median_us"], entry["new"]["median_us"], args.blocks, entry["old"]["min_us"],
            entry["old"]["max_us"], entry["new"]["min_us"], entry["new"]["max_us"]))
    print("card:", res["card"])
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "binding_overhead.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
