"""Per-kernel device time of one bench head step (bench.py --config head) for both record modes of the bucket-path render.

Builds the bench scene (bench.packed_scene, HeadWorkload, capacity 8 G), captures one step in a CUDA graph as
bench.run_ours does, and replays it under torch.profiler (CUDA activities) with the L2 flushed before each replay.
Each record mode (GOLIATH_B200_RECORDS=packed / ranked) runs in a subprocess of its own, because the mode is read when
goliath_b200.gsplat.fused is imported.  The step time beside the table comes from CUDA events around the same replays
in a separate run without the profiler.

  python scripts/profile_head_step.py [--replays 20] [--modes packed,ranked] [--out profile.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLUSH_TAG = "bitwise_not"  # the L2 flush is a bitwise NOT over 256 MiB: no kernel of the step has that name


def card():
    import torch

    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")[:2]]
    except Exception as e:  # reported, not guessed
        info["power_limit"] = info["max_sm_clock"] = "unknown (%s)" % type(e).__name__
    return info


def short_name(name):
    """Kernel name without the return type, anonymous namespace and parameter list."""
    n = name.replace("(anonymous namespace)::", "")
    n = re.sub(r"^void ", "", n)
    depth = 0
    for i, ch in enumerate(n):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0 and i > 0:
            return n[:i]
    return n


def per_kernel(prof):
    """{kernel: [total device us, launches]} over the profiled window, the L2 flush left out."""
    import torch

    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA or FLUSH_TAG in e.name:
            continue
        d = per.setdefault(short_name(e.name), [0.0, 0])
        d[0] += e.time_range.elapsed_us()
        d[1] += 1
    return per


def child(mode, replays):
    os.environ["GOLIATH_B200_RECORDS"] = mode
    sys.path.insert(0, ROOT)
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    args = argparse.Namespace(gaussians=300_000, lights=32, eager_sync=False)
    wl = bench.HeadWorkload(args, 0, 1, dev)
    static_in = bench.packed_scene(wl.G).to(dev)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def flush():
        flush_buf.bitwise_not_()  # > 50 MB L2

    wl.compute(static_in)
    wl.compute(static_in)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            wl.compute(static_in)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        wl.compute(static_in)
    for _ in range(5):
        flush()
        g.replay()
    torch.cuda.synchronize()

    # step time without the profiler: events around each replay, L2 flushed before it
    ts = []
    for _ in range(max(replays, 50)):
        flush()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(replays):
            flush()
            g.replay()
        torch.cuda.synchronize()
    source = "graph replay"
    per = per_kernel(prof)
    if not per:  # a profiler that does not see kernels inside graphs: fall back to eager steps, and say so
        source = "eager steps (the profiler recorded no kernels inside the graph)"
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(replays):
                flush()
                wl.compute(static_in)
            torch.cuda.synchronize()
        per = per_kernel(prof)
    from goliath_b200.gsplat import fused

    kernels = {k: {"us_per_step": v[0] / replays, "launches_per_step": v[1] / replays} for k, v in per.items()}
    print(json.dumps({"mode": mode, "ranked_flag": bool(fused.RANKED), "replays": replays, "source": source,
                      "step_ms_median": ts[len(ts) // 2], "step_ms_min": ts[0], "step_ms_max": ts[-1],
                      "kernels": kernels}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--modes", default="packed,ranked")
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.replays)
        return
    res = {}
    for mode in a.modes.split(","):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mode, "--replays", str(a.replays)],
                           capture_output=True, text=True, cwd=ROOT)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise SystemExit("profile of mode %s failed (exit %d)" % (mode, r.returncode))
        res[mode] = json.loads(r.stdout.strip().splitlines()[-1])
    sys.path.insert(0, ROOT)
    c = card()
    modes = list(res)
    names = sorted({k for m in modes for k in res[m]["kernels"]},
                   key=lambda k: -max(res[m]["kernels"].get(k, {"us_per_step": 0})["us_per_step"] for m in modes))
    print("%s, power limit %s, max SM clock %s; %d graph replays per mode, L2 flushed before each"
          % (c["name"], c["power_limit"], c["max_sm_clock"], a.replays))
    print("kernel times from: " + "; ".join("%s: %s" % (m, res[m]["source"]) for m in modes))
    print("| kernel | " + " | ".join("%s us/step" % m for m in modes) + " |")
    print("|---|" + "---|" * len(modes))
    for k in names:
        cells = []
        for m in modes:
            v = res[m]["kernels"].get(k)
            cells.append("-" if v is None else "%.1f" % v["us_per_step"] +
                         ("" if abs(v["launches_per_step"] - 1) < 1e-6 else " (x%g)" % v["launches_per_step"]))
        print("| %s | %s |" % (k[:90], " | ".join(cells)))
    print("| sum of kernel time | " + " | ".join("%.1f" % sum(v["us_per_step"] for v in res[m]["kernels"].values())
                                                for m in modes) + " |")
    print("| step, events, median (min-max) ms | " + " | ".join(
        "%.3f (%.3f-%.3f)" % (res[m]["step_ms_median"], res[m]["step_ms_min"], res[m]["step_ms_max"]) for m in modes)
        + " |")
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": c, "modes": res}, f, indent=1)


if __name__ == "__main__":
    main()
