"""In-tree build of libgoliath_b200.so: every CUDA translation unit compiled for sm_90a with nvcc.

`python -m goliath_b200.build` (or `__graft_entry__.build()`).  nvcc cross-compiles without a GPU; the
resulting .so is git-ignored.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libgoliath_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]
# per-file extra flags.  splat_project.cu carries the bit-exact binning contract, mesh_raster.cu the bit-exact index
# image: no FMA contraction.
# sg_shade.cu mirrors the reference extension's own flag (extensions/sgutils/setup.py:31) for last-bit parity.
EXTRA = {"splat_project.cu": ["-fmad=false"], "mesh_raster.cu": ["-fmad=false"], "sg_shade.cu": ["-use_fast_math"],
         "mvp_raymarch.cu": ["-use_fast_math"]}  # extensions/mvpraymarch/setup.py:31


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.abspath(__file__))
    jobs = []
    objs = []
    for src in sources():
        o = os.path.join(OBJ, src[:-3] + ".o")
        objs.append(o)
        if force or _stale(o, [os.path.join(CSRC, src)] + headers):
            cmd = ["nvcc"] + ARCH + COMMON + EXTRA.get(src, []) + ["-c", os.path.join(CSRC, src), "-o", o]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    if force or jobs or _stale(LIB, objs):
        run(["nvcc"] + ARCH + ["-shared", "--cudart", "shared", "-o", LIB] + objs)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
