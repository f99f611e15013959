"""Build the REFERENCE's own CUDA extensions for sm_90a into oracle/_ref/ (git-ignored).

TEST INFRASTRUCTURE ONLY.  Compiles the sources WHERE THEY LIE under /root/reference/extensions (nothing is copied
into the repo) with the reference's own flags (setup.py of each extension: -use_fast_math where it says so,
-std=c++17, -lineinfo) except the gencode, which is sm_90a.  The outputs are the reference's pybind modules
`sgutilslib`, `utilslib`, `mvpraymarchlib`; tests load them from oracle/_ref as the GPU witness that pins the
oracle and the product kernels (tests/test_ref_witness_gpu.py) and bench.py times them as the reference arm of
the extension-level ratios.  gsplat is third-party and absent: it cannot be built here.

It also byte-compiles the reference's L1 PYTHON wrappers (extensions/*/X.py and ca_code/utils/render_gsplat.py: the
`autograd.Function`s that call into the pybind modules) to sourceless .pyc files under oracle/_ref/pyc/ — compiled
artefacts like the .so files, no source text enters the repo — so that tests/test_dropins.py can run the reference's
OWN wrappers, unchanged, over `goliath_b200.install_dropins()` on the GPU box (where /root/reference does not exist).

Usage: python oracle/build_ref.py [sgutilslib utilslib mvpraymarchlib]
"""
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

REF = "/root/reference/extensions"
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")

EXTS = {
    "sgutilslib": dict(dir="sgutils", sources=["sg.cu"], fast_math=True),
    "utilslib": dict(dir="utils", sources=["utils.cpp", "utils_kernel.cu"], fast_math=False),
    "mvpraymarchlib": dict(dir="mvpraymarch", sources=["mvpraymarch.cpp", "mvpraymarch_kernel.cu", "bvh.cu"],
                           fast_math=True),
}


def torch_flags():
    import torch
    from torch.utils import cpp_extension as ce

    inc = ce.include_paths("cuda") if "device_type" in ce.include_paths.__code__.co_varnames else ce.include_paths(True)
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    return inc, libdir, abi


def build_one(name):
    spec = EXTS[name]
    inc, libdir, abi = torch_flags()
    os.makedirs(os.path.join(OUT, "obj"), exist_ok=True)
    pyinc = sysconfig.get_paths()["include"]
    common = ["-I" + os.path.join(REF, "include"), "-I" + os.path.join(REF, spec["dir"]), "-I" + pyinc] + \
             ["-I" + p for p in inc] + ["-DTORCH_EXTENSION_NAME=" + name, "-DTORCH_API_INCLUDE_EXTENSION_H",
                                        "-D_GLIBCXX_USE_CXX11_ABI=%d" % abi]
    objs = []
    for src in spec["sources"]:
        path = os.path.join(REF, spec["dir"], src)
        obj = os.path.join(OUT, "obj", name + "_" + src.replace(".", "_") + ".o")
        objs.append(obj)
        if src.endswith(".cu"):
            cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-lineinfo", "-O3",
                   "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-D__CUDA_NO_HALF_OPERATORS__",
                   "-D__CUDA_NO_HALF_CONVERSIONS__", "-D__CUDA_NO_HALF2_OPERATORS__"] + \
                  (["-use_fast_math"] if spec["fast_math"] else []) + common + ["-c", path, "-o", obj]
        else:
            cmd = ["g++", "-std=c++17", "-O3", "-fPIC", "-DNDEBUG"]  # setuptools CFLAGS carry -DNDEBUG; utils.cpp:67 only compiles with it
            cmd = cmd + common + ["-c", path, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("%s\n%s" % (" ".join(cmd), r.stderr[-4000:]))
    so = os.path.join(OUT, name + ".so")
    link = ["g++", "-shared", "-o", so] + objs + ["-L" + libdir, "-L/usr/local/cuda/lib64", "-lc10", "-lc10_cuda",
                                                  "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python",
                                                  "-lcudart", "-Wl,-rpath," + libdir]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("%s\n%s" % (" ".join(link), r.stderr[-4000:]))
    return so


WRAPPERS = {  # module name under oracle/_ref/pyc -> reference file
    "ref_sgutils": "/root/reference/extensions/sgutils/sgutils.py",
    "ref_utils": "/root/reference/extensions/utils/utils.py",
    "ref_mvpraymarch": "/root/reference/extensions/mvpraymarch/mvpraymarch.py",
    "ref_render_gsplat": "/root/reference/ca_code/utils/render_gsplat.py",
}


def build_wrappers():
    """py_compile the reference's L1 wrappers (unchanged) into oracle/_ref/pyc/<name>.pyc."""
    import py_compile

    out = os.path.join(OUT, "pyc")
    os.makedirs(out, exist_ok=True)
    done = []
    for name, src in WRAPPERS.items():
        if os.path.exists(src):
            done.append(py_compile.compile(src, cfile=os.path.join(out, name + ".pyc"), doraise=True))
    return done


def build(names=None):
    if not os.path.isdir(REF):
        return []  # GPU box: use the prebuilt files
    names = names or list(EXTS)
    with ThreadPoolExecutor(max_workers=3) as ex:
        return list(ex.map(build_one, names)) + build_wrappers()


if __name__ == "__main__":
    if sys.argv[1:] == ["wrappers"]:
        print(build_wrappers())
    else:
        print(build(sys.argv[1:] or None))
