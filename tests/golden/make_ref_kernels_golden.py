"""Golden vectors of the reference's own CUDA kernels (its extensions sgutils, utils and mvpraymarch, rebuilt for sm_90a
into oracle/_ref by oracle/build_ref.py) on the inputs of tests/test_sg_gpu.py::test_sg_vs_reference_kernels and the
reference-kernel tests of tests/test_raymarch_gpu.py.  Needs a GPU and oracle/_ref; the .npz is committed.

Arrays of at most WHOLE elements are stored whole.  Larger ones are stored at a fixed, seeded sample of their elements
plus their last TAIL elements (the partial last block of a launch), see sample_index below, together with the largest
magnitude of the full array, so that the tests apply the same tolerances as against the live kernels.
    python tests/golden/make_ref_kernels_golden.py [out.npz]"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(HERE, "ref_kernels_ref.npz")


def sample_index(size, n, seed):
    """Sorted flat indices of the stored elements of an array of `size` elements: all of them when size <= WHOLE, else
    a fixed sample of n of the first size - TAIL elements and the last TAIL elements."""
    if size <= WHOLE:
        return np.arange(size)
    head = np.random.default_rng(seed).choice(size - TAIL, n, replace=False)
    return np.concatenate([np.sort(head), np.arange(size - TAIL, size)])


def sg_case(dev, w_type):
    """Inputs of the reference-kernel SG test (N, D, L = 2, 20000, 32)."""
    from test_oracle_sg import make

    N, D, L = 2, 20000, 32
    dirs, sig, lv, lp, pp, nl = make(N=N, D=D, L=L, seed=123)
    if w_type >= 2:
        sig = sig * 0 + 0.3
    c = lambda t: t.to(dev).contiguous()
    g = c(torch.randn(N, D, 3, generator=torch.Generator().manual_seed(3)))
    return [c(dirs), c(sig), c(lv), c(lp), c(pp), c(nl)], g, (N, D, L)


def raydirs_case(dev):
    from goliath_b200 import synthetic

    s = synthetic.mvp_scene(N=3, img_h=37, img_w=45)
    t = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in s.items()}
    px, py = torch.meshgrid(torch.arange(45.0), torch.arange(37.0), indexing="xy")
    pix = (torch.stack([px, py], -1)[None].repeat(3, 1, 1, 1) + 0.5).contiguous().to(dev)
    return t, pix


def aabb_case(dev):
    from goliath_b200 import synthetic

    s = synthetic.mvp_scene(N=2, side=8)
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in s.items()}


def march_case(dev, algo):
    from goliath_b200 import synthetic
    from goliath_b200.mvpraymarch import build_accel
    from goliath_b200.utils import compute_raydirs

    s = synthetic.mvp_scene(with_warp=(algo == 1), N=2, side=12, T=(4, 8, 8), img_h=96, img_w=72, density=150.0)
    t = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in s.items()}
    raypos, raydir, tminmax = compute_raydirs(t["viewpos"], t["viewrot"], t["focal"], t["princpt"], (t["img_w"], t["img_h"]),
                                              t["volradius"])
    sid, ch, aabb = build_accel((t["primpos"], t["primrot"], t["primscale"]), algo, fixedorder=True)
    g = torch.randn(*raypos.shape[:3], 4, generator=torch.Generator().manual_seed(11)).to(dev)
    return t, (raypos, raydir, tminmax), (sid, ch, aabb), g


def march_fwd(lib, t, rays, accel, algo, dev):
    raypos, raydir, tminmax = rays
    sid, ch, aabb = accel
    N, H, W = raypos.shape[:3]
    rgba = torch.empty(N, H, W, 4, device=dev)
    sat = torch.full((N, H, W, 3), -1.0, device=dev)
    lib.raymarch_forward(raypos, raydir, 0.01, tminmax, sid, ch, aabb, t["primpos"], t["primrot"], t["primscale"],
                         t["template"], t["warp"] if algo == 1 else None, rgba, sat, None, None, algo, False, 512, True, True,
                         8.0, 8.0, 0, 0.99, 3, 8, 16)
    return rgba, sat


def march_bwd(lib, t, rays, accel, algo, rgba, sat, g):
    raypos, raydir, tminmax = rays
    sid, ch, aabb = accel
    warp = t["warp"] if algo == 1 else None
    gp, gr, gs = torch.zeros_like(t["primpos"]), torch.zeros_like(t["primrot"]), torch.zeros_like(t["primscale"])
    gt = torch.zeros_like(t["template"])
    gw = torch.zeros_like(warp) if warp is not None else None
    lib.raymarch_backward(raypos, raydir, 0.01, tminmax, sid, ch, aabb, t["primpos"], gp, t["primrot"], gr, t["primscale"],
                          gs, t["template"], gt, warp, gw, rgba, g, sat, None, algo, False, 512, True, True, 8.0, 8.0, 0, 0.99,
                          3, 8, 16)
    return dict(grad_primpos=gp, grad_primrot=gr, grad_primscale=gs, grad_template=gt,
                **({"grad_warp": gw} if gw is not None else {}))


# arrays up to WHOLE elements are stored whole; larger ones as SAMPLE sampled elements + the last TAIL elements
WHOLE, SAMPLE, TAIL = 16384, 2048, 64


def _ref(name):
    so = os.path.join(ROOT, "oracle", "_ref", name + ".so")
    spec = importlib.util.spec_from_file_location(name, so)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def main(out_path):
    dev = torch.device("cuda:0")
    sg, ut, mv = _ref("sgutilslib"), _ref("utilslib"), _ref("mvpraymarchlib")
    res = {}

    def put(key, arr, seed):
        arr = arr.detach().cpu().numpy()
        flat = arr.reshape(-1)
        res[key] = flat[sample_index(flat.size, SAMPLE, seed)]
        res[key + "_absmax"] = np.float64(np.abs(flat).max() if flat.size else 0.0)

    for w in range(4):
        a, g, (N, D, L) = sg_case(dev, w)
        o = torch.empty(N, D, 3, device=dev)
        sg.evaluate_gaussian_fwd(*a, o, w)
        gd, gs, gl = torch.zeros(N, D, 3, device=dev), torch.zeros(N, D, device=dev), torch.zeros(N, L, 3, device=dev)
        sg.evaluate_gaussian_bwd(*a, g, gd, gs, gl, w)
        torch.cuda.synchronize()
        for k, v in (("integral", o), ("grad_dirs", gd), ("grad_sigmas", gs), ("grad_light_values", gl)):
            put("sg%d_%s" % (w, k), v, 100 + w)

    t, pix = raydirs_case(dev)
    rr = [torch.empty(*pix.shape[:3], c, device=dev) for c in (3, 3, 2)]
    ut.compute_raydirs_forward(t["viewpos"], t["viewrot"], t["focal"], t["princpt"], pix, 45, 37, 1.0, *rr)
    torch.cuda.synchronize()
    for k, v in zip(("raypos", "raydir", "tminmax"), rr):
        put("raydirs_" + k, v, 200)

    from goliath_b200.mvpraymarch import _fixedorder_topology, build_accel

    t = aabb_case(dev)
    _, _, aabb = build_accel((t["primpos"], t["primrot"], t["primscale"]), 0, fixedorder=True)
    sid, ch, par = _fixedorder_topology(2, 64, dev)
    ra = torch.empty_like(aabb)
    mv.compute_aabb(t["primpos"], t["primrot"], t["primscale"], sid, ch, par, ra, 0)
    torch.cuda.synchronize()
    res["aabb"] = ra.cpu().numpy()

    for algo in (0, 1):
        t, rays, accel, g = march_case(dev, algo)
        rgba, sat = march_fwd(mv, t, rays, accel, algo, dev)
        grads = march_bwd(mv, t, rays, accel, algo, rgba, sat, g)
        torch.cuda.synchronize()
        put("march%d_rgba" % algo, rgba, 300 + algo)
        put("march%d_sat" % algo, sat, 300 + algo)
        for k, v in grads.items():
            put("march%d_%s" % (algo, k), v, 310 + algo)
    np.savez_compressed(out_path, **res)
    print(out_path, sum(v.nbytes for v in res.values()), "bytes")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else OUT)
