"""Generate tests/golden/envspin_ref.npz from the REFERENCE's own `prefilterEnvmapSG` (ca_code/utils/envmap.py:305-323)
and `EnvSpinDecorator` (ca_code/utils/light_decorator.py:18-164), run on the CPU in fp32.  Nothing is copied: the code is
imported from a reference checkout.  The inputs are not stored: `prefilter_case` and `probe` rebuild them from numpy
PCG64 seeds, and tests/test_envspin_gpu.py reads the fixture through this file.

1. prefilterEnvmapSG with th.rand_like patched to hand out seeded draws xi [S,B,2,H,W] (S = 64), for 6x10 fields of
   unit directions v (a third of them with n_z above the 0.999 switch of importance_sample_sg's `up`, some just below
   it) on 3x16x32 and 3x8x16 textures (B = 1 and B = 2), sigma 0.2 and 0.6.  Stored raw: pf_<case> [B,3,6,10].
2. EnvSpinDecorator(ydown=True, env_scale=8.0, run_vis_relight.py's settings) on a smooth synthetic 512x1024 HDR probe
   with a bright region, handed in through a patched cv2.imread; Tensor.cuda is the identity and prefilterEnvmapSG
   returns its input texture (the random prefilter is pinned by part 1), so mipmap_<i> (i >= 1) is the area-halved
   sin-weighted probe.  Frames: B = 1 at index 37, B = 3 at indices 0, 129, 255.  Stored per frame f: envmap, lightrot,
   light_intensity, light_pos, n_lights, the mip scale 2 pi norm_scale[0]; once: perc90, mipmap_1..3 and frame 0's
   envbg (through make_envmap_golden.encode).

Usage: python tests/golden/make_envspin_golden.py /path/to/goliath-checkout
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "envspin_ref.npz")
_spec = importlib.util.spec_from_file_location("make_envmap_golden", os.path.join(HERE, "make_envmap_golden.py"))
envgold = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(envgold)

S = 64
PF_CASES = {"t16x32_s02": (16, 32, 1, 0.2), "t16x32_s06": (16, 32, 1, 0.6), "t8x16_s02": (8, 16, 2, 0.2),
            "t8x16_s06": (8, 16, 2, 0.6)}
FRAMES = ((37,), (0, 129, 255))
DECORATOR = dict(ydown=True, env_scale=8.0)
MIP_QSCALE = float(2 ** 12)  # mip levels up to ~40: a step of 2^-12 is < 1.3e-5 relative at the bright end


def prefilter_case(name):
    """v [B,3,6,10], env_tex [B,3,He,We], xi [S,B,2,6,10] and sigma of one prefilter case"""
    He, We, B, sigma = PF_CASES[name]
    rng = np.random.default_rng(2511 + list(PF_CASES).index(name))
    v = rng.standard_normal((B, 3, 6, 10))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    # columns 0-2: n_z above 0.999 (up = (1,0,0)); column 3: n_z just below (up = (0,0,1))
    for b in range(B):
        for y in range(6):
            for x, nz in ((0, 1.0), (1, 0.9995), (2, 0.99905), (3, 0.9989)):
                a = rng.uniform(0, 2 * np.pi)
                r = np.sqrt(1.0 - nz * nz)
                v[b, :, y, x] = (r * np.cos(a), r * np.sin(a), nz)
    env = envgold._smooth(rng, (B, 3, He, We), 0.2, 3.0)
    xi = rng.random((S, B, 2, 6, 10), dtype=np.float32)
    return v.astype(np.float32), env, xi, sigma


def probe():
    """the synthetic HDR probe as cv2.imread(path, -1) returns it: 512 x 1024 x 3 float32 (BGR), smooth, 0.05 .. 2
    with a bright region of up to ~40"""
    rng = np.random.default_rng(4096)
    img = envgold._smooth(rng, (1, 3, 512, 1024), 0.05, 2.0)[0].transpose(1, 2, 0)
    y, x = np.mgrid[0:512, 0:1024].astype(np.float64)
    sun = 38.0 * np.exp(-((y - 140.0) ** 2 + (x - 700.0) ** 2) / (2 * 18.0 ** 2))
    return np.ascontiguousarray(img + (sun[..., None] * np.array([0.8, 0.9, 1.0]))).astype(np.float32)


def main():
    if len(sys.argv) != 2 or not os.path.isdir(os.path.join(sys.argv[1], "ca_code")):
        sys.exit(__doc__)
    sys.path.insert(0, sys.argv[1])
    import torch as th
    from ca_code.utils import envmap, light_decorator

    d = {}
    rand_like = th.rand_like
    try:
        for name in PF_CASES:
            v, env, xi, sigma = prefilter_case(name)
            draws = iter(th.from_numpy(xi))
            th.rand_like = lambda t: next(draws).clone()
            d["pf_" + name] = envmap.prefilterEnvmapSG(sigma, th.from_numpy(v), th.from_numpy(env), S).numpy()
            print("prefilter %s: NaN %d" % (name, int(np.isnan(d["pf_" + name]).sum())))
    finally:
        th.rand_like = rand_like

    img = probe()
    cuda, imread, prefilter = th.Tensor.cuda, light_decorator.cv2.imread, envmap.prefilterEnvmapSG
    th.Tensor.cuda = lambda self, *a, **k: self
    light_decorator.cv2.imread = lambda path, flag: img.copy()
    envmap.prefilterEnvmapSG = lambda sigma, v, env_tex, num_samples=1: env_tex.clone()
    try:
        got = {}
        dec = light_decorator.EnvSpinDecorator(lambda **data: got.update(data) or data, "probe.hdr", **DECORATOR)
        scales = []
        mip = dec.mipmap
        dec.mipmap = lambda bsize, device, scale=1.0: scales.append(float(scale)) or mip(bsize, device, scale)
        for f, idx in enumerate(FRAMES):
            got.clear()
            dec(campos=th.zeros(len(idx), 3), index=list(idx))
            for k in ("envmap", "lightrot", "light_intensity", "light_pos", "n_lights"):
                d["f%d_%s" % (f, k)] = got[k].numpy()
            d["f%d_scale" % f] = np.float32(scales[-1])
            assert got["light_type"] == "envmap" and got["sigma_step"] == dec.sigma_step
            if f == 0:
                envgold.encode(d, "f0_envbg", got["envbg"].numpy())
        d["perc90"] = np.float64(np.percentile(dec.image.numpy(), 90))
        for i in range(1, dec.miplevel):
            envgold.encode(d, "mipmap_%d" % i, getattr(dec, "mipmap_%d" % i).numpy(), MIP_QSCALE)
    finally:
        th.Tensor.cuda, light_decorator.cv2.imread, envmap.prefilterEnvmapSG = cuda, imread, prefilter
    np.savez(OUT, **d)
    print("wrote %s (%d bytes), perc90 %.6f" % (OUT, os.path.getsize(OUT), d["perc90"]))


if __name__ == "__main__":
    main()
