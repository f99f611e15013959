"""Environment-spin lighting (goliath_b200.envmap.prefilter_envmap_sg, goliath_b200.light_decorator.EnvSpinDecorator;
csrc/envmap_prefilter.cu):

1. the prefilter with injected draws against the reference's prefilterEnvmapSG (tests/golden/envspin_ref.npz, made by
   tests/golden/make_envspin_golden.py), every element;
2. a torch restatement of prefilterEnvmapSG, pinned to the same golden, against the Philox path at the decorator's
   sizes (4096 samples): per-texel z-scores from the restatement's sample variance;
3. seeds: bit-identical for one seed, different for another, reproduced by torch.manual_seed;
4. the decorator's dict against the reference's (random prefilter patched out on both sides), envbg against the
   pinned rotate_envmap_mat in the reference's operation order;
5. the per-frame step captured in a CUDA graph, replay equal to eager;
6. the decorator's outputs driving PrimDecoder's environment-map branch and render_views_envmap, against the same
   call given the golden's tensors;
7. the argument checks (host side, no GPU needed)."""
import importlib.util
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import assert_close, t2n

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_envspin_golden", os.path.join(HERE, "golden", "make_envspin_golden.py"))
golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(golden)
envgold = golden.envgold

BAR = dict(rtol=1e-4, atol=1e-5, equal_nan=True)
gpu = pytest.mark.gpu
_Z = {}


def _z():
    if not _Z:
        _Z["z"] = np.load(os.path.join(HERE, "golden", "envspin_ref.npz"))
    return _Z["z"]


def torch_prefilter(sigma, v, env_tex, num_samples, xi=None, chunk=32, generator=None):
    """prefilterEnvmapSG (ca_code/utils/envmap.py:251-323) restated in torch, `chunk` samples per pass.  xi: the
    draws [S,B,2,H,W], or None for torch.rand.  Returns the mean [B,3,H,W] and the per-texel sample variance."""
    B, _, H, W = v.shape
    acc = torch.zeros(B, 3, H, W, dtype=torch.float64, device=v.device)
    acc2 = torch.zeros_like(acc)
    s2 = math.sqrt(2.0) * sigma
    n = v[None]
    up = torch.where(n[:, :, 2:3] < 0.999, torch.tensor([0.0, 0.0, 1.0], device=v.device)[:, None, None],
                     torch.tensor([1.0, 0.0, 0.0], device=v.device)[:, None, None])
    t = F.normalize(torch.cross(up.expand_as(n), n, dim=2), dim=2)
    b = torch.cross(n, t, dim=2)
    for s0 in range(0, num_samples, chunk):
        c = min(chunk, num_samples - s0)
        x = xi[s0:s0 + c] if xi is not None else torch.rand(c, B, 2, H, W, device=v.device, generator=generator)
        phi = 2.0 * np.pi * x[:, :, 0:1]
        theta = s2 * torch.special.erfinv(x[:, :, 1:2] * math.erf(np.pi / s2))
        st = torch.sin(theta)
        d = F.normalize(t * (torch.cos(phi) * st) + b * (torch.sin(phi) * st) + n * torch.cos(theta), dim=2)
        uv = torch.stack([(1 / np.pi) * torch.atan2(d[:, :, 0], d[:, :, 2]),
                          2 * ((1 / np.pi) * torch.acos(d[:, :, 1])) - 1.0], -1)
        tex = env_tex[None].expand(c, -1, -1, -1, -1).reshape(c * B, *env_tex.shape[1:])
        col = F.grid_sample(tex, uv.reshape(c * B, H, W, 2), padding_mode="border", align_corners=False)
        col = col.reshape(c, B, 3, H, W).double()
        acc += col.sum(0)
        acc2 += (col * col).sum(0)
    mean = acc / num_samples
    var = (acc2 - num_samples * mean * mean) / (num_samples - 1)
    return mean.float(), var


def _pf_case(name, cuda):
    v, env, xi, sigma = golden.prefilter_case(name)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return d(v), d(env), d(xi), sigma


# --------------------------------------------------------------------------------------- 1. injected draws, every element
@gpu
@pytest.mark.parametrize("case", list(golden.PF_CASES))
def test_prefilter_injected_xi_matches_reference(cuda, case):
    from goliath_b200.envmap import prefilter_envmap_sg

    v, env, xi, sigma = _pf_case(case, cuda)
    want = _z()["pf_" + case]
    got = prefilter_envmap_sg(sigma, v, env, golden.S, xi=xi)
    np.testing.assert_allclose(t2n(got), want, **BAR, err_msg=case)
    if v.shape[0] == 1:  # the [S,2,H,W] form of the draws with B = 1
        assert torch.equal(prefilter_envmap_sg(sigma, v, env, golden.S, xi=xi[:, 0]), got)


# ------------------------------------------------------------------------------- 2. restatement, then the Philox stream
@gpu
@pytest.mark.parametrize("case", list(golden.PF_CASES))
def test_torch_prefilter_matches_reference(cuda, case):
    v, env, xi, sigma = _pf_case(case, cuda)
    got, _ = torch_prefilter(sigma, v, env, golden.S, xi=xi)
    np.testing.assert_allclose(t2n(got), _z()["pf_" + case], **BAR, err_msg=case)


def _decorator_levels(cuda, miplevel=4, sigma_step=0.2):
    """the decorator's prefilter inputs for a smooth 512x1024 probe: (sigma, v, area-halved sin-weighted probe)"""
    from goliath_b200.light_decorator import _sph_grid

    img = torch.from_numpy(envgold._smooth(np.random.default_rng(77), (1, 3, 512, 1024), 0.05, 2.5)).to(cuda)
    img = img * torch.sin((torch.arange(512, device=cuda) + 0.5) * np.pi / 512)[None, None, :, None]
    out = []
    for i in range(miplevel - 1):
        img = F.interpolate(img, None, scale_factor=0.5, mode="area")
        out.append(((i + 1) * sigma_step, _sph_grid(img.shape[2], img.shape[3], cuda), img))
    return out


@gpu
def test_philox_prefilter_matches_torch_statistically(cuda):
    """at 256x512, 128x256, 64x128 with sigma 0.2, 0.4, 0.6 and 4096 samples: z = (ours - torch) / sqrt(2 var / S)
    per texel and channel, var the restatement's sample variance; the draws are independent, so z ~ N(0, 1)"""
    from goliath_b200.envmap import _prefilter_levels

    S = 4096
    levels = _decorator_levels(cuda)
    ours = _prefilter_levels([lv + (None,) for lv in levels], S, seed=20261016)
    gen = torch.Generator(device=cuda).manual_seed(11)
    zs = []
    for (sigma, v, env), got in zip(levels, ours):
        mean, var = torch_prefilter(sigma, v, env, S, generator=gen)
        assert got.shape == mean.shape and torch.isfinite(got).all()
        assert float(var.min()) > 0.0
        zs.append(((got.double() - mean.double()) / torch.sqrt(2.0 * var / S)).flatten())
    z = torch.cat(zs)
    zmax, zmean, zrms = float(z.abs().max()), float(z.mean()), float(z.pow(2).mean().sqrt())
    assert zmax < 6.0 and abs(zmean) < 0.05 and 0.9 <= zrms <= 1.1, (zmax, zmean, zrms)


# ----------------------------------------------------------------------------------------------------------- 3. seeds
@gpu
def test_prefilter_seeds(cuda):
    from goliath_b200.envmap import prefilter_envmap_sg

    sigma, v, env = _decorator_levels(cuda, miplevel=3)[1]
    a = prefilter_envmap_sg(sigma, v, env, 256, seed=5)
    assert torch.equal(a, prefilter_envmap_sg(sigma, v, env, 256, seed=5))
    assert not torch.equal(a, prefilter_envmap_sg(sigma, v, env, 256, seed=6))
    torch.manual_seed(3)
    b = prefilter_envmap_sg(sigma, v, env, 256)
    torch.manual_seed(3)
    assert torch.equal(b, prefilter_envmap_sg(sigma, v, env, 256))


# ------------------------------------------------------------------------------------------------- 4. the decorator dict
def _decorator(mod, monkeypatch=None):
    from goliath_b200 import light_decorator

    if monkeypatch is not None:  # the reference run had prefilterEnvmapSG return its input texture
        monkeypatch.setattr(light_decorator, "_prefilter_levels", lambda levels, n, seed=None: [l[2].clone() for l in levels])
    return light_decorator.EnvSpinDecorator(mod, golden.probe(), **golden.DECORATOR)


OUT_KEYS = {"preconv_envmap", "sigma_step", "envmap", "lightrot", "light_intensity", "light_pos", "envbg", "light_type",
            "n_lights", "is_fullylit_frame"}


@gpu
def test_decorator_matches_reference(cuda, monkeypatch):
    from goliath_b200.envmap import rotate_envmap_mat

    z = _z()
    got = {}
    dec = _decorator(lambda **d: got.update(d) or "out", monkeypatch)
    assert {k for k, _ in dec.named_buffers() if k in dec.state_dict()} == {"sphvec"} | {"mipmap_%d" % i for i in range(4)}
    assert dec.perc90 == float(z["perc90"])
    probe = golden.probe()[:, :, ::-1][::-1, ::-1]  # BGR -> RGB, ydown
    assert torch.equal(dec.image.cpu(), torch.from_numpy(np.ascontiguousarray(probe.transpose(2, 0, 1))))
    mip_tol = dict(rtol=1e-5, atol=0.5 / golden.MIP_QSCALE + 1e-6)
    for i in range(1, 4):
        np.testing.assert_allclose(t2n(getattr(dec, "mipmap_%d" % i)), envgold.decode(z, "mipmap_%d" % i, golden.MIP_QSCALE),
                                   **mip_tol, err_msg="mipmap_%d" % i)
    for f, idx in enumerate(golden.FRAMES):
        B = len(idx)
        got.clear()
        campos = torch.zeros(B, 3, device=cuda)
        assert dec(campos=campos, index=list(idx)) == "out"
        assert set(got) == OUT_KEYS | {"campos", "index"}, set(got)
        assert got["light_type"] == "envmap" and got["sigma_step"] == dec.sigma_step
        assert got["is_fullylit_frame"].shape == (1,) and float(got["is_fullylit_frame"]) == 0.0
        for k in ("envmap", "lightrot", "light_intensity", "light_pos", "n_lights"):
            want = z["f%d_%s" % (f, k)]
            assert got[k].dtype == torch.float32 and got[k].is_cuda and tuple(got[k].shape) == want.shape, k
            assert got[k].is_contiguous(), k
            np.testing.assert_allclose(t2n(got[k]), want, rtol=1e-5, atol=1e-6, err_msg="frame %d %s" % (f, k))
        if idx[0] == 0:
            assert torch.equal(got["lightrot"][0], torch.eye(3, device=cuda))
        scale = float(z["f%d_scale" % f])
        assert len(got["preconv_envmap"]) == 4
        for i, lv in enumerate(got["preconv_envmap"]):
            base = getattr(dec, "mipmap_%d" % i)
            assert lv.shape == (B,) + tuple(base.shape[1:]) and lv.dtype == torch.float32
            np.testing.assert_allclose(t2n(lv), np.repeat(t2n(base), B, 0) * np.float32(scale), rtol=1e-5, atol=1e-7)
        # envbg: the pinned rotate_envmap_mat, / perc90 * 255 / 255 as the reference orders it (true divisions)
        e = got["envbg"]
        assert e.shape == (B, 3, 512, 1024) and e.dtype == torch.float32
        rot = rotate_envmap_mat(dec.image[None].expand(B, -1, -1, -1).contiguous(), got["lightrot"])
        f32 = lambda x: torch.tensor(x, dtype=torch.float32, device=cuda)
        want = rot / f32(dec.perc90) * 255 / f32(255.0)
        assert_close(t2n(e), t2n(want), rtol=1e-6, atol=0.0, what="frame %d envbg" % f)
        if f == 0:
            np.testing.assert_allclose(t2n(e), envgold.decode(z, "f0_envbg"), rtol=1e-5, atol=0.5 / envgold.QSCALE + 1e-6)


# ------------------------------------------------------------------------------------------------------ 5. graph capture
@gpu
def test_decorator_frame_graph_capture(cuda):
    dec = _decorator(lambda **d: d)
    data = dict(campos=torch.zeros(3, 3, device=cuda), index=[0, 129, 255])
    eager = dec(**dict(data))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        dec(**dict(data))
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = dec(**dict(data))
    g.replay()
    torch.cuda.synchronize()
    for k, v in eager.items():
        if torch.is_tensor(v):
            assert torch.equal(out[k], v), k
        elif isinstance(v, list) and k == "preconv_envmap":
            assert all(torch.equal(a, b) for a, b in zip(out[k], v)), k
        else:
            assert out[k] == v, k


# ------------------------------------------------------------------------------------------------------- 6. end to end
@gpu
def test_decorator_drives_decoder_and_render(cuda, monkeypatch):
    from goliath_b200 import synthetic
    from goliath_b200.rgca import PrimDecoder
    from goliath_b200.render import render_views_envmap

    S, H, W = 128, 240, 216

    class Geo:
        def __init__(self, nml): self.nml = nml
        def to_uv(self, x): return x
        def vn(self, g): return self.nml

    gen = torch.Generator().manual_seed(21)
    pos = (torch.randn(1, 3, S, S, generator=gen) * 60).to(cuda)
    nml = F.normalize(torch.randn(1, 3, S, S, generator=gen), dim=1).to(cuda)
    model = PrimDecoder(16, Geo(nml), 255 * torch.rand(3, S, S, generator=gen), slabsize=S).to(cuda).eval()
    embs = torch.randn(1, 16, generator=gen).to(cuda)
    lsh = torch.randn(1, 3, 81, generator=gen).to(cuda)
    cam = synthetic.ring_camera(2, img_h=H, img_w=W)
    K = torch.tensor([[[cam["fx"], 0, cam["cx"]], [0, cam["fy"], cam["cy"]], [0, 0, 1]]], dtype=torch.float32, device=cuda)
    Rt = cam["viewmat"][None].to(cuda)
    intr = [(cam["fx"], cam["fy"], cam["cx"], cam["cy"])]

    def frame(**d):
        preds = model(embs, pos, d["campos"], d["light_intensity"], d["light_pos"], lsh, d["n_lights"],
                      preconv_envmap=d["preconv_envmap"], lightrot=d["lightrot"])
        return render_views_envmap(W, H, K, Rt, Rt, preds, d["envbg"], intrinsics_host=intr, capacity=1 << 18)

    z = _z()
    dec = _decorator(frame, monkeypatch)
    campos = torch.tensor([[0.0, 0.0, 1000.0]], device=cuda)
    with torch.no_grad():
        rgb, alpha, depth = dec(campos=campos, index=[golden.FRAMES[0][0]])
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
        scale = np.float32(z["f0_scale"])
        levels = [dec.mipmap_0 * scale] + [d(envgold.decode(z, "mipmap_%d" % i, golden.MIP_QSCALE)) * scale
                                           for i in range(1, 4)]
        rgb_g, alpha_g, depth_g = frame(campos=campos, light_intensity=d(z["f0_light_intensity"]),
                                        light_pos=d(z["f0_light_pos"]), n_lights=d(z["f0_n_lights"]),
                                        preconv_envmap=levels, lightrot=d(z["f0_lightrot"]),
                                        envbg=d(envgold.decode(z, "f0_envbg")))
    torch.cuda.synchronize()
    assert rgb.shape == (1, 3, H, 3 * W) and torch.isfinite(rgb).all()
    assert float(alpha.max()) > 0.5 and float(alpha.min()) < 0.1, "the head must cover part of the image"
    assert float(rgb[..., 2 * W:].abs().max()) > 0.0, "the specular render must see the environment"
    assert torch.equal(alpha, alpha_g) and torch.equal(depth, depth_g)
    assert_close(t2n(rgb), t2n(rgb_g), rtol=1e-4, atol=1e-5, what="rgb")


# ----------------------------------------------------------------------------------------------------------- 7. checks
def test_prefilter_rejects_bad_arguments():
    from goliath_b200.envmap import prefilter_envmap_sg

    v, env = torch.zeros(1, 3, 4, 8), torch.zeros(1, 3, 8, 16)
    for args, kw, msg in (((0.2, v, env, 4), {}, "CUDA tensor"),
                          ((0.2, v[:, :2], env, 4), {}, "v must be"),
                          ((0.2, v, env[:, :2], 4), {}, "env_tex must be"),
                          ((0.2, v, torch.zeros(2, 3, 8, 16), 4), {}, "env_tex must be"),
                          ((0.0, v, env, 4), {}, "sigma"),
                          ((0.2, v, env, 0), {}, "num_samples"),
                          ((0.2, v, env, 4), dict(xi=torch.zeros(3, 2, 4, 8)), "xi must be"),
                          ((0.2, v, env, 4), dict(xi=torch.zeros(4, 2, 4, 4)), "xi must be")):
        with pytest.raises(RuntimeError, match=msg):
            prefilter_envmap_sg(*args, **kw)


def test_decorator_rejects_bad_arguments():
    from goliath_b200.light_decorator import EnvSpinDecorator

    probe = np.ones((64, 128, 3), np.float32)
    for kw, msg in ((dict(miplevel=0), "miplevel"), (dict(miplevel=9), "miplevel"), (dict(miplevel=2.0), "miplevel"),
                    (dict(sigma_step=0.0), "sigma_step"), (dict(cycle=0), "cycle")):
        with pytest.raises(ValueError, match=msg):
            EnvSpinDecorator(None, probe, **kw)
    with pytest.raises(ValueError, match="H x W x 3"):
        EnvSpinDecorator(None, np.ones((64, 128, 4), np.float32))
    with pytest.raises(ValueError, match="90th percentile"):
        EnvSpinDecorator(None, np.zeros((64, 128, 3), np.float32))
