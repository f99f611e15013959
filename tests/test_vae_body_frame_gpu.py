"""GPU checks of the body avatar's frame (csrc/body_frame.cu, goliath_b200/{geom,photo_loss,mesh_vae}.py): the
depth-discontinuity mask and the camera pixel bias against their torch formulas in fp64, CalV5 / LearnableBlur /
CameraPixelBias against the reference restated in fp64 (tests/body_frame_restate.py), `mesh_vae.AutoEncoder` against
tests/golden/body_frame_ref.npz (the reference's own AutoEncoder), and the frame's forward + backward without a host
synchronisation.

The module's name sorts it after tests/test_body_texture_gpu.py, whose test_unet_vs_oracle calibrates its bound on
torch's own fp32 error and is sensitive to what ran before it (see tests/test_vae_body_encoder_gpu.py)."""
import functools
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import body_frame_restate as bf

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "body_frame_ref.npz")
THRESHOLD = 40.0


def _maxrel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _nrel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _rendered_depth(cuda, B, H, W, seed=3):
    """the depth image of overlapping random triangles (30-400 px) through the project's RenderLayer: each triangle
    nearly fronto-parallel at a depth in 1000-5000, so the Sobel norm is far below the threshold inside a triangle and
    far above it across a silhouette"""
    from goliath_b200.mesh_render import RenderLayer

    g = torch.Generator().manual_seed(seed)
    n = 300
    ctr = torch.rand(n, 1, 2, generator=g) * torch.tensor([W, H])
    ang = torch.rand(n, 1, generator=g) * 6.283 + torch.arange(3) * 2.1
    rad = 30 + 370 * torch.rand(n, 3, generator=g)
    verts = []
    for b in range(B):
        xy = ctr + rad[..., None] * torch.stack([ang.cos(), ang.sin()], -1) + 3.7 * b
        z = 1000 + 100 * torch.randint(0, 41, (n, 1, 1), generator=g) + torch.rand(n, 3, 1, generator=g)
        verts.append(torch.cat([xy * z, z], -1).reshape(-1, 3))     # K = I, Rt = [I | 0]: v_pix = (x, y, z)
    vi = torch.arange(3 * n).reshape(n, 3)
    layer = RenderLayer(H, W, vi, torch.rand(3 * n, 2, generator=g), vi).to(cuda)
    eye = torch.eye(3, device=cuda).expand(B, 3, 3)
    Rt = torch.cat([eye, torch.zeros(B, 3, 1, device=cuda)], 2)
    out = layer(torch.stack(verts).to(cuda), torch.zeros(B, 1, 4, 4, device=cuda), eye, Rt)
    return out["depth_img"][:, None]


def _steps(cuda, B, H, W, seed=5):
    """plateaus and steps: random constant rectangles over a gentle ramp, step heights not on the threshold"""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    d = torch.empty(B, 1, H, W, dtype=torch.float64)
    for b in range(B):
        img = 2000 + 1.3 * xx + 0.7 * yy
        for _ in range(120):
            y0, x0 = int(torch.randint(0, H - 8, (1,), generator=g)), int(torch.randint(0, W - 8, (1,), generator=g))
            h, w = int(torch.randint(4, 300, (1,), generator=g)), int(torch.randint(4, 300, (1,), generator=g))
            img[y0:y0 + h, x0:x0 + w] = float(1000 + 3000 * torch.rand(1, generator=g, dtype=torch.float64))
        d[b, 0] = img
    return d.float().to(cuda)


@pytest.mark.parametrize("kind", ["rendered", "steps"])
def test_depth_disc_mask_vs_torch_fp64(cuda, kind):
    from goliath_b200.geom import depth_discontuity_mask

    B, H, W = 4, 2048, 1334
    depth = _rendered_depth(cuda, B, H, W) if kind == "rendered" else _steps(cuda, B, H, W)
    got = depth_discontuity_mask(depth)
    want, norm = bf.depth_disc_mask(depth.double(), THRESHOLD)
    assert got.dtype == torch.bool and got.shape == (B, 1, H, W)
    near = (norm - THRESHOLD).abs() <= 1e-4 * THRESHOLD     # where the summation order could decide
    assert int(near.sum()) == 0
    assert torch.equal(got, want)
    assert 0.001 < float(want.double().mean()) < 0.5
    assert torch.equal(got, depth_discontuity_mask(depth))


@pytest.mark.parametrize("H,W,ds", [(2048, 1334, 8), (100, 70, 3)])
def test_pixel_bias_vs_interpolate_fp64(cuda, H, W, ds):
    from goliath_b200.mesh_vae import CameraPixelBias

    g = torch.Generator(device=cuda).manual_seed(H)
    m = CameraPixelBias(H, W, ["a", "b", "c", "d"], ds).to(cuda)
    with torch.no_grad():
        m.bias.normal_(generator=g)
    idx = torch.tensor([1, 0, 1], device=cuda)          # items 0 and 2 share camera 1
    rgb = torch.randn(3, 3, H, W, device=cuda, generator=g, requires_grad=True)
    cot = torch.randn(3, 3, H, W, device=cuda, generator=g)
    out = m(idx, rgb)
    b64 = m.bias.detach().double().requires_grad_()
    want = bf.pixel_bias(rgb.detach().double(), b64, idx, H, W)
    # torch's fp32 interpolate takes the same fp32 source index; in fp64 the index itself differs by an ulp of the
    # source coordinate (up to 2^-16 of the bilinear weights at 256 texels)
    assert _maxrel(out, bf.pixel_bias(rgb.detach(), m.bias.detach(), idx, H, W)) <= 1e-6
    assert _maxrel(out, want) <= 5e-5
    (gw,) = torch.autograd.grad((want * cot.double()).sum(), [b64])
    g1 = torch.autograd.grad((m(idx, rgb) * cot).sum(), [m.bias, rgb])
    g2 = torch.autograd.grad((m(idx, rgb) * cot).sum(), [m.bias, rgb])
    assert _maxrel(g1[0], gw) <= 1e-4
    assert torch.equal(g1[0], g2[0]) and torch.equal(g1[1], cot)
    assert torch.equal(g1[0][[2, 3]], torch.zeros_like(g1[0][[2, 3]]))   # cameras no item uses
    # without an image: the reference's forward, bias_up [B,1,H,W]
    assert _maxrel(m(idx), F.interpolate(b64[idx], size=(H, W), mode="bilinear")) <= 5e-5


def _camera_batch():
    return [bf.IDENTITY, "410244", "401033", "410244", "402100"]     # identity, grey, colour, grey again, colour


@pytest.mark.parametrize("training", [False, True])
def test_calv5_vs_reference_fp64(cuda, training):
    from goliath_b200.photo_loss import CalV5

    cal = bf.seeded_fill(CalV5(bf.CAMERAS, bf.IDENTITY)).to(cuda).train(training)
    names = _camera_batch()
    g = torch.Generator(device=cuda).manual_seed(9)
    img = 100 * torch.rand(len(names), 3, 64, 48, device=cuda, generator=g)
    cot = torch.randn(img.shape, device=cuda, generator=g)
    idx = cal.name_to_idx(names)
    out = cal(img, idx)
    p64 = cal.holder.params.detach().double().requires_grad_()
    want = bf.cal_v5(img.double(), p64, idx, cal.identity_idx, cal.grey_idxs, training=training)
    assert _maxrel(out, want) <= 1e-6
    assert torch.equal(out[0], img[0])                            # the identity camera passes through
    (gp,) = torch.autograd.grad((out * cot).sum(), [cal.holder.params])
    (gw,) = torch.autograd.grad((want * cot.double()).sum(), [p64])
    assert _nrel(gp, gw) <= 1e-5
    assert torch.equal(gp[cal.identity_idx], torch.zeros(6, device=cuda))


def test_learnable_blur_vs_reference_fp64(cuda):
    from goliath_b200.photo_loss import LearnableBlur

    lb = bf.seeded_fill(LearnableBlur(bf.CAMERAS)).to(cuda)
    names = _camera_batch()
    g = torch.Generator(device=cuda).manual_seed(10)
    img = 100 * torch.rand(len(names), 3, 64, 48, device=cuda, generator=g, requires_grad=True)
    cot = torch.randn(img.shape, device=cuda, generator=g)
    idx = torch.tensor([bf.CAMERAS.index(c) for c in names], device=cuda)
    w64 = lb.weights_raw.detach().double().requires_grad_()
    want = bf.learn_blur(img.detach().double(), w64, idx)
    out = lb(img, names)
    assert _maxrel(out, want) <= 1e-5
    gw, gi = torch.autograd.grad((out * cot).sum(), [lb.weights_raw, img])
    (gw64,) = torch.autograd.grad((want * cot.double()).sum(), [w64])
    assert _nrel(gw, gw64) <= 1e-4
    assert torch.equal(lb.reg(names), lb.weights_raw[idx])


# ------------------------------------------------------------------------------------------ the frame
@pytest.fixture(scope="module")
def frame(cuda):
    from goliath_b200.mesh_vae import AutoEncoder

    z = np.load(GOLD)
    m = bf.seeded_fill(AutoEncoder(**bf.config(), assets=bf.assets())).to(cuda).eval()
    # the fixture's drtk stand-in has no edge-gradient estimator
    m.renderer.forward = functools.partial(m.renderer.forward, edge_grad=False)
    inp = {k: torch.from_numpy(z["in_" + k]).to(cuda) for k in ("pose", "campos", "registration_vertices", "K", "Rt")}
    inp["ambient_occlusion"] = bf.ambient_occlusion(2).to(cuda)
    inp["camera_id"] = list(bf.BATCH_CAMERAS)
    return m, inp, z


def _summary(t):
    f = t.detach().double().reshape(-1).cpu()
    idx = torch.linspace(0, f.numel() - 1, 256, dtype=torch.float64).long()
    return np.concatenate([[f.mean().item(), f.std().item(), f.abs().max().item(), float(f.numel())], f[idx].numpy()])


def _check(z, kind, k, t, factor=4.0, floor=1e-4):
    """None, or (key, error, bound) when the summary of t is further from the fixture's than the bound"""
    s, ref = _summary(t), z["%s_%s" % (kind, k)]
    assert tuple(t.shape) == tuple(z["shape_%s_%s" % (kind, k)]), k
    a, b = np.delete(s, 3), np.delete(ref, 3)
    err = float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))
    bound = max(floor, factor * float(z["err32_%s_%s" % (kind, k)]))
    return None if err <= bound else (kind, k, err, bound)


def test_autoencoder_vs_reference_fixture(frame):
    m, inp, z = frame
    preds = m(**inp)
    assert list(preds) == json.loads(bytes(z["out_keys_json"]).decode())
    bad = []
    for k, t in preds.items():
        if k == "depth_disc_mask":
            want = torch.from_numpy(z["depth_disc_mask"])
            assert t.dtype == torch.bool and t.shape == want.shape
            assert int((t.cpu() != want).sum()) <= 20       # pixels next to a threshold crossing of the fp32 depth
        else:
            bad.append(_check(z, "out", k, t))
    g = torch.Generator().manual_seed(77)
    wr = torch.randn(preds["rgb"].shape, generator=g, dtype=torch.float64).float().to(preds["rgb"].device)
    wa = torch.randn(preds["alpha"].shape, generator=g, dtype=torch.float64).float().to(preds["rgb"].device)
    names = json.loads(bytes(z["grad_names_json"]).decode())
    params = dict(m.named_parameters())
    grads = torch.autograd.grad((preds["rgb"] * wr).sum() + (preds["alpha"] * wa).sum(), [params[n] for n in names])
    for n, gr in zip(names, grads):
        # every parameter gradient reaches back through the render's backward, this project's own fp32 formulation
        # (fixed-order gathers, DESIGN.md R9''), which sits further from the fp64 reference than the reference's own
        # fp32 run: the texture path up to 1.7e-4 norm-wise (upscale_net's untied bias), hence a floor of 5e-4; the
        # encoders and verts_conv see the image only through the geometry gradient, up to 12x the fp32 run's error
        # there (2 % norm-wise for verts_conv), hence 16x on that path
        geometry = n.startswith("encoder") or n.startswith("decoder.verts_conv")
        bad.append(_check(z, "grad", n, gr, factor=16.0 if geometry else 4.0, floor=5e-4))
    bad = [b for b in bad if b is not None]
    assert not bad, bad


def test_autoencoder_training_mode_scales_the_calibration_gradient(frame):
    """with the encoders' noise_std = 0 the training-mode frame equals eval; only CalV5's per-camera scale differs"""
    m, inp, _ = frame
    params = [m.cal.holder.params, m.pixel_cal.bias]

    def run():
        p = m(**inp)
        return p["rgb"].detach(), torch.autograd.grad(p["rgb"].sum() + p["alpha"].sum(), params)

    rgb_e, (gc_e, gp_e) = run()
    old = m.encoder.noise_std, m.encoder_face.encoder.noise_std
    m.encoder.noise_std = m.encoder_face.encoder.noise_std = 0.0
    m.train()
    try:
        rgb_t, (gc_t, gp_t) = run()
    finally:
        m.eval()
        m.encoder.noise_std, m.encoder_face.encoder.noise_std = old
    assert _maxrel(rgb_t, rgb_e) <= 1e-6
    assert _nrel(gp_t, gp_e) <= 1e-6
    grey, colour = (m.cal.holder.key_list.index(c) for c in bf.BATCH_CAMERAS)
    assert _nrel(gc_t[grey], m.cal.gs_lrscale * gc_e[grey]) <= 1e-5
    assert _nrel(gc_t[colour], m.cal.col_lrscale * gc_e[colour]) <= 1e-5


def test_frame_forward_backward_without_host_sync(frame):
    m, inp, _ = frame
    params = [p for p in m.parameters() if p.requires_grad]

    def step():
        p = m(**inp)
        return torch.autograd.grad(p["rgb"].sum() + p["alpha"].sum(), params, allow_unused=True)

    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
