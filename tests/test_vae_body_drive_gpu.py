"""GPU checks of the drivable body avatar (csrc/body_drive.cu, goliath_b200/{face,shadow,mesh_vae_drivable}.py): the
three kernels against fp64 torch restatements (tests/body_drive_restate.py) at the frame's sizes and at odd sizes, the
face decoder's grad-disabled path against its differentiable one, `mesh_vae_drivable.AutoEncoder` against
tests/golden/body_drive_ref.npz (the reference's own model) in eval and in training mode, and the frame without a host
synchronisation.

Each kernel's forward bound is calibrated on torch's own fp32 error against fp64 on the same inputs (TF32 off)."""
import json
import os

import numpy as np
import pytest
import torch

import body_drive_restate as bd

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "body_drive_ref.npz")


def _maxrel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _nrel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture
def no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


@pytest.mark.parametrize("B", [1, 4])
def test_face_tex_tail_vs_fp64(cuda, no_tf32, B):
    from goliath_b200.face import face_tex_tail
    from goliath_b200.nn import ConvTranspose2dWNUB

    g = torch.Generator(device=cuda).manual_seed(B)
    layer = ConvTranspose2dWNUB(8, 3, 1024, 1024).to(cuda)
    with torch.no_grad():
        layer.bias.normal_(0, 0.05, generator=g)
        layer.weight_g.uniform_(0.5, 1.5, generator=g)
    fb = 0.05 * torch.randn(3, 1024, 1024, device=cuda, generator=g)
    x = torch.nn.functional.leaky_relu(torch.randn(B, 8, 512, 512, device=cuda, generator=g), 0.2)
    with torch.no_grad():
        raw, tex = face_tex_tail(x, layer, fb)
        args = (layer.weight_v, layer.weight_g, layer.bias, fb)
        want = bd.face_tex_tail(x.double(), *(t.double() for t in args))
        torch32 = bd.face_tex_tail(x, *args)
    for got, w, t in zip((raw, tex), want, torch32):
        bound = max(4.0 * _maxrel(t, w), 1e-6)
        assert _maxrel(got, w) <= bound, (_maxrel(got, w), bound)


@pytest.mark.parametrize("B,Hs,Ws", [(1, 1024, 1024), (4, 1024, 1024), (2, 777, 1023)])
def test_face_tex_cond_vs_fp64(cuda, B, Hs, Ws):
    from goliath_b200.mesh_vae_drivable import face_tex_cond

    g = torch.Generator(device=cuda).manual_seed(Hs + B)
    tex = 255 * torch.rand(B, 3, Hs, Ws, device=cuda, generator=g)
    mask = torch.rand(1, 1, 512, 512, device=cuda, generator=g)
    got = face_tex_cond(tex, mask)
    want = bd.face_tex_cond(tex.double(), mask.double())
    bound = max(4.0 * _maxrel(bd.face_tex_cond(tex, mask), want), 1e-6)
    assert got.shape == (B, 3, 512, 512)
    assert _maxrel(got, want) <= bound, (_maxrel(got, want), bound)


@pytest.mark.parametrize("B,size", [(1, 2048), (4, 2048), (2, 1000)])
def test_pose_shadow_vs_fp64(cuda, B, size):
    from goliath_b200.shadow import pose_shadow

    g = torch.Generator(device=cuda).manual_seed(size + B)
    x = (2 * torch.randn(B, 1, 128, 128, device=cuda, generator=g)).requires_grad_()
    cot = torch.randn(B, 1, size, size, device=cuda, generator=g)
    out = pose_shadow(x, 1.0, size)
    x64 = x.detach().double().requires_grad_()
    want = bd.pose_shadow(x64, 1.0, size)
    bound = max(4.0 * _maxrel(bd.pose_shadow(x.detach(), 1.0, size), want), 1e-6)
    assert _maxrel(out, want) <= bound, (_maxrel(out, want), bound)
    (g1,) = torch.autograd.grad((out * cot).sum(), [x])
    (g2,) = torch.autograd.grad((pose_shadow(x, 1.0, size) * cot).sum(), [x])
    (g64,) = torch.autograd.grad((want * cot.double()).sum(), [x64])
    (g32,) = torch.autograd.grad((bd.pose_shadow(x, 1.0, size) * cot).sum(), [x])
    assert torch.equal(g1, g2)                                          # gather-only: the same bits on every call
    assert _nrel(g1, g64) <= max(4.0 * _nrel(g32, g64), 1e-6), (_nrel(g1, g64), _nrel(g32, g64))


def test_face_decoder_fast_path_matches_autograd_path(cuda):
    from goliath_b200.face import FaceDecoderFrontal

    dec = bd.seeded_fill(FaceDecoderFrontal(bd.assets(), n_vert_out=3 * bd.N_FACE_VERTS)).to(cuda)
    z = torch.randn(2, 256, device=cuda, generator=torch.Generator(device=cuda).manual_seed(3))
    with torch.no_grad():
        fast = dec(z)
    slow = dec(z)
    assert list(fast) == ["face_geom", "face_tex_raw", "face_tex"] and list(slow) == list(fast)
    assert torch.equal(fast["face_geom"], slow["face_geom"].detach())
    for k in ("face_tex_raw", "face_tex"):
        assert fast[k].shape == (2, 3, 1024, 1024)
        assert _maxrel(fast[k], slow[k]) <= 1e-5, (k, _maxrel(fast[k], slow[k]))


# ------------------------------------------------------------------------------------------ the frame
@pytest.fixture(scope="module")
def frame(cuda):
    from goliath_b200.mesh_vae_drivable import AutoEncoder

    z = np.load(GOLD)
    m = bd.seeded_fill(AutoEncoder(**bd.config(), assets=bd.assets())).to(cuda).eval()
    inp = {k: torch.from_numpy(z["in_" + k]).to(cuda) for k in ("lbs_motion", "campos", "geom", "ao", "K", "Rt",
                                                                "face_embs")}
    inp["_index"] = {"camera": ["410244", "401033"]}
    return m, inp, z


def _summary(t):
    f = t.detach().double().reshape(-1).cpu()
    idx = torch.linspace(0, f.numel() - 1, 256, dtype=torch.float64).long()
    return np.concatenate([[f.mean().item(), f.std().item(), f.abs().max().item(), float(f.numel())], f[idx].numpy()])


def _check(z, mode, kind, k, t, factor=4.0, floor=1e-4):
    s, ref = _summary(t), z["%s_%s_%s" % (mode, kind, k)]
    assert tuple(t.shape) == tuple(z["%s_shape_%s_%s" % (mode, kind, k)]), k
    a, b = np.delete(s, 3), np.delete(ref, 3)
    err = float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))
    bound = max(floor, factor * float(z["%s_err32_%s_%s" % (mode, kind, k)]))
    return None if err <= bound else (kind, k, err, bound)


def _flat(preds):
    out = {}
    for k, v in preds.items():
        out.update({"%s.%s" % (k, kk): vv for kk, vv in v.items()} if isinstance(v, dict) else {k: v})
    return out


_COTANGENTS = {}


def _run(m, inp, mode):
    """the frame's predictions (face_dec_preds flattened) and the fixture's seeded loss; the cotangents reach the
    device on the first call of each mode only, so later calls issue no copy"""
    i = dict(inp)
    if mode == "eval":
        i["ao"] = None
    preds = _flat(m(**i))
    if mode not in _COTANGENTS:
        g = torch.Generator().manual_seed(77)
        keys = ["rgb"] + (["pose_shadow_map"] if "pose_shadow_map" in preds else [])
        _COTANGENTS[mode] = {k: torch.randn(preds[k].shape, generator=g, dtype=torch.float64).float()
                             .to(preds[k].device) for k in keys}
    loss = sum((preds[k] * w).sum() for k, w in _COTANGENTS[mode].items())
    return preds, loss


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_autoencoder_vs_reference_fixture(frame, mode):
    m, inp, z = frame
    old = m.encoder.noise_std, m.encoder_face.noise_std
    m.encoder.noise_std = m.encoder_face.noise_std = 0.0
    m.train(mode == "train")
    try:
        preds, loss = _run(m, inp, mode)
        assert list(preds) == json.loads(bytes(z[mode + "_out_keys_json"]).decode())
        bad = [_check(z, mode, "out", k, t) for k, t in preds.items()]
        names = json.loads(bytes(z[mode + "_grad_names_json"]).decode())
        params = dict(m.named_parameters())
        grads = torch.autograd.grad(loss, [params[n] for n in names])
    finally:
        m.eval()
        m.encoder.noise_std, m.encoder_face.noise_std = old
    for n, gr in zip(names, grads):
        # as in tests/test_vae_body_frame_gpu.py: every gradient reaches back through the render's own fp32 backward,
        # and the encoders and verts_conv see the image only through the geometry gradient
        geometry = n.startswith("encoder") or n.startswith("decoder.verts_conv")
        bad.append(_check(z, mode, "grad", n, gr, factor=16.0 if geometry else 4.0, floor=5e-4))
    bad = [b for b in bad if b is not None]
    assert not bad, bad


def test_decoder_leaves_callers_embs_conv(frame):
    m, inp, _ = frame
    B = inp["lbs_motion"].shape[0]
    embs_conv = torch.randn(B, 32, 64, 64, device=inp["lbs_motion"].device)
    before = embs_conv.clone()
    face_embs = torch.randn(B, 256, device=embs_conv.device)
    with torch.no_grad():
        out = m.decoder(inp["lbs_motion"], None, face_embs, embs_conv=embs_conv)
    assert torch.equal(embs_conv, before)
    assert not torch.equal(out["embs_conv"], before)
    assert torch.equal(out["embs_conv"][:, :, :32], before[:, :, :32])      # only the face block [32:, :32] merges


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_frame_without_host_sync(frame, mode):
    m, inp, _ = frame
    params = [p for p in m.parameters() if p.requires_grad]

    def step():
        if mode == "eval":
            with torch.no_grad():
                m(**{**inp, "ao": None})
            return
        _, loss = _run(m, inp, mode)
        torch.autograd.grad(loss, params, allow_unused=True)

    m.train(mode == "train")
    try:
        step()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            step()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
    finally:
        m.eval()
