"""GPU checks of the hand avatar's frame (csrc/hand_frame.cu, goliath_b200/hand_mvp.py): the valid-primitive gather
against torch's boolean indexing, the render finish against a torch restatement, `hand_mvp.AutoEncoder` against
tests/golden/hand_frame_ref.npz (the reference's own AutoEncoder) in eval and both training branches, the frame's
forward + backward without a host synchronisation, and one training step at the example configuration's size."""
import json
import os

import numpy as np
import pytest
import torch

import hand_frame_restate as hf

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hand_frame_ref.npz")
VOLRADIUS = 2000.0


def _nrel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------ valid-primitive gather
def _prims(cuda, B, K, seed):
    g = torch.Generator(device=cuda).manual_seed(seed)
    tpl = torch.randn(B, K, 8, 16, 16, 4, device=cuda, generator=g)
    pos = 1000 * torch.randn(B, K, 3, device=cuda, generator=g)
    rot = torch.randn(B, K, 3, 3, device=cuda, generator=g)
    scale = 512 + torch.randn(B, K, 3, device=cuda, generator=g)
    return tpl, pos, rot, scale


@pytest.mark.parametrize("which", ["tube", "none", "all"])
def test_valid_gather_vs_boolean_indexing(cuda, which):
    from goliath_b200.hand_mvp import slot_table, valid_gather

    B, K = 2, 4096
    if which == "tube":
        valid = torch.as_tensor(np.load(GOLD)["valid_prims"]).to(cuda)
    else:
        valid = torch.full((K,), which == "all", dtype=torch.bool, device=cuda)
    slot, n = slot_table(valid)
    assert n == int(valid.sum())
    ins = [t.requires_grad_() for t in _prims(cuda, B, K, 1)]
    outs = valid_gather(*ins, slot, n, VOLRADIUS)
    tpl, pos, rot, scale = ins
    want = (tpl[:, valid].contiguous(), (pos / VOLRADIUS)[:, valid].contiguous(), rot[:, valid].contiguous(),
            scale[:, valid].contiguous())
    for o, w in zip(outs, want):
        assert o.shape == w.shape and torch.equal(o, w)
    g = torch.Generator(device=cuda).manual_seed(2)
    cots = [torch.randn(o.shape, device=cuda, generator=g) for o in outs]
    grads = torch.autograd.grad(outs, ins, cots)
    again = torch.autograd.grad(valid_gather(*ins, slot, n, VOLRADIUS), ins, cots)
    for a, b in zip(grads, again):
        assert torch.equal(a, b)
    for i, (gr, c) in enumerate(zip(grads, cots)):
        full = torch.zeros_like(ins[i]).index_put((torch.arange(B, device=cuda)[:, None],
                                                   valid.nonzero()[:, 0][None]), c)
        if i == 1:      # d(pos / volradius): the incoming gradient times 1 / volradius
            full = full / VOLRADIUS
        assert torch.equal(gr, full), i
        assert not gr[:, ~valid].any()


# ------------------------------------------------------------------------------------------ render finish
def _finish_ref(rayrgba, w, b, grey, bg):
    """render_raymarcher.py:69-70, CalV5 (color_cal.py:211-241) with a grey camera, hand_mvp.py:252-255"""
    x = rayrgba.permute(0, 3, 1, 2)
    rgb, alpha = x[:, :3], x[:, 3:4]
    if w is not None:
        out = []
        for i in range(rgb.shape[0]):
            if grey[i]:
                out.append((rgb[i:i + 1] * w[i, :, None, None]).sum(1, keepdim=True).expand(-1, 3, -1, -1) + b[i].sum())
            else:
                out.append(rgb[i:i + 1] * w[i, :, None, None] + b[i, :, None, None])
        rgb = torch.cat(out)
    if bg is not None:
        rgb = rgb + (1.0 - alpha) * bg
    return rgb, alpha


@pytest.mark.parametrize("cal,bg", [(True, True), (False, True), (True, False), (False, False)])
def test_finish_vs_torch(cuda, cal, bg):
    from goliath_b200.hand_mvp import hand_finish

    B, H, W = 2, 667, 1024
    g = torch.Generator(device=cuda).manual_seed(4)
    ray = torch.rand(B, H, W, 4, device=cuda, generator=g)
    ray[..., :3] *= 255.0
    ray.requires_grad_()
    w = (1.0 + 0.1 * torch.randn(B, 3, device=cuda, generator=g)).requires_grad_() if cal else None
    b = (0.05 * torch.randn(B, 3, device=cuda, generator=g)).requires_grad_() if cal else None
    grey = torch.tensor([0, 1], dtype=torch.int32, device=cuda) if cal else None
    back = 255.0 * torch.rand(B, 3, H, W, device=cuda, generator=g) if bg else None
    rgb, alpha = hand_finish(ray, w, b, grey, back)
    r64 = ray.detach().double().requires_grad_()
    w64 = w.detach().double().requires_grad_() if cal else None
    b64 = b.detach().double().requires_grad_() if cal else None
    want_rgb, want_alpha = _finish_ref(r64, w64, b64, grey, None if back is None else back.double())
    assert _nrel(rgb, want_rgb) <= 1e-6 and torch.equal(alpha, ray.detach()[..., 3:].permute(0, 3, 1, 2))
    if not cal and not bg:
        assert torch.equal(rgb, ray.detach()[..., :3].permute(0, 3, 1, 2))
    gr = torch.randn(rgb.shape, device=cuda, generator=g)
    ga = torch.randn(alpha.shape, device=cuda, generator=g)
    leaves = [ray] + ([w, b] if cal else [])
    got = torch.autograd.grad((rgb * gr).sum() + (alpha * ga).sum(), leaves)
    rgb2, alpha2 = hand_finish(ray, w, b, grey, back)
    got2 = torch.autograd.grad((rgb2 * gr).sum() + (alpha2 * ga).sum(), leaves)
    for x, y in zip(got, got2):
        assert torch.equal(x, y)
    want = torch.autograd.grad((want_rgb * gr.double()).sum() + (want_alpha * ga.double()).sum(),
                               [r64] + ([w64, b64] if cal else []))
    for x, y, n in zip(got, want, ("rayrgba", "cal_w", "cal_b")):
        assert _nrel(x, y) <= 1e-5, n
        assert _nrel(x[0], y[0]) <= 1e-5 and _nrel(x[1], y[1]) <= 1e-5, n


# ------------------------------------------------------------------------------------------ the frame
@pytest.fixture(scope="module")
def frame(cuda):
    from goliath_b200.hand_mvp import AutoEncoder

    z = np.load(GOLD)
    a = hf.assets()
    m = AutoEncoder(**hf.config(), assets=a)
    want = json.loads(bytes(z["keys_json"]).decode())
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == want
    m.load_state_dict(hf.seeded_fill(AutoEncoder(**hf.config(), assets=a)).state_dict(), strict=True)
    m = m.to(cuda)
    inp = {k: torch.from_numpy(z["in_" + k]).to(cuda)
           for k in ("pose", "campos", "ambient_occlusion", "K", "Rt", "background")}
    inp["camera_id"] = list(hf.BATCH_CAMERAS)
    return m, inp, z


class _Capture:
    """wraps the frame's mvpraymarch to keep its inputs and output"""

    def __init__(self, monkeypatch):
        import goliath_b200.mvpraymarch as mod

        self.fn, self.call = mod.mvpraymarch, None
        monkeypatch.setattr(mod, "mvpraymarch", self)

    def __call__(self, raypos, raydir, stepsize, tminmax, primtransf, template, warp=None, **kw):
        out = self.fn(raypos, raydir, stepsize, tminmax, primtransf, template=template, warp=warp, **kw)
        pos, rot, scale = primtransf
        self.call = {"raypos": raypos, "raydir": raydir, "tminmax": tminmax, "primpos": pos, "primrot": rot,
                     "primscale": scale, "template": template, "rayrgba": out}
        return out


def _check(z, mode, kind, k, t, factor):
    s, ref = hf.summarise(t), z["%s_%s_%s" % (mode, kind, k)]
    assert tuple(t.shape) == tuple(z["%s_shape_%s_%s" % (mode, kind, k)]), (mode, kind, k)
    err = hf.nrel_summary(s, ref)
    bound = factor * float(z["%s_err32_%s_%s" % (mode, kind, k)])
    return None if err <= bound else (mode, kind, k, err, bound)


# each comparison is bounded by a multiple of the reference frame's own fp32-vs-fp64 error for that quantity; where
# that error is zero (exact gathers, the zero-delta primitive scale) the result must be exact
FACTOR = 8.0


@pytest.mark.parametrize("mode", hf.MODES)
def test_autoencoder_vs_reference_fixture(frame, monkeypatch, mode):
    m, inp, z = frame
    cap = _Capture(monkeypatch)
    m.train(mode != "eval")
    try:
        preds = m(**inp, iteration=hf.ITERATION[mode])
    finally:
        m.eval()
    assert list(preds) == json.loads(bytes(z["%s_out_keys_json" % mode]).decode())
    assert torch.equal(preds["valid_prims"].cpu(), torch.as_tensor(z["valid_prims"]))
    bad = []
    for k, t in preds.items():
        if t.dtype == torch.bool:
            continue
        if k == "learn_blur_weights":
            assert np.array_equal(hf.summarise(t), z["%s_out_%s" % (mode, k)])
            continue
        bad.append(_check(z, mode, "out", k, t, FACTOR))
    for k in ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "template"):
        bad.append(_check(z, mode, "march", k, cap.call[k], FACTOR))
    names = json.loads(bytes(z["grad_names_json"]).decode())
    params = dict(m.named_parameters())
    w = hf.functional_weights({k: preds[k].shape for k in hf.PRIM_KEYS})
    f = sum((preds[k] * w[k].float().to(preds[k].device)).sum() for k in hf.PRIM_KEYS)
    pre = torch.autograd.grad(f, [params[n] for n in names], retain_graph=True)
    for n, g in zip(names, pre):
        bad.append(_check(z, mode, "pre", n, g, FACTOR))
    wr, wa = hf.cotangents(preds["rgb"].shape, preds["alpha"].shape)
    extra = ["cal.holder.params", "learn_blur.weights_raw"]
    post = torch.autograd.grad((preds["rgb"] * wr.float().cuda()).sum() + (preds["alpha"] * wa.float().cuda()).sum(),
                               [cap.call["rayrgba"]] + [params[k] for k in extra])
    for k, g in zip(["rayrgba"] + extra, post):
        bad.append(_check(z, mode, "post", k, g, FACTOR))
    bad = [b for b in bad if b is not None]
    assert not bad, bad


@pytest.mark.parametrize("training", [False, True])
def test_frame_forward_backward_without_host_sync(frame, training):
    m, inp, _ = frame
    params = [p for p in m.parameters() if p.requires_grad]
    m.train(training)

    def step():
        p = m(**inp, iteration=5000)
        return torch.autograd.grad(p["rgb"].sum() + p["alpha"].sum(), params, allow_unused=True)

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


def test_training_step_at_example_size(cuda):
    """B = 2 at 1024 x 667 (hand_mvp_example.yml's 2048 x 1334 at the loader's downsample of 2) with the background,
    an L2 loss on rgb and an L1 loss on alpha: every parameter gets a finite gradient, and alphadecoder a nonzero one
    through the alpha path alone"""
    from goliath_b200.hand_mvp import AutoEncoder

    z = np.load(GOLD)
    H, W = 667, 1024
    m = hf.seeded_fill(AutoEncoder(**hf.config(H, W), assets=hf.assets())).to(cuda).train()
    pose = torch.from_numpy(z["in_pose"]).to(cuda)
    K, Rt, campos = hf.side_cameras(_posed_points(m, pose), H, W)
    inp = {"pose": pose, "campos": campos.float().to(cuda), "K": K.float().to(cuda), "Rt": Rt.float().to(cuda),
           "ambient_occlusion": torch.from_numpy(z["in_ambient_occlusion"]).to(cuda),
           "camera_id": list(hf.BATCH_CAMERAS), "background": hf.background(2, H, W).to(cuda)}
    preds = m(**inp, iteration=5000)
    g = torch.Generator(device=cuda).manual_seed(5)
    target = 255.0 * torch.rand(preds["rgb"].shape, device=cuda, generator=g)
    mask = (torch.rand(preds["alpha"].shape, device=cuda, generator=g) > 0.5).float()
    params = dict(m.named_parameters())
    l2 = ((preds["rgb"] - target) ** 2).mean()
    l1 = (preds["alpha"] - mask).abs().mean()
    grads = torch.autograd.grad(0.0016 * l2 + 10.0 * l1, list(params.values()), allow_unused=True)
    for (n, p), gr in zip(params.items(), grads):
        assert gr is not None and bool(torch.isfinite(gr).all()), n
    alpha_only = torch.autograd.grad(m(**inp, iteration=5000)["alpha"].sub(mask).abs().mean(),
                                     [params["geomdecoder.alphadecoder.texbranch.6.bias"]])[0]
    assert float(alpha_only.abs().max()) > 0
    assert 0.05 < float((preds["alpha"] > 0.5).float().mean()) < 0.95


def _posed_points(m, pose):
    with torch.no_grad():
        return m.lbs_fn.pose(torch.zeros_like(m.lbs_fn.lbs_template_verts), pose).cpu().double()
