"""GPU checks of the relightable hand teacher's frame (`goliath_b200.hand_teacher.AutoEncoder`): every mode of
tests/golden/hand_teacher_frame_ref.npz (the reference's own teacher AutoEncoder), the flow that initialises a
teacher from a hand_mvp checkpoint, SingleLightCycleDecorator's [B,1,1] intensity, one EnvSpinDecorator frame at the
example size with 512 lights, forward + backward without a host synchronisation, and one training step at the example
size with the real chunk size."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

import hand_frame_restate as hf
import hand_teacher_frame_restate as ht

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "hand_teacher_frame_ref.npz")
H, W = 667, 1024       # hand_teacher_mvp_example.yml's 2048 x 1334 at the data loader's downsample of 2
MARCH_KEYS = ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "template")
# each comparison is bounded by a multiple of the reference frame's own fp32-vs-fp64 error for that quantity, as in
# tests/test_hand_frame_gpu.py
FACTOR = 8.0


def _teacher(config, seeded=True):
    from goliath_b200.hand_teacher import AutoEncoder

    m = AutoEncoder(**config, assets=hf.assets())
    if seeded:
        hf.seeded_fill(m)
    return m


def _posed_points(m, pose):
    with torch.no_grad():
        return m.lbs_fn.pose(torch.zeros_like(m.lbs_fn.lbs_template_verts), pose).cpu().double()


@pytest.fixture(scope="module")
def frame(cuda):
    z = np.load(GOLD)
    m = _teacher(hf.config(), seeded=False)
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == json.loads(bytes(z["keys_json"]).decode())
    sd = hf.seeded_fill(_teacher(hf.config(), seeded=False)).state_dict()
    m.load_state_dict(sd, strict=True)
    env = _teacher(ht.env_config(), seeded=False)
    res = env.load_state_dict(sd, strict=False)
    assert not res.missing_keys
    m, env = ht.reduce(m.to(cuda)), ht.reduce(env.to(cuda)).eval()
    inp = {k: torch.from_numpy(z["in_" + k]).to(cuda)
           for k in ("pose", "campos", "K", "Rt", "light_pos", "light_intensity", "background")}
    inp["camera_id"] = list(hf.BATCH_CAMERAS)
    env_inp = {k: torch.from_numpy(z["env_in_" + k]).to(cuda)
               for k in ("campos", "K", "Rt", "light_pos", "light_intensity", "envbg")}
    env_inp.update(pose=inp["pose"], camera_id=list(hf.BATCH_CAMERAS), index=[3, 4], n_lights=torch.ones(2, 1))
    return m, env, inp, env_inp, z


class _Capture:
    """wraps the frame's mvpraymarch to keep the inputs and output of its last call"""

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


def _check(z, mode, kind, k, t):
    s, ref = hf.summarise(t), z["%s_%s_%s" % (mode, kind, k)]
    assert tuple(t.shape) == tuple(z["%s_shape_%s_%s" % (mode, kind, k)]), (mode, kind, k)
    err = hf.nrel_summary(s, ref)
    bound = FACTOR * float(z["%s_err32_%s_%s" % (mode, kind, k)])
    return None if err <= bound else (mode, kind, k, err, bound)


def _set_mode(m, mode):
    """the fixture's training state of each mode; `fresh` is the constructor's: geometry in eval, the rest training"""
    if mode in ("eval", "env"):
        m.eval()
    elif mode == "fresh":
        m.train()
        m.geomdecoder.eval()
    else:
        m.train()


@pytest.mark.parametrize("mode", ht.MODES)
def test_autoencoder_vs_reference_fixture(frame, monkeypatch, mode):
    m, env, inp, env_inp, z = frame
    model, x = (env, env_inp) if mode == "env" else (m, inp)
    cap = _Capture(monkeypatch)
    _set_mode(model, mode)
    try:
        preds = model(**x, iteration=ht.ITERATION[mode])
        call = cap.call
        with torch.no_grad():
            sp = dict(preds)
            sp["primrgb"] = 255.0 * preds["primshadow"]
            srgb, salpha, none = model.render(x["K"], x["Rt"], sp)
    finally:
        model.eval()
    assert none is None
    assert list(preds) == json.loads(bytes(z["%s_out_keys_json" % mode]).decode())
    assert preds["ae"] is model
    assert torch.equal(preds["valid_prims"].cpu(), torch.as_tensor(z["valid_prims"]))
    bad = []
    for k, t in preds.items():
        if not torch.is_tensor(t) or t.dtype == torch.bool:
            continue
        if k == "learn_blur_weights":
            assert np.array_equal(hf.summarise(t), z["%s_out_%s" % (mode, k)])
            continue
        bad.append(_check(z, mode, "out", k, t))
    for k in MARCH_KEYS:
        bad.append(_check(z, mode, "march", k, call[k]))
    for k, t in (("rgb", srgb), ("alpha", salpha), ("primrgba", sp["primrgba"])):
        bad.append(_check(z, mode, "shadow", k, t))
    if mode in ht.GRAD_MODES:
        names = json.loads(bytes(z["grad_names_json"]).decode())
        params = dict(model.named_parameters())
        w = ht.functional_weights({k: preds[k].shape for k in ht.PRIM_KEYS if k in preds})
        f = sum((preds[k] * w[k].float().to(preds[k].device)).sum() for k in w)
        pre = torch.autograd.grad(f, [params[n] for n in names], retain_graph=True, allow_unused=True)
        for n, g in zip(names, pre):
            bad.append(_check(z, mode, "pre", n, torch.zeros_like(params[n]) if g is None else g))
        wr, wa = hf.cotangents(preds["rgb"].shape, preds["alpha"].shape)
        extra = ["cal.holder.params", "learn_blur.weights_raw"]
        f_post = (preds["rgb"] * wr.float().cuda()).sum() + (preds["alpha"] * wa.float().cuda()).sum()
        post = torch.autograd.grad(f_post, [call["rayrgba"]] + [params[k] for k in extra])
        for k, g in zip(["rayrgba"] + extra, post):
            bad.append(_check(z, mode, "post", k, g))
    bad = [b for b in bad if b is not None]
    assert not bad, bad


def test_fresh_model_runs_geometry_in_eval(cuda):
    m = _teacher(hf.config(), seeded=False)
    assert m.training and not m.geomdecoder.training and m.relightdecoder.training and m.poseencoder2.training


def test_teacher_initialised_from_hand_checkpoint(frame):
    """train.ckpt of hand_teacher_mvp_example.yml: a hand_mvp state dict loads non-strictly, missing exactly the two
    modules the teacher adds, and the loaded teacher renders"""
    from goliath_b200.hand_mvp import AutoEncoder as HandAE

    _, _, inp, _, _ = frame
    hand = hf.seeded_fill(HandAE(**hf.config(), assets=hf.assets()))
    t = _teacher(hf.config(), seeded=False)
    res = t.load_state_dict(hand.state_dict(), strict=False)
    assert not res.unexpected_keys
    assert set(res.missing_keys) == {k for k in t.state_dict() if k.startswith(("poseencoder2.", "relightdecoder."))}
    assert any(k.startswith("poseencoder2.") for k in res.missing_keys)
    assert any(k.startswith("relightdecoder.enc_layers.") for k in res.missing_keys)
    assert any(k.startswith("relightdecoder.dec_layers.") for k in res.missing_keys)
    for k, v in hand.state_dict().items():
        assert torch.equal(t.state_dict()[k], v), k
    t = ht.reduce(t.to(inp["pose"].device)).eval()
    with torch.no_grad():
        p = t(**inp, iteration=5000)
    assert bool(torch.isfinite(p["rgb"]).all()) and float(p["alpha"].max()) > 0


def test_single_light_cycle_intensity_broadcast(frame, monkeypatch):
    """SingleLightCycleDecorator's [B,1,1] intensity gives the bits of the same light at intensity ones [B,1,3].  The
    shadow splat adds with atomics, so its last bits vary from call to call: both calls read one shadow volume."""
    from goliath_b200.light_decorator import SingleLightCycleDecorator

    m, _, inp, _, _ = frame
    march, volume = m.relightdecoder.shadow_march, []

    def shadow_once(prims, light_pos):
        if not volume:
            volume.append(march(prims, light_pos))
        return volume[0].clone()

    monkeypatch.setattr(m.relightdecoder, "shadow_march", shadow_once)
    x = {k: v for k, v in inp.items() if k not in ("light_pos", "light_intensity", "background")}
    seen = {}

    def spy(**d):
        seen.update(d)
        return m(**d)

    with torch.no_grad():
        got = SingleLightCycleDecorator(spy, light_rotate_axis=1)(**x, index=[180, 180], iteration=5000)
        assert tuple(seen["light_intensity"].shape) == (2, 1, 1)
        want = m(**x, light_pos=seen["light_pos"], light_intensity=torch.ones(2, 1, 3, device=m.valid_slot.device),
                 iteration=5000)
    assert list(got) == list(want)
    for k, v in got.items():
        if torch.is_tensor(v):
            assert torch.equal(v, want[k]), k


def _envspin():
    spec = importlib.util.spec_from_file_location("make_envspin_golden",
                                                  os.path.join(HERE, "golden", "make_envspin_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_env_frame_at_example_size(cuda):
    """one EnvSpinDecorator frame (512 lights at distance 10 000: 103 chunks of 5) at B = 1, 1024 x 667, full-size
    shadow images: finite, and wherever nothing is rendered the composite of the environment alone"""
    from goliath_b200.envmap import compose_envmap
    from goliath_b200.light_decorator import EnvSpinDecorator

    golden = _envspin()
    c = ht.env_config()
    c.update(image_height=H, image_width=W)
    m = _teacher(c).to(cuda).eval()
    pose = torch.from_numpy(np.load(GOLD)["in_pose"][:1]).to(cuda)
    K, Rt, campos = hf.side_cameras(_posed_points(m, pose), H, W)
    K, Rt, campos = K.float().to(cuda), Rt.float().to(cuda), campos.float().to(cuda)
    seen = {}

    def spy(**d):
        seen.update(d)
        return m(**d)

    dec = EnvSpinDecorator(spy, golden.probe(), **golden.DECORATOR)
    with torch.no_grad():
        p = dec(pose=pose, campos=campos, K=K, Rt=Rt, camera_id=[hf.BATCH_CAMERAS[0]], index=[5])
        assert tuple(seen["light_pos"].shape) == (1, 512, 3)
        rgb, alpha = p["rgb"], p["alpha"]
        assert tuple(rgb.shape) == (1, 3, H, W) and bool(torch.isfinite(rgb).all())
        empty = alpha[:, 0] == 0
        assert 0.05 < float(empty.float().mean()) < 0.95
        bg = compose_envmap(torch.zeros_like(rgb), torch.zeros_like(alpha), seen["envbg"], K, Rt)
    assert torch.equal(rgb.permute(0, 2, 3, 1)[empty], bg.permute(0, 2, 3, 1)[empty])


@pytest.mark.parametrize("training", [False, True])
def test_frame_forward_backward_without_host_sync(frame, training):
    m, _, inp, _, _ = frame
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
    """B = 2 at 1024 x 667 with L = 6 (a chunk of 5 and one of 1), full-size shadow images and the background, the
    example's rgb L2 and negative-colour penalty on texolat: every poseencoder2 / relightdecoder parameter gets a
    finite, nonzero gradient"""
    m = _teacher(hf.config(H, W)).to(cuda).train()
    assert m.relightdecoder.chunksize == 5 and m.relightdecoder.pixel_coords.shape[:2] == (1024, 1024)
    z = np.load(GOLD)
    pose = torch.from_numpy(z["in_pose"]).to(cuda)
    points = _posed_points(m, pose)
    K, Rt, campos = hf.side_cameras(points, H, W)
    light_pos, light_intensity = ht.lights(points, n=6)
    inp = {"pose": pose, "campos": campos.float().to(cuda), "K": K.float().to(cuda), "Rt": Rt.float().to(cuda),
           "light_pos": light_pos.to(cuda), "light_intensity": light_intensity.to(cuda),
           "camera_id": list(hf.BATCH_CAMERAS), "background": hf.background(2, H, W).to(cuda)}
    preds = m(**inp, iteration=5000)
    assert tuple(preds["texolat"].shape) == (2, 1, 8, 3, 1024, 1024)
    g = torch.Generator(device=cuda).manual_seed(5)
    target = 255.0 * torch.rand(preds["rgb"].shape, device=cuda, generator=g)
    loss = 0.0016 * ((preds["rgb"] - target) ** 2).mean() + 1e-2 * preds["texolat"].clamp(max=0.0).pow(2).mean()
    params = {n: p for n, p in m.named_parameters() if n.startswith(("poseencoder2.", "relightdecoder."))}
    grads = torch.autograd.grad(loss, list(params.values()))
    for (n, p), gr in zip(params.items(), grads):
        assert bool(torch.isfinite(gr).all()), n
        assert float(gr.abs().max()) > 0, n
    assert 0.05 < float((preds["alpha"] > 0.5).float().mean()) < 0.95
