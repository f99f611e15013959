"""GPU checks of the head avatar's frame (`goliath_b200.rgca.AutoEncoder`, `head_lights`, csrc/head_frame.cu):

* the light kernel against an fp64 torch restatement (sh.dir2sh's basis) at L in {1, 5, 460, 512} and C in {1, 3},
  with zero-padded lights, a light at the head centre and lightrot given or absent, within 1e-5 sum |terms| per
  coefficient; against the reference's own light statements (tests/golden/head_frame_ref.npz); two calls give the
  same bits; an input that requires grad is refused;
* the frame in its three modes (eval point lights, training with a background, eval environment map), a
  reference-shaped state dict loaded with strict=True and then seeded, against the reference frame's fp64 run
  (tests/golden/make_head_frame_golden.py): output keys, statistics and samples of every output, the render's
  arguments, pre-render and post-render gradients, each within max(1e-4, 4 x) the reference's fp32 error;
* self-consistency: the frame's rgb equals, bit for bit, the stage chain called by hand;
* the rgca_example.yml size (slab 1024, 2048 x 1334, B = 2): training forward + backward, finite gradients;
* SingleLightCycleDecorator and EnvSpinDecorator around the frame."""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import head_frame_restate as hr  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(HERE, "golden", "head_frame_ref.npz")
cuda = torch.device("cuda")


def _light_case(L, C, lightrot, seed):
    g = torch.Generator().manual_seed(seed)
    B = 3
    hp = torch.stack([torch.cat([hr.rotation(torch.randn(3, generator=g, dtype=torch.float64), 0.3 + b),
                                 10.0 * torch.randn(3, 1, generator=g, dtype=torch.float64)], 1) for b in range(B)])
    campos = 1000.0 * torch.randn(B, 3, generator=g, dtype=torch.float64)
    Rt = torch.randn(B, 3, 4, generator=g, dtype=torch.float64)
    d = torch.randn(B, L, 3, generator=g, dtype=torch.float64)
    lpos = 1100.0 * d / d.norm(dim=-1, keepdim=True)
    lint = torch.rand(B, L, C, generator=g, dtype=torch.float64)
    if L > 2:
        lint[1, L // 2:] = 0.0                # zero-padded lights
        lpos[1, L // 2:] = 0.0
    lpos[0, 0] = hp[0, :, 3]                  # a light at the head centre
    rot = torch.stack([hr.rotation(torch.randn(3, generator=g, dtype=torch.float64), 1.0 + b) for b in range(B)])
    f = lambda t: t.float().contiguous()
    return [f(hp), f(campos), f(Rt), f(lpos), f(lint), f(rot) if lightrot else None]


@pytest.mark.parametrize("L", [1, 5, 460, 512])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("lightrot", [False, True])
def test_light_kernel_against_fp64(L, C, lightrot):
    from goliath_b200.rgca import head_lights

    args = _light_case(L, C, lightrot, seed=L * 10 + C)
    got = head_lights(*[None if a is None else a.to(cuda) for a in args])
    want = hr.head_lights64(*args, with_terms=True)
    for k in ("headrel_Rt", "headrel_campos", "headrel_light_pos"):
        w = want[k]
        err = (got[k].cpu().double() - w).abs().max() / max(float(w.abs().max()), 1.0)
        assert err < 1e-6, (k, float(err))
    err = (got["headrel_light_sh"].cpu().double() - want["headrel_light_sh"]).abs()
    bound = 1e-5 * want["terms_abs"] + 1e-30
    assert bool((err <= bound).all()), float((err / bound).max())
    assert torch.isfinite(got["headrel_light_sh"]).all()
    if lightrot:
        assert (got["lightrot"].cpu().double() - want["lightrot"]).abs().max() < 1e-6
    else:
        assert got["lightrot"] is None
    again = head_lights(*[None if a is None else a.to(cuda) for a in args])
    for k in ("headrel_Rt", "headrel_campos", "headrel_light_pos", "headrel_light_sh"):
        assert torch.equal(got[k], again[k]), k


@pytest.mark.parametrize("tag", ["c1", "c3"])
def test_light_kernel_against_reference_statements(tag):
    from goliath_b200.rgca import head_lights

    z = np.load(GOLDEN)
    inp = [torch.from_numpy(z["%s_in_%s" % (tag, k)]).to(cuda)
           for k in ("head_pose", "campos", "Rt", "light_pos", "light_intensity", "lightrot")]
    got = head_lights(*inp)
    want = hr.head_lights64(*[t.cpu() for t in inp], with_terms=True)
    for k in ("headrel_Rt", "headrel_campos", "headrel_light_pos", "lightrot"):
        ref = torch.from_numpy(z["%s_out_%s" % (tag, k)])
        assert (got[k].cpu().double() - ref).abs().max() <= 1e-6 * max(float(ref.abs().max()), 1.0), k
    ref = torch.from_numpy(z["%s_out_headrel_light_sh" % tag])
    err = (got["headrel_light_sh"].cpu().double() - ref).abs()
    assert bool((err <= 1e-5 * want["terms_abs"] + 1e-30).all())


def test_light_kernel_refuses_grad():
    from goliath_b200.rgca import head_lights

    args = [a.to(cuda) for a in _light_case(5, 3, False, 1)[:5]]
    args[3].requires_grad_()
    with pytest.raises(RuntimeError, match="requires grad"):
        head_lights(*args)


def _reference_state_dict():
    """a state dict with the reference's keys and shapes (tests/golden/head_frame_ref.npz), zero-filled"""
    keys = json.loads(np.load(GOLDEN)["keys_json"].tobytes().decode())
    return {k: torch.zeros(s) for k, s in keys.items()}


def _frame(**kw):
    """the frame at hr.config() (+ kw) on the seeded parameters of head_frame_restate.seeded_fill, after a
    reference-shaped state dict was loaded with strict=True"""
    from goliath_b200.rgca import AutoEncoder

    torch.manual_seed(0)
    cfg = {**hr.config(), **kw}
    m = AutoEncoder(**cfg, assets=hr.assets())
    ref = {k: v for k, v in _reference_state_dict().items()       # the reference has no cal / blur keys without them
           if not (k.startswith("cal.") and cfg["cal"] is None) and not (k.startswith("learn_blur.")
                                                                            and not cfg["learn_blur"])}
    ref.update({k: v for k, v in m.state_dict().items() if k not in dict(m.named_parameters())})  # asset buffers
    m.load_state_dict(ref, strict=True)
    hr.seeded_fill(m)
    return m.to(cuda)


def _inputs(**kw):
    return {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in hr.inputs(**kw).items()}


def _envmap_inputs(inp, B=2):
    g = torch.Generator().manual_seed(3)
    inp["preconv_envmap"] = [(2.0 * torch.rand(B, 3, 16 >> i, 32 >> i, generator=g)).to(cuda) for i in range(4)]
    inp["envbg"] = torch.rand(B, 3, 64, 128, generator=g).to(cuda)
    inp["lightrot"] = torch.stack([hr.rotation([0.0, 1.0, 0.0], 0.7 * (b + 1)) for b in range(B)]).float().to(cuda)
    return inp


REF_KEYS = {"geom", "headrel_light_sh", "embs", "embs_mu", "embs_logvar", "color", "opacity", "primpos", "primqvec",
            "primscale", "primscale_preclip", "sigma", "spec_vis", "spec_nml", "spec_dnml", "diff_color", "spec_color",
            "primnmlbase", "rgb", "alpha", "depth", "learn_blur_weights"}


def _check_outputs(preds, B, width, training=False):
    want = REF_KEYS | ({"cos_weight", "color_rand"} if training else set())
    assert want <= set(preds), want - set(preds)
    G = hr.SLAB ** 2
    assert preds["rgb"].shape == (B, 3, hr.H, width)
    assert preds["alpha"].shape == (B, 1, hr.H, hr.W) and preds["depth"].shape == (B, 1, hr.H, hr.W)
    assert preds["primpos"].shape == (B, G, 3) and preds["headrel_light_sh"].shape == (B, 3, 81)
    assert preds["learn_blur_weights"].shape == (B, 3)
    for k in want:
        assert torch.isfinite(preds[k]).all(), k
    assert float(preds["alpha"].max()) > 0.1          # the head is in view


@pytest.mark.parametrize("mode", ["point", "train", "envmap"])
def test_frame_against_reference(mode, monkeypatch):
    """outputs, render arguments, pre-render and post-render gradients against the reference frame's fp64 run, each
    within max(1e-4, 4 x) the reference's own fp32 error"""
    import goliath_b200.gsplat.olat as olat
    import goliath_b200.render as render

    z = np.load(GOLDEN)
    m = _frame(**{k: v for k, v in hr.mode_config(mode).items() if k in ("encoder", "cal")})
    m.train(mode == "train")
    inp = {k: (v.to(cuda) if torch.is_tensor(v) else [x.to(cuda) for x in v] if isinstance(v, list) and
               torch.is_tensor(v[0]) else v) for k, v in hr.mode_inputs(mode).items()}
    seen = {}

    def spy(fn, name):
        def wrapped(*a, **kw):
            out = fn(*a, **kw)
            seen[name] = (a, kw, out[0])
            return out
        return wrapped

    monkeypatch.setattr(render, "render_views", spy(render.render_views, "views"))
    monkeypatch.setattr(olat, "render_views_shared", spy(olat.render_views_shared, "shared"))
    preds = m(**inp)

    keys = set(json.loads(z["%s_out_keys_json" % mode].tobytes().decode()))
    assert keys == set(preds), keys ^ set(preds)
    bad = []

    def check(kind, k, t):
        ref = z["%s_%s_%s" % (mode, kind, k)]
        assert tuple(t.shape) == tuple(z["%s_shape_%s_%s" % (mode, kind, k)]), (kind, k, tuple(t.shape))
        assert torch.isfinite(t).all(), (kind, k)
        err, bound = hr.nrel_summary(hr.summarise(t), ref), max(1e-4, 4 * float(z["%s_err32_%s_%s" % (mode, kind, k)]))
        if err > bound:
            bad.append((kind, k, err, bound))

    for k in sorted(keys):
        if k in hr.RANDOM_KEYS:
            assert torch.isfinite(preds[k]).all() and preds[k].shape[:2] == preds["primpos"].shape[:2], k
        else:
            check("out", k, preds[k])

    # the render's arguments: the intrinsics and the head-relative Rt of each view (one call per view and colour set)
    a, kw, rendered = seen["shared" if mode == "envmap" else "views"]
    intr = np.array(kw["intrinsics_host"] if mode != "envmap" else a[5], dtype=np.float64)
    Rt = (a[3] if mode != "envmap" else a[2]).detach().cpu().numpy()
    reps = 3 if mode == "envmap" else 1
    want_i, want_R = z["%s_args_intrinsics" % mode], z["%s_args_Rt" % mode]
    order = [v * reps + c for c in range(reps) for v in range(2)] if reps > 1 else list(range(2))
    np.testing.assert_array_equal(np.repeat(intr, reps, 0)[order] if reps > 1 else intr, want_i)
    np.testing.assert_allclose(np.repeat(Rt, reps, 0)[order] if reps > 1 else Rt, want_R, rtol=0, atol=1e-4)

    # pre-render: a seeded linear functional of the per-Gaussian outputs
    params = dict(m.named_parameters())
    names = json.loads(z["%s_grad_names_json" % mode].tobytes().decode())
    w = hr.functional_weights(preds)
    f = sum((preds[k] * w[k].float().to(cuda)).sum() for k in hr.PRIM_KEYS)
    grads = torch.autograd.grad(f, [params[n] for n in names], retain_graph=True, allow_unused=True)
    for n, g in zip(names, grads):
        check("pre", n, g if g is not None else torch.zeros_like(params[n]))

    # post-render: a seeded cotangent on rgb, against the rendered images (the reference renders one colour set per
    # call: [colour set, view] in call order), the calibration rows and the blur logits
    extra = [k for k in ("cal.holder.params", "learn_blur.weights_raw") if k in params]
    cot = hr.rgb_cotangent(preds["rgb"].shape).float().to(cuda)
    gr = torch.autograd.grad((preds["rgb"] * cot).sum(), [rendered] + [params[k] for k in extra])
    g_img = gr[0].transpose(0, 1).reshape(-1, *gr[0].shape[2:]) if mode == "envmap" else gr[0]
    check("post", "renders", g_img)
    for k, g in zip(extra, gr[1:]):
        check("post", k, g)
    assert not bad, bad


def test_frame_point_lights_eval_matches_stage_chain():
    from goliath_b200.photo_loss import post_render
    from goliath_b200.rgca import head_lights
    from goliath_b200.render import render_views

    m = _frame().eval()
    inp = _inputs()
    with torch.no_grad():
        preds = m(**inp)
    _check_outputs(preds, 2, hr.W)
    lights = head_lights(inp["head_pose"], inp["campos"], inp["Rt"], inp["light_pos"], inp["light_intensity"])
    assert torch.equal(preds["headrel_light_sh"], lights["headrel_light_sh"])
    with torch.no_grad():
        rgb, alpha, depth = render_views(hr.W, hr.H, inp["K"], lights["headrel_Rt"], preds)
        w, b, grey = m.cal.rows(m.cal.name_to_idx(inp["camera_id"]))
        want = post_render(rgb, None, None, w, b, grey, m.learn_blur.weights(inp["camera_id"]))
    assert torch.equal(preds["rgb"], want)
    assert torch.equal(preds["alpha"], alpha) and torch.equal(preds["depth"], depth)
    assert torch.equal(preds["learn_blur_weights"], m.learn_blur.weights_raw[[2, 0]])


def test_frame_training_with_background_matches_stage_chain():
    from goliath_b200.photo_loss import post_render
    from goliath_b200.rgca import head_lights
    from goliath_b200.render import render_views

    m = _frame(encoder={**hr.config()["encoder"], "noise_std": 0.0}).train()
    inp = _inputs()
    inp["background"] = torch.rand(2, 3, hr.H, hr.W, generator=torch.Generator().manual_seed(9)).to(cuda)
    inp["is_fully_lit_frame"] = torch.tensor([True, False], device=cuda)
    preds = m(**inp)
    _check_outputs(preds, 2, hr.W, training=True)
    g = torch.randn(preds["rgb"].shape, generator=torch.Generator().manual_seed(4)).to(cuda)
    (preds["rgb"] * g).sum().backward()
    for n, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    lights = head_lights(inp["head_pose"], inp["campos"], inp["Rt"], inp["light_pos"], inp["light_intensity"])
    with torch.no_grad():
        rgb, alpha, _ = render_views(hr.W, hr.H, inp["K"], lights["headrel_Rt"], preds)
        w, b, grey = m.cal.rows(m.cal.name_to_idx(inp["camera_id"]))
        bg = inp["background"].clone()
        bg[1] = 0.0
        want = post_render(rgb, alpha, bg, w, b, grey, m.learn_blur.weights(inp["camera_id"]))
    assert torch.equal(preds["rgb"].detach(), want)


def test_frame_envmap_matches_stage_chain():
    from goliath_b200.envmap import compose_envmap
    from goliath_b200.gsplat.olat import render_views_shared
    from goliath_b200.photo_loss import post_render
    from goliath_b200.rgca import head_lights

    m = _frame(cal=None).eval()
    inp = _envmap_inputs(_inputs(n_lights=512, n_active=(512,), C=3))
    with torch.no_grad():
        preds = m(**inp)
    _check_outputs(preds, 2, 3 * hr.W)
    assert torch.equal(preds["color"], preds["spec_color"].clamp(min=0.0))
    lights = head_lights(inp["head_pose"], inp["campos"], inp["Rt"], inp["light_pos"], inp["light_intensity"],
                         inp["lightrot"])
    with torch.no_grad():
        full = (preds["diff_color"].clamp(min=0.0) + preds["spec_color"]).clamp(min=0.0)
        colors = torch.stack([full, preds["diff_color"].clamp(min=0.0), preds["spec_color"].clamp(min=0.0)], 1)
        geo = {k: preds[k] for k in ("primpos", "primqvec", "primscale", "opacity")}
        intr = m.intrinsics(inp["K"])
        rgbs, alpha, _ = render_views_shared(hr.W, hr.H, lights["headrel_Rt"], geo, colors, intr)
        img = compose_envmap(rgbs[:, 0], alpha, inp["envbg"], inp["K"], inp["Rt"])
        want = post_render(torch.cat([img, rgbs[:, 1], rgbs[:, 2]], -1),
                           blur_weights=m.learn_blur.weights(inp["camera_id"]))
    assert torch.equal(preds["rgb"], want)


def test_cal_without_camera_id_raises():
    m = _frame().eval()
    inp = _inputs()
    inp.pop("camera_id")
    with pytest.raises(ValueError, match="camera_id"):
        with torch.no_grad():
            m(**inp)


def test_flags_off_give_the_plain_render():
    from goliath_b200.rgca import head_lights
    from goliath_b200.render import render_views

    m = _frame().eval()
    m.cal_enabled = m.learn_blur_enabled = False
    inp = _inputs()
    inp.pop("camera_id")
    with torch.no_grad():
        preds = m(**inp)
        lights = head_lights(inp["head_pose"], inp["campos"], inp["Rt"], inp["light_pos"], inp["light_intensity"])
        rgb, _, _ = render_views(hr.W, hr.H, inp["K"], lights["headrel_Rt"], preds)
    assert torch.equal(preds["rgb"], rgb) and "learn_blur_weights" not in preds


def test_config_size_training_forward_backward():
    from goliath_b200.rgca import AutoEncoder

    torch.manual_seed(0)
    m = AutoEncoder(**hr.config(h=2048, w=1334, slab=1024), assets=hr.assets(slab=1024)).to(cuda).train()
    inp = _inputs(h=2048, w=1334, slab=1024)
    inp["background"] = torch.rand(2, 3, 2048, 1334, device=cuda)
    inp["is_fully_lit_frame"] = torch.tensor([True, False], device=cuda)
    preds = m(**inp)
    assert preds["rgb"].shape == (2, 3, 2048, 1334) and preds["primpos"].shape == (2, 1024 ** 2, 3)
    (preds["rgb"] * torch.randn_like(preds["rgb"])).sum().backward()
    for n, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n


def test_single_light_cycle_decorator_wraps_frame():
    from goliath_b200.light_decorator import SingleLightCycleDecorator

    m = _frame(cal=None, learn_blur=False).eval()
    inp = _inputs()
    inp["index"] = [3, 40]
    with torch.no_grad():
        preds = SingleLightCycleDecorator(m, cycle=256, light_rotate_axis=0)(**inp)
    assert preds["rgb"].shape == (2, 3, hr.H, hr.W) and torch.isfinite(preds["rgb"]).all()


def test_envspin_decorator_wraps_frame():
    from goliath_b200.light_decorator import EnvSpinDecorator

    m = _frame(cal=None).eval()
    m.learn_blur_enabled = False
    inp = _inputs()
    inp["index"] = [0, 64]
    probe = np.random.default_rng(2).uniform(0.0, 4.0, (64, 128, 3)).astype(np.float32)
    with torch.no_grad():
        preds = EnvSpinDecorator(m, probe).to(cuda)(**inp)
    assert preds["rgb"].shape == (2, 3, hr.H, 3 * hr.W) and torch.isfinite(preds["rgb"]).all()
