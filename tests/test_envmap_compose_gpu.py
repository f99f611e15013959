"""Environment-map relighting frame (goliath_b200.envmap, render.render_views_envmap; csrc/envmap_compose.cu):

1. rotate_envmap_mat and compose_envmap against the reference's own functions (tests/golden/envmap_compose_ref.npz,
   made by tests/golden/make_envmap_golden.py): every element, NaNs where the reference has them, the mirror mask
   exactly (through the backward);
2. a torch restatement of compose_envmap, pinned to the same golden, as the oracle at 1024x667 and 2048x1334;
3. render_views_envmap against the CPU splat oracle (three colour sets on one projection and binning) + the pinned
   compose, forward and backward, eager and with a capacity; captured in a CUDA graph; at the benchmarked scene size;
4. the argument checks (host side, no GPU needed)."""
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fullstep import oracle_shared_view
from util import assert_close, small_scene, t2n

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_envmap_golden", os.path.join(HERE, "golden", "make_envmap_golden.py"))
golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(golden)

BAR = dict(rtol=1e-4, atol=2e-5, equal_nan=True)  # every element, no exemption fraction
PIX = dict(rtol=1e-4, atol=2e-5, frac=0.9995)      # the OLAT tests' pixel bar (splat blend vs the oracle)
gpu = pytest.mark.gpu


def _gtol(want):
    return dict(rtol=1e-4, atol=1e-5 * float(np.abs(want).max()), frac=0.999)


_Z = {}


def _golden(case):
    if not _Z:
        _Z["z"] = np.load(os.path.join(HERE, "golden", "envmap_compose_ref.npz"))
    z = _Z["z"]
    x = golden.case_inputs(case)
    out, rot = golden.golden_case(z, case)
    x.update(out=out, rot=rot, mask=z["mask"])
    return x


def torch_compose(render, alpha, envbg, K, Rt):
    """compose_envmap (ca_code/utils/envmap.py:325-345) restated in torch on any device: bicubic grid_sample, the
    dense 101x101 conv2d blur in fp32 (TF32 off), the mirror ball on torch.linspace's grid."""
    B, _, H, W = render.shape
    f32 = dict(device=render.device, dtype=torch.float32)
    R = Rt[:, :3, :3]

    def sample(d):
        u = (1 / np.pi) * torch.atan2(d[..., 0], d[..., 2])
        v = 2 * ((1 / np.pi) * torch.acos(d[..., 1])) - 1.0
        return F.grid_sample(envbg, torch.stack([u, v], -1), mode="bicubic", padding_mode="border", align_corners=True)

    lin = torch.linspace(-1.0, 1.0, 200, **f32)
    py, px = torch.meshgrid(lin, lin, indexing="ij")
    pc = torch.stack([px, py], -1)[None].expand(B, -1, -1, -1)
    zsq = pc.pow(2).sum(-1, keepdim=True)
    mask = (zsq < 1.0).float()[:, None, :, :, 0]
    nz = -(1.0 - zsq).clamp(min=0.0).sqrt()
    ref = -2.0 * nz * torch.cat([pc, nz], -1)
    ref = torch.cat([ref[..., :2], 1.0 + ref[..., 2:]], -1)
    ball = sample(torch.einsum("bxy,bhwx->bhwy", R, ref))

    y, x = torch.meshgrid(torch.arange(H, device=render.device), torch.arange(W, device=render.device), indexing="ij")
    d = torch.stack([x, y], -1)[None] - K[:, None, None, :2, 2]
    d = d / (torch.stack([K[:, 0, 0], K[:, 1, 1]], -1)[:, None, None] * 0.2)
    d = torch.cat([d, torch.ones_like(d[..., :1])], -1)
    bg = sample(F.normalize(torch.einsum("bxy,bhwx->bhwy", R, d), dim=-1))
    k = torch.exp(-torch.linspace(-4.0, 4.0, 101, **f32) ** 2)
    k2 = k[:, None] * k[None, :]
    k2 = (k2 / k2.sum())[None, None].repeat(3, 1, 1, 1)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        bg = F.conv2d(bg, k2, padding=50, groups=3)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    out = render + (1.0 - alpha) * bg.clamp(0, 1.0)
    m = torch.zeros_like(alpha)
    m[:, :, -200:, -200:] = mask
    mi = torch.zeros_like(render)
    mi[:, :, -200:, -200:] = ball
    return (1.0 - m) * out + m * mi


def _dev(x, cuda):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda) if isinstance(v, np.ndarray) else v
            for k, v in x.items()}


# ------------------------------------------------------------------------------------------- 1. against the reference
@gpu
@pytest.mark.parametrize("case", golden.CASES)
def test_rotate_matches_reference(cuda, case):
    from goliath_b200.envmap import rotate_envmap_mat

    x = _golden(case)
    t = _dev(x, cuda)
    got = rotate_envmap_mat(t["envbg"], t["Rt"][:, :3, :3])
    np.testing.assert_allclose(t2n(got), x["rot"], **BAR, err_msg=case)
    one = rotate_envmap_mat(t["envbg"][1], t["Rt"][1, :3, :3])  # the reference's unbatched signature
    assert one.shape == t["envbg"].shape[1:] and torch.equal(one, got[1])


@gpu
@pytest.mark.parametrize("case", golden.CASES)
def test_compose_matches_reference(cuda, case):
    from goliath_b200.envmap import compose_envmap

    x = _golden(case)
    t = _dev(x, cuda)
    render = t["render"].clone().requires_grad_()
    out = compose_envmap(render, t["alpha"], t["envbg"], t["K"], t["Rt"])
    np.testing.assert_allclose(t2n(out), x["out"], **BAR, err_msg=case)
    if case == "b200x200":
        assert np.isnan(x["out"]).sum() > 1000, "the scaled camera must drive acos past its domain in the mirror ball"
    else:
        assert not np.isnan(x["out"]).any()
    # the backward is (1 - mirror mask) * g: with g = 1 it reads the mask back, which must match the reference's exactly
    out.backward(torch.ones_like(out))
    H, W = out.shape[2:]
    want = np.ones((H, W), np.float32)
    want[-200:, -200:] = 1.0 - x["mask"]
    for b in range(2):
        for c in range(3):
            assert np.array_equal(t2n(render.grad[b, c]), want), (case, b, c)


@gpu
@pytest.mark.parametrize("case", golden.CASES)
def test_torch_formulation_matches_reference(cuda, case):
    """the oracle of the at-size test is pinned to the reference first"""
    x = _golden(case)
    t = _dev(x, cuda)
    got = torch_compose(t["render"], t["alpha"], t["envbg"], t["K"], t["Rt"])
    np.testing.assert_allclose(t2n(got), x["out"], **BAR, err_msg=case)


# -------------------------------------------------------------------------------------------------------- 2. at size
@gpu
@pytest.mark.parametrize("hw", [(1024, 667), (2048, 1334)])
def test_compose_at_size(cuda, hw):
    from goliath_b200.envmap import compose_envmap

    H, W = hw
    rng = np.random.default_rng(H)
    render = golden._smooth(rng, (2, 3, H, W), 0.0, 1.0)
    alpha = np.clip(golden._smooth(rng, (2, 1, H, W), -0.3, 1.3), 0.0, 1.0)
    envbg = golden._smooth(rng, (2, 3, 128, 256), 0.0, 2.5)
    f = 3300.0 * W / 1334.0
    cams = [golden._camera(golden._random_rot(rng), f, f, W / 2.0, H / 2.0),
            golden._camera(golden._rot("y", 150), 1.1 * f, f, 0.4 * W, 0.6 * H)]
    t = _dev(dict(render=render, alpha=alpha, envbg=envbg, K=np.stack([c[0] for c in cams]),
                  Rt=np.stack([c[1] for c in cams])), cuda)
    got = compose_envmap(t["render"], t["alpha"], t["envbg"], t["K"], t["Rt"])
    want = torch_compose(t["render"], t["alpha"], t["envbg"], t["K"], t["Rt"])
    assert not torch.isnan(want).any()
    np.testing.assert_allclose(t2n(got), t2n(want), **BAR, err_msg=str(hw))


# -------------------------------------------------------------------------------------------- 3. the frame-level render
def _frame_inputs(H, W, G=3000, seed=5):
    s = small_scene(G=G, img_h=H, img_w=W, seed=seed)
    rng = np.random.default_rng(seed)
    from goliath_b200 import synthetic

    cams = [synthetic.ring_camera(k, img_h=H, img_w=W) for k in (1, 6)]
    for c in cams:
        c.update(fx=s["fx"], fy=s["fy"])
    head = golden._rot("y", 20) @ golden._rot("x", -10)  # the world camera differs from the head-relative one
    world = [np.concatenate([c["viewmat"].numpy()[:, :3].astype(np.float64) @ head, c["viewmat"].numpy()[:, 3:]], 1)
             for c in cams]
    G = s["means3d"].shape[0]
    return dict(
        s=s, cams=cams, scales=(s["scales"] * np.float32(6.0)).astype(np.float32),
        color=rng.random((2, G, 3)).astype(np.float32),
        diff=(0.4 + 0.3 * rng.standard_normal((2, G, 3))).astype(np.float32),
        spec=(0.1 + 0.2 * rng.standard_normal((2, G, 3))).astype(np.float32),
        K=np.stack([np.array([[c["fx"], 0, c["cx"]], [0, c["fy"], c["cy"]], [0, 0, 1]], np.float32) for c in cams]),
        headrel=np.stack([c["viewmat"].numpy() for c in cams]), world=np.stack(world).astype(np.float32),
        envbg=golden._smooth(rng, (2, 3, 32, 64), 0.0, 2.5),
        w=rng.standard_normal((2, 3, H, 3 * W)).astype(np.float32),
        w_d=(1e-3 * rng.standard_normal((2, 1, H, W))).astype(np.float32))


def _frame_tensors(x, cuda, grad):
    s = x["s"]
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rep = lambda a: d(np.repeat(a[None], 2, 0))
    preds = dict(primpos=rep(s["means3d"]), primscale=rep(x["scales"]), primqvec=rep(s["quats"]), opacity=rep(s["opacity"]),
                 color=d(x["color"]), diff_color=d(x["diff"]), spec_color=d(x["spec"]))
    if grad:
        for v in preds.values():
            v.requires_grad_()
    intr = [(c["fx"], c["fy"], c["cx"], c["cy"]) for c in x["cams"]]
    return dict(width=s["img_w"], height=s["img_h"], K=d(x["K"]), headrel_Rt=d(x["headrel"]), Rt=d(x["world"]),
                preds=preds, envbg=d(x["envbg"]), intrinsics_host=intr)


def _run_frame(x, cuda, capacity):
    from goliath_b200.render import render_views_envmap

    a = _frame_tensors(x, cuda, True)
    preds = a["preds"]
    before = dict(preds)
    rgb, alpha, depth = render_views_envmap(capacity=capacity, **a)
    assert set(preds) == set(before) and all(preds[k] is before[k] for k in preds), "preds must not be modified"
    d = lambda v: torch.from_numpy(v).to(cuda)
    ((rgb * d(x["w"])).sum() + (depth * d(x["w_d"])).sum()).backward()
    torch.cuda.synchronize()
    return preds, rgb, alpha, depth


def _frame_oracle(orc, x, cuda, mask):
    """per view: oracle_shared_view with C = 3 (v_rgb[0] = w * (1 - mirror mask)) + the pinned compose"""
    s = x["s"]
    H, W = s["img_h"], s["img_w"]
    inv_a = lambda a: (1.0 / np.clip(a, 0.05, 1.0)).astype(np.float32)
    m = np.zeros((H, W), np.float32)
    m[-200:, -200:] = mask
    refs = []
    for v in range(2):
        c = x["cams"][v]
        cols = np.stack([x["color"][v], np.maximum(x["diff"][v], 0), np.maximum(x["spec"][v], 0)])
        w = x["w"][v]
        v_rgb = np.stack([w[..., :W] * (1.0 - m), w[..., W:2 * W], w[..., 2 * W:]]).transpose(0, 2, 3, 1)
        ref = oracle_shared_view(orc, s["means3d"], x["scales"], s["quats"], s["opacity"], cols, np.zeros(3, np.float32),
                                 x["headrel"][v], (c["fx"], c["fy"], c["cx"], c["cy"]), H, W, np.ascontiguousarray(v_rgb),
                                 v_depth=lambda a, v=v: x["w_d"][v, 0] * inv_a(a))
        ref["depth"] = ref["depth_raw"] * inv_a(ref["alpha"])
        refs.append(ref)
    dd = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    full = torch_compose(dd(np.stack([r["rgb"][0].transpose(2, 0, 1) for r in refs])),
                         dd(np.stack([r["alpha"][None] for r in refs])), dd(x["envbg"]), dd(x["K"]), dd(x["world"]))
    return refs, t2n(full)


_FRAME = {}


@gpu
@pytest.mark.parametrize("hw", [(216, 240), (203, 231)])
@pytest.mark.parametrize("capacity", [None, 1 << 17])
def test_render_views_envmap_matches_oracle(orc, cuda, hw, capacity):
    from goliath_b200.gsplat.fused import check_overflow

    H, W = hw
    if hw not in _FRAME:
        x = _frame_inputs(H, W)
        _FRAME[hw] = x, _frame_oracle(orc, x, cuda, _golden("a216x240")["mask"])
    x, (refs, full) = _FRAME[hw]
    preds, rgb, alpha, depth = _run_frame(x, cuda, capacity)
    assert not check_overflow(cuda) and not alpha.requires_grad
    assert rgb.shape == (2, 3, H, 3 * W) and alpha.shape == (2, 1, H, W) and depth.shape == (2, 1, H, W)
    rgb, alpha, depth = t2n(rgb), t2n(alpha), t2n(depth)
    for v, ref in enumerate(refs):
        what = "%s cap=%s view %d" % (hw, capacity, v)
        assert (ref["alpha"] > 0.1).mean() > 0.05 and (ref["alpha"] < 0.9).mean() > 0.05, "scene must cover part of it"
        assert_close(rgb[v, :, :, :W], full[v], what=what + " full", **PIX)
        assert_close(rgb[v, :, :, W:2 * W], ref["rgb"][1].transpose(2, 0, 1), what=what + " diffuse", **PIX)
        assert_close(rgb[v, :, :, 2 * W:], ref["rgb"][2].transpose(2, 0, 1), what=what + " specular", **PIX)
        assert_close(alpha[v, 0], ref["alpha"], rtol=1e-4, atol=2e-6, frac=0.9995, what=what + " alpha")
        assert_close(depth[v, 0], ref["depth"], rtol=1e-4, atol=2e-2, frac=0.9995, what=what + " depth")
        g = ref["grads"]
        got = dict(means3d=preds["primpos"].grad[v], scales=preds["primscale"].grad[v], quats=preds["primqvec"].grad[v],
                   opacity=preds["opacity"].grad[v])
        for k, gt in got.items():
            assert_close(t2n(gt).reshape(g[k].shape), g[k], what="%s grad %s" % (what, k), **_gtol(g[k]))
        # colour gradients; clamp(min=0) passes the gradient where the colour is >= 0
        want = dict(color=g["colors"][0], diff_color=g["colors"][1] * (x["diff"][v] >= 0),
                    spec_color=g["colors"][2] * (x["spec"][v] >= 0))
        for k, wv in want.items():
            assert_close(t2n(preds[k].grad[v]), wv, what="%s grad %s" % (what, k), **_gtol(wv))


@gpu
def test_render_views_envmap_graph_capture(cuda):
    from goliath_b200.graph import Graphed
    from goliath_b200.gsplat.fused import check_overflow
    from goliath_b200.render import render_views_envmap

    a = _frame_tensors(_frame_inputs(216, 240), cuda, False)
    with torch.no_grad():
        eager = [t.clone() for t in render_views_envmap(capacity=1 << 17, **a)]
        g = Graphed(lambda: render_views_envmap(capacity=1 << 17, **a))
        got = g()
        torch.cuda.synchronize()
    assert not check_overflow(cuda)
    for x, y in zip(got, eager):
        assert torch.equal(x, y)


@gpu
def test_render_views_envmap_bench_size(orc, cuda):
    """300 000 Gaussians at 1024x667 (bench.py's scene and image size), two ring cameras, forward"""
    from goliath_b200 import synthetic
    from goliath_b200.gsplat.fused import check_overflow
    from goliath_b200.render import render_views_envmap

    H, W, G = 1024, 667, 300_000
    sc = {k: v.numpy() for k, v in synthetic.head_gaussians(G).items()}
    cams = [synthetic.ring_camera(k, img_h=H, img_w=W) for k in (0, 5)]
    rng = np.random.default_rng(3)
    cols = np.stack([sc["colors"], rng.standard_normal((G, 3)).astype(np.float32),
                     (0.2 * rng.standard_normal((G, 3))).astype(np.float32)])
    K = np.stack([np.array([[c["fx"], 0, c["cx"]], [0, c["fy"], c["cy"]], [0, 0, 1]], np.float32) for c in cams])
    Rt = np.stack([c["viewmat"].numpy() for c in cams])
    envbg = golden._smooth(rng, (2, 3, 64, 128), 0.0, 2.5)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rep = lambda a: d(np.repeat(a[None], 2, 0))
    preds = dict(primpos=rep(sc["means3d"]), primscale=rep(sc["scales"]), primqvec=rep(sc["quats"]),
                 opacity=rep(sc["opacity"]), color=rep(cols[0]), diff_color=rep(cols[1]), spec_color=rep(cols[2]))
    intr = [(c["fx"], c["fy"], c["cx"], c["cy"]) for c in cams]
    with torch.no_grad():
        rgb, alpha, depth = render_views_envmap(W, H, d(K), d(Rt), d(Rt), preds, d(envbg), intrinsics_host=intr,
                                                capacity=8 * G)
    torch.cuda.synchronize()
    assert not check_overflow(cuda)
    rgb, alpha, depth = t2n(rgb), t2n(alpha), t2n(depth)
    ccols = np.stack([cols[0], np.maximum(cols[1], 0), np.maximum(cols[2], 0)])
    refs = []
    for v, c in enumerate(cams):
        ref = oracle_shared_view(orc, sc["means3d"], sc["scales"], sc["quats"], sc["opacity"], ccols, np.zeros(3, np.float32),
                                 Rt[v], intr[v], H, W, np.zeros((3, H, W, 3), np.float32))
        assert ref["n_isect"] > 2 * G, "the scene must be the dense bench scene"
        refs.append(ref)
    full = t2n(torch_compose(d(np.stack([r["rgb"][0].transpose(2, 0, 1) for r in refs])),
                             d(np.stack([r["alpha"][None] for r in refs])), d(envbg), d(K), d(Rt)))
    for v, ref in enumerate(refs):
        assert_close(rgb[v, :, :, :W], full[v], what="view %d full" % v, **PIX)
        for c in (1, 2):
            assert_close(rgb[v, :, :, c * W:(c + 1) * W], ref["rgb"][c].transpose(2, 0, 1), what="view %d rgb[%d]" % (v, c),
                         **PIX)
        assert_close(alpha[v, 0], ref["alpha"], rtol=1e-4, atol=2e-6, frac=0.9995, what="view %d alpha" % v)
        a = np.clip(ref["alpha"], 0.05, 1.0)
        assert_close(depth[v, 0], ref["depth_raw"] / a, rtol=1e-4, atol=2e-2, frac=0.9995, what="view %d depth" % v)


# ----------------------------------------------------------------------------------------------------- 4. the checks
def _args(dev="cpu", B=2, H=216, W=240, Be=None, dtype=torch.float32):
    z = lambda *s: torch.zeros(*s, dtype=dtype, device=dev)
    return (z(B, 3, H, W), z(B, 1, H, W), z(Be or B, 3, 8, 16), z(B, 3, 3), z(B, 3, 4))


def test_compose_rejects_bad_arguments():
    from goliath_b200.envmap import compose_envmap, rotate_envmap_mat

    for kw, msg in ((dict(H=199), "at least 200x200"), (dict(W=150), "at least 200x200"), (dict(Be=3), "envbg"),
                    (dict(), "CUDA tensor")):
        with pytest.raises(RuntimeError, match=msg):
            compose_envmap(*_args(**kw))
    r, a, e, K, Rt = _args()
    with pytest.raises(RuntimeError, match="alpha"):
        compose_envmap(r, a[:1], e, K, Rt)
    with pytest.raises(RuntimeError, match="K must be"):
        compose_envmap(r, a, e, K[:1], Rt)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        rotate_envmap_mat(e[0], K[0])


@gpu
def test_compose_rejects_bad_arguments_on_gpu(cuda):
    from goliath_b200.envmap import compose_envmap

    with pytest.raises(RuntimeError, match="dtype"):
        compose_envmap(*_args(cuda, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="at least 200x200"):
        compose_envmap(*_args(cuda, H=150))
    with pytest.raises(RuntimeError, match="envbg"):
        compose_envmap(*_args(cuda, Be=1))
