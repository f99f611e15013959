"""GPU checks of the body render (DESIGN.md R9'': csrc/mesh_raster.cu, goliath_b200/mesh_render.py): the index image
bit-exact against the C oracle on the raster edge cases and at the configuration's size, the forward outputs and both
gradients against the fp64 oracle, the whole layer against the reference's fixture (tests/golden/mesh_render_ref.npz),
two drtk-independent anchors for the edge term (the area derivative of a flat triangle, and a finite difference of a
supersampled render), bitwise-repeatable gradients, and a sync-free forward and backward with a graph replay."""
import math
import os

import numpy as np
import pytest
import torch

import mesh_render_restate as mr

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mesh_render_ref.npz")


@pytest.fixture(scope="module")
def morc():
    from oracle import mesh

    mesh.lib()
    return mesh


def _nrel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _run(m, tex, cuda, g=None, edge_grad=True):
    """our render of the pixel-space mesh m through the autograd node -> (outputs, g_v_pix, g_tex)"""
    from goliath_b200.mesh_render import RenderLayer, _MeshRender

    layer = RenderLayer(m["H"], m["W"], m["vi"], m["vt"], m["vti"]).to(cuda)
    v = m["v_pix"].to(cuda).requires_grad_()
    t = torch.as_tensor(tex).to(cuda).requires_grad_()
    out = dict(zip(("render", "depth_img", "bary_img", "vt_img", "index_img", "mask"),
                   _MeshRender.apply(v, t, layer, edge_grad)))
    if g is None:
        return out, None, None
    gv, gt = torch.autograd.grad((out["render"] * torch.as_tensor(g).to(cuda)).sum(), [v, t])
    return out, gv, gt


@pytest.mark.parametrize("name", sorted(mr.cases()))
def test_index_bit_exact_on_edge_cases(cuda, morc, name):
    m = mr.cases()[name]
    out, _, _ = _run(m, np.zeros((m["v_pix"].shape[0], 1, 4, 4), np.float32), cuda)
    ref = morc.mesh_raster(m["v_pix"].numpy(), m["vi"].numpy(), m["H"], m["W"])
    assert np.array_equal(out["index_img"].cpu().numpy(), ref)


def test_index_bit_exact_at_configuration_size(cuda, morc):
    from goliath_b200 import synthetic
    from goliath_b200.mesh_render import transform

    s = synthetic.body_mesh(100_000)
    v_pix = transform(s["verts"][None].expand(4, -1, -1), s["K"], s["Rt"]).contiguous()
    m = dict(v_pix=v_pix, vi=s["vi"], vti=s["vti"], vt=s["vt"], H=2048, W=1334)
    out, _, _ = _run(m, np.zeros((4, 1, 4, 4), np.float32), cuda)
    ref = morc.mesh_raster(v_pix.numpy(), s["vi"].numpy(), 2048, 1334)
    got = out["index_img"].cpu().numpy()
    assert (ref >= 0).mean() > 0.05
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("C,Ht,Wt", [(1, 17, 29), (4, 64, 48)])
@pytest.mark.parametrize("name", ["random", "uv_out", "huge", "on_edges"])
def test_forward_vs_oracle(cuda, morc, C, Ht, Wt, name):
    m = mr.random_mesh() if name == "random" else mr.cases()[name]
    B = m["v_pix"].shape[0]
    tex = np.random.default_rng(C).uniform(-1, 1, size=(B, C, Ht, Wt)).astype(np.float32)
    out, _, _ = _run(m, tex, cuda)
    idx = out["index_img"].cpu().numpy()
    ref = morc.mesh_render_fwd(m["v_pix"].numpy(), m["vi"].numpy(), m["vti"].numpy(), m["vt"].numpy(), tex, idx)
    assert out["render"].shape == (B, C, m["H"], m["W"]) and out["bary_img"].shape == (B, 3, m["H"], m["W"])
    for k, v in ref.items():
        got = out[k].detach().cpu().numpy().astype(np.float64)
        assert np.abs(got - v).max() <= 1e-4 * max(1.0, np.abs(v).max()), (k, np.abs(got - v).max())
    assert out["index_img"].dtype == torch.int32 and all(out[k].dtype == torch.float32 for k in ref)


def _grads_vs_oracle(cuda, morc, m, C, edge_grad):
    B = m["v_pix"].shape[0]
    rng = np.random.default_rng(11)
    tex = rng.uniform(-1, 1, size=(B, C, 24, 20)).astype(np.float32)
    g = rng.standard_normal((B, C, m["H"], m["W"])).astype(np.float32)
    out, gv, gt = _run(m, tex, cuda, g, edge_grad)
    idx = out["index_img"].cpu().numpy()
    rv, rt = morc.mesh_render_bwd(m["v_pix"].numpy(), m["vi"].numpy(), m["vti"].numpy(), m["vt"].numpy(), tex, idx, g,
                                 edge_grad=edge_grad)
    return (gv.cpu(), gt.cpu()), (rv, rt), (tex, g, idx)


@pytest.mark.parametrize("C", [1, 4])
def test_interior_gradients_vs_fp64_oracle(cuda, morc, C):
    m = mr.random_mesh()
    (gv, gt), (rv, rt), (tex, g, idx) = _grads_vs_oracle(cuda, morc, m, C, edge_grad=False)
    # the fp32 error of the same restatement (torch autograd at the same index image)
    res = {}
    for dt in (torch.float32, torch.float64):
        v = m["v_pix"].to(cuda, dt).requires_grad_()
        t = torch.from_numpy(tex).to(cuda, dt).requires_grad_()
        r = mr.render_at(v, m["vi"].to(cuda), m["vti"].to(cuda), m["vt"].to(cuda, dt), t,
                         torch.from_numpy(idx).to(cuda))["render"]
        res[dt] = torch.autograd.grad((r * torch.from_numpy(g).to(cuda, dt)).sum(), [v, t])
    for ours, ref, k in ((gv, rv, 0), (gt, rt, 1)):
        bound = max(1e-4, 4 * _nrel(res[torch.float32][k].cpu(), res[torch.float64][k].cpu()))
        assert _nrel(ours, ref) <= bound, (k, _nrel(ours, ref), bound)


def test_edge_term_vs_fp64_oracle(cuda, morc):
    m = mr.random_mesh()
    (gv, gt), (rv, rt), _ = _grads_vs_oracle(cuda, morc, m, 3, edge_grad=True)
    (gv0, _), (rv0, _), _ = _grads_vs_oracle(cuda, morc, m, 3, edge_grad=False)
    assert _nrel(rv - rv0, rv0) > 0.05                 # the edge term is a visible part of the gradient
    assert _nrel(gv - gv0, rv - rv0) <= 1e-3
    assert _nrel(gv, rv) <= 1e-3


def _flat(cuda, xy, faces, H, W, tex, uv):
    """RenderLayer on verts (x, y, 1) with K = I, Rt = [I | 0]: v_pix = verts"""
    from goliath_b200.mesh_render import RenderLayer

    layer = RenderLayer(H, W, torch.as_tensor(faces), torch.as_tensor(uv, dtype=torch.float32),
                        torch.as_tensor(faces)).to(cuda)
    verts = torch.cat([xy, torch.ones_like(xy[..., :1])], -1)
    K = torch.eye(3, device=cuda, dtype=xy.dtype)[None]
    Rt = torch.eye(4, device=cuda, dtype=xy.dtype)[None, :3]
    return layer(verts, tex, K, Rt)


def test_edge_gradient_matches_area_derivative(cuda):
    """constant colour over background, cotangent 1: d(sum render)/dv is the derivative of the triangle's area"""
    rng = np.random.default_rng(5)
    H = W = 640
    tex = torch.ones(1, 1, 8, 8, device=cuda)
    uv = [[0.3, 0.3], [0.7, 0.4], [0.5, 0.7]]
    for _ in range(8):
        th0, r = rng.uniform(0, 2 * math.pi), rng.uniform(150, 280)
        ang = th0 + np.array([0.0, 2.0, 4.1]) + rng.uniform(-0.3, 0.3, 3)
        xy = torch.tensor(np.stack([320 + r * np.cos(ang), 320 + r * np.sin(ang)], -1)[None], dtype=torch.float32,
                          device=cuda).requires_grad_()
        out = _flat(cuda, xy, [[0, 1, 2]], H, W, tex, uv)
        (g,) = torch.autograd.grad(out["render"].sum(), [xy])
        p = xy.detach().double().requires_grad_()
        a = p[0]
        area = 0.5 * ((a[1, 0] - a[0, 0]) * (a[2, 1] - a[0, 1]) - (a[1, 1] - a[0, 1]) * (a[2, 0] - a[0, 0])).abs()
        (ga,) = torch.autograd.grad(area, [p])
        assert _nrel(g.double(), ga) <= 0.02, (_nrel(g.double(), ga), g, ga)


def test_edge_gradient_matches_supersampled_finite_difference(cuda):
    """a textured quad translated by t along (1, 0.3): dL/dt from the layer vs a central difference of the same loss
    on a 16 x 16 supersampled, box-filtered render"""
    H, W, S = 48, 64, 16
    gen = torch.Generator(device=cuda).manual_seed(3)
    tex = torch.rand(1, 3, 16, 16, device=cuda, generator=gen) + 0.5
    base = torch.tensor([[[14.3, 9.2], [47.6, 12.1], [44.8, 38.7], [17.1, 35.3]]], device=cuda)
    faces, uv = [[0, 1, 2], [0, 2, 3]], [[0.1, 0.1], [0.9, 0.1], [0.9, 0.9], [0.1, 0.9]]
    d = torch.tensor([1.0, 0.3], device=cuda)
    G = (torch.arange(W, device=cuda) / W)[None, None, None].expand(1, 3, H, W) + 0.2 * torch.rand(
        1, 3, H, W, device=cuda, generator=gen)

    t = torch.zeros((), device=cuda, requires_grad=True)
    out = _flat(cuda, base + t * d, faces, H, W, tex, uv)
    (dLdt,) = torch.autograd.grad((out["render"] * G).sum(), [t])

    def loss(tv):
        with torch.no_grad():
            r = _flat(cuda, (base + tv * d) * S, faces, H * S, W * S, tex, uv)["render"]
            return float((torch.nn.functional.avg_pool2d(r, S) * G).sum())

    h = 0.25
    fd = (loss(h) - loss(-h)) / (2 * h)
    assert np.sign(fd) == np.sign(float(dLdt)) and abs(float(dLdt) - fd) <= 0.1 * abs(fd), (float(dLdt), fd)


def _layer_inputs(cuda, B=2):
    m = mr.random_mesh(B=B, H=96, W=128, n=200, seed=4)
    gen = torch.Generator(device=cuda).manual_seed(9)
    tex = torch.rand(B, 4, 64, 64, device=cuda, generator=gen)
    return m, m["v_pix"].to(cuda), tex


def test_gradients_bitwise_repeatable_sync_free_and_graphed(cuda):
    from goliath_b200.graph import Graphed
    from goliath_b200.mesh_render import RenderLayer, _MeshRender

    m, v_pix, tex = _layer_inputs(cuda)
    layer = RenderLayer(96, 128, m["vi"], m["vt"], m["vti"]).to(cuda)
    w = torch.randn(2, 4, 96, 128, device=cuda, generator=torch.Generator(device=cuda).manual_seed(2))
    v = v_pix.clone().requires_grad_()
    t = tex.clone().requires_grad_()

    def step():
        return torch.autograd.grad((_MeshRender.apply(v, t, layer, True)[0] * w).sum(), [v, t])

    first = step()                                          # builds the vertex incidence lists
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        second = step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    assert first[0].abs().sum() > 0 and first[1].abs().sum() > 0
    with torch.no_grad():
        eager = [x.clone() for x in _MeshRender.apply(v.detach(), t.detach(), layer, True)]
        gr = Graphed(lambda: _MeshRender.apply(v.detach(), t.detach(), layer, True))
        for a, b in zip(gr(), eager):
            assert torch.equal(a, b)


def test_layer_vs_reference_fixture(cuda):
    from goliath_b200.mesh_render import RenderLayer

    gold = dict(np.load(GOLD))
    layer = RenderLayer(int(gold["h"]), int(gold["w"]), torch.from_numpy(gold["vi"]).long(),
                        torch.from_numpy(gold["vt_in"]), torch.from_numpy(gold["vti"]).long(),
                        flip_uvs=bool(gold["flip_uvs"])).to(cuda)
    layer.load_state_dict({"image_size": torch.from_numpy(gold["sd_image_size"])}, strict=True)
    verts = torch.from_numpy(gold["verts"]).float().to(cuda).requires_grad_()
    tex = torch.from_numpy(gold["tex"]).float().to(cuda).requires_grad_()
    K, Rt = torch.from_numpy(gold["K"]).float().to(cuda), torch.from_numpy(gold["Rt"]).float().to(cuda)
    out = layer(verts, tex, K, Rt, edge_grad=False)
    assert sorted(out) == sorted(str(k) for k in gold["keys"])
    # v_pix comes from an fp32 transform here and an fp64 one in the fixture (a few 1e-6 px apart): a sample point
    # within rounding of an edge may change face, and the sampled texture moves with the UVs; the other outputs are
    # compared where the index images agree, at a tolerance that covers the fp32 transform
    agree = out["index_img"].cpu().numpy() == gold["index_img"]
    assert agree.mean() >= 0.998, agree.mean()
    for k in ("render", "depth_img", "v_pix", "vt_img", "bary_img", "mask"):
        got, r = out[k].detach().cpu().numpy(), gold[k]
        if k != "v_pix":
            sel = np.broadcast_to(agree[:, None] if got.ndim == 4 else agree, got.shape)
            got, r = got[sel], r[sel]
        assert np.abs(got - r).max() <= 2e-3 * max(1.0, np.abs(r).max()), (k, np.abs(got - r).max())
    gv, gt = torch.autograd.grad((out["render"] * torch.from_numpy(gold["cotangent"]).float().to(cuda)).sum(),
                                 [verts, tex])
    assert _nrel(gt.cpu(), gold["g_tex"]) <= 1e-3, _nrel(gt.cpu(), gold["g_tex"])
    assert _nrel(gv.cpu(), gold["g_verts"]) <= 1e-2, _nrel(gv.cpu(), gold["g_verts"])
