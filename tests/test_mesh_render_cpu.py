"""CPU checks of the body render (DESIGN.md R9''): the C oracle (oracle/mesh_oracle.c through oracle/mesh.py) against a brute-force fp64
torch restatement on the raster edge cases, its interior gradient against torch autograd of the restatement, and
`RenderLayer`'s buffers."""
import numpy as np
import pytest
import torch

import mesh_render_restate as mr


@pytest.fixture(scope="module")
def morc():
    from oracle import mesh

    mesh.lib()
    return mesh


def _tex(C, Ht, Wt, seed=0):
    return np.random.default_rng(seed).uniform(-1, 1, size=(1, C, Ht, Wt)).astype(np.float32)


@pytest.mark.parametrize("name", sorted(mr.cases()))
def test_oracle_index_and_render_vs_bruteforce(morc, name):
    m = mr.cases()[name]
    v, vi = m["v_pix"], m["vi"]
    idx = morc.mesh_raster(v.numpy(), vi.numpy(), m["H"], m["W"])
    ref, dep = mr.raster_bruteforce(v, vi, m["H"], m["W"])
    diff = idx != ref.numpy()
    if diff.any():  # only rounding ties: both faces contain the pixel at (almost) the same fp64 depth
        lam, _, z = mr.screen_bary(v[0].double(), vi, torch.arange(m["W"], dtype=torch.float64)[None] + 0.5,
                                   torch.arange(m["H"], dtype=torch.float64)[:, None] + 0.5)
        q = lam / z[:, :, None, None]
        d = 1 / q.sum(1)
        for b, y, x in zip(*np.nonzero(diff)):
            f = int(idx[b, y, x])
            assert f >= 0 and (lam[f, :, y, x] >= 0).all(), (name, b, y, x)
            assert abs(float(d[f, y, x]) - float(dep[b, y, x])) <= 1e-6 * float(dep[b, y, x]), (name, b, y, x)
    assert diff.mean() < 0.01, name
    tex = _tex(4, 16, 24)
    tex = np.repeat(tex, v.shape[0], 0)
    o = morc.mesh_render_fwd(v.numpy(), vi.numpy(), m["vti"].numpy(), m["vt"].numpy(), tex, idx)
    r = mr.render_at(v.double(), vi, m["vti"], m["vt"].double(), torch.from_numpy(tex).double(), torch.from_numpy(idx))
    for k in ("depth_img", "bary_img", "vt_img", "mask", "render"):
        np.testing.assert_allclose(o[k], r[k].numpy(), rtol=1e-9, atol=1e-9, err_msg=k)
    assert (idx >= 0).any()


def test_raster_case_expectations(morc):
    c = mr.cases()
    idx = {k: morc.mesh_raster(m["v_pix"].numpy(), m["vi"].numpy(), m["H"], m["W"]) for k, m in c.items()}
    assert set(np.unique(idx["duplicates"])) == {-1, 0, 1}    # 1: the smallest id of three coplanar copies
    assert set(np.unique(idx["behind"])) == {-1, 2}           # faces with a z <= 0 vertex are not drawn
    assert set(np.unique(idx["zero_area"])) == {-1, 2}        # collinear / repeated-vertex faces are skipped
    assert set(np.unique(idx["off_screen"])) == {-1, 0, 1}    # partly visible faces only
    assert (idx["huge"] == 1).sum() > 10 and (idx["huge"] == 0).sum() + (idx["huge"] == 1).sum() == 24 * 32


def test_oracle_interior_gradient_vs_autograd(morc):
    m = mr.random_mesh()
    v, vi, vti, vt = m["v_pix"], m["vi"], m["vti"], m["vt"]
    B = v.shape[0]
    idx = morc.mesh_raster(v.numpy(), vi.numpy(), m["H"], m["W"])
    tex = np.random.default_rng(3).uniform(-1, 1, size=(B, 3, 20, 28)).astype(np.float32)
    g = np.random.default_rng(4).standard_normal((B, 3, m["H"], m["W"])).astype(np.float32)
    gv, gt = morc.mesh_render_bwd(v.numpy(), vi.numpy(), vti.numpy(), vt.numpy(), tex, idx, g, edge_grad=False)
    vv = v.double().requires_grad_()
    tt = torch.from_numpy(tex).double().requires_grad_()
    r = mr.render_at(vv, vi, vti, vt.double(), tt, torch.from_numpy(idx))["render"]
    rv, rt = torch.autograd.grad((r * torch.from_numpy(g).double()).sum(), [vv, tt])
    np.testing.assert_allclose(gv, rv.numpy(), rtol=1e-8, atol=1e-9)
    np.testing.assert_allclose(gt, rt.numpy(), rtol=1e-8, atol=1e-9)
    # the edge term adds only x, y gradients, and only to faces at a visibility boundary
    ge, _ = morc.mesh_render_bwd(v.numpy(), vi.numpy(), vti.numpy(), vt.numpy(), tex, idx, g, edge_grad=True)
    assert np.array_equal(ge[..., 2], gv[..., 2]) and not np.allclose(ge, gv)


def _layer(**kw):
    from goliath_b200.mesh_render import RenderLayer

    m = mr.random_mesh()
    return RenderLayer(40, 56, m["vi"].long(), m["vt"], m["vti"].long(), **kw), m


def test_layer_buffers_strict_load_and_flip_uvs():
    layer, m = _layer()
    assert list(layer.state_dict()) == ["image_size"]
    sd = {"image_size": torch.tensor([40, 56], dtype=torch.int32)}
    layer.load_state_dict(sd, strict=True)
    assert layer.image_size.dtype == torch.int32 and layer.image_size.tolist() == [40, 56]
    vt = m["vt"].clone()
    from goliath_b200.mesh_render import RenderLayer

    flipped = RenderLayer(40, 56, m["vi"], vt, m["vti"], flip_uvs=True)
    assert torch.equal(vt, m["vt"])                                   # the caller's vt is unchanged
    assert torch.equal(flipped.vt[:, 1], 1 - m["vt"][:, 1]) and torch.equal(flipped.vt[:, 0], m["vt"][:, 0])


def test_layer_refuses_cpu_and_unsupported_arguments():
    layer, m = _layer()
    B = m["v_pix"].shape[0]
    verts = torch.randn(B, m["v_pix"].shape[1], 3)
    tex = torch.rand(B, 4, 8, 8)
    K, Rt = torch.eye(3).expand(B, 3, 3), torch.eye(4)[:3].expand(B, 3, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(verts, tex, K, Rt)
    with pytest.raises(ValueError):
        layer(verts, tex, K, Rt, background=torch.zeros(3))
    with pytest.raises(ValueError):
        layer(verts, tex, K, Rt, output_filters=["render"])


def test_transform_matches_pinhole():
    from goliath_b200.mesh_render import transform

    g = torch.Generator().manual_seed(0)
    v = torch.randn(2, 5, 3, generator=g, dtype=torch.float64)
    R = torch.linalg.qr(torch.randn(2, 3, 3, generator=g, dtype=torch.float64))[0]
    t = torch.tensor([[0.1, -0.2, 6.0], [0.0, 0.3, 7.0]], dtype=torch.float64)
    K = torch.tensor([[500.0, 0, 40], [0, 510.0, 30], [0, 0, 1]], dtype=torch.float64).expand(2, 3, 3)
    out = transform(v, K, torch.cat([R, t[:, :, None]], 2))
    vc = v @ R.transpose(1, 2) + t[:, None]
    assert torch.allclose(out[..., 0], 500 * vc[..., 0] / vc[..., 2] + 40)
    assert torch.allclose(out[..., 1], 510 * vc[..., 1] / vc[..., 2] + 30)
    assert torch.allclose(out[..., 2], vc[..., 2])
