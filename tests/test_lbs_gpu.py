"""GPU parity of the skinning and hand front-end kernels (DESIGN.md row R8': csrc/lbs.cu, gb_mvp_prim_frames_fwd,
goliath_b200/lbs.py, hand_mvp.GeomDecoder) against tests/golden/lbs_ref.npz, which RUNS the reference's own code on
CPU in fp64 (tests/golden/make_lbs_golden.py) on the seeded models of tests/lbs_recipe.py."""
import json
import os

import numpy as np
import pytest
import torch

import lbs_recipe as R

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lbs_ref.npz")
B = 2


def _close(got, ref, what, r=1e-4):
    """|got - ref| <= r * max|ref| everywhere, with NaN exactly where the reference has NaN"""
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    ref = np.asarray(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), "%s: NaN pattern differs" % what
    scale = float(np.abs(ref[~nan]).max()) if (~nan).any() else 1.0
    err = float(np.abs(got[~nan] - ref[~nan]).max()) if (~nan).any() else 0.0
    assert err <= r * scale, "%s: max abs err %.3e > %.1e * %.3e" % (what, err, r, scale)


def _module(kind, cuda, idx):
    from goliath_b200.lbs import LBSModule

    model, cfg, template, scales = R.skinned_model(kind, 100 + idx)
    return LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0]).to(cuda)


@pytest.mark.parametrize("idx,kind", list(enumerate(R.SKELETONS)))
def test_skeleton_matrices_and_states(cuda, idx, kind):
    g = np.load(GOLD)
    m = _module(kind, cuda, idx)
    _close(m.lbs_fn.bind_state, g[kind + "_bind"], kind + " bind_state")
    mo = R.motion(B, 200 + idx).to(cuda)
    mats, states = m.lbs_fn.skeleton(mo, m.lbs_scale.reshape(1, -1).expand(B, -1), return_states=True)
    _close(states, g[kind + "_states"], kind + " states")
    _close(mats, g[kind + "_mats"], kind + " matrices")


@pytest.mark.parametrize("vb", [1, B])
@pytest.mark.parametrize("idx,kind", list(enumerate(R.SKELETONS)))
def test_pose_and_vertex_gradient(cuda, idx, kind, vb):
    g = np.load(GOLD)
    m = _module(kind, cuda, idx)
    mo = R.motion(B, 200 + idx).to(cuda)
    gen = torch.Generator().manual_seed(300 + idx)
    V = m.lbs_fn.num_verts
    for b in (1, B):  # the generator's draws in the fixture's order
        vu = 0.1 * torch.randn(b, V, 3, generator=gen)
        w = torch.randn(B, V, 3, generator=gen)
        if b == vb:
            break
    vu = vu.to(cuda).requires_grad_()
    out = m.pose(vu, mo)
    _close(out, g["%s_pose%d" % (kind, vb)], "%s pose (vertex batch %d)" % (kind, vb))
    (out * w.to(cuda)).sum().backward()
    _close(vu.grad, g["%s_gv%d" % (kind, vb)], "%s grad verts_unposed (vertex batch %d)" % (kind, vb))
    if kind == "tree24":
        _close(m.template_pose(mo), g["tree24_template_pose"], "template_pose")


def test_state_dict_matches_reference_and_loads_strict(cuda):
    from goliath_b200.lbs import LBSModule

    g = np.load(GOLD)
    ref = json.loads(str(g["state_keys"]))
    model, cfg, template, scales = R.skinned_model("tree24", 100)
    m = LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0])
    sd = m.state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert list(m.lbs_fn.state_dict().keys()) == json.loads(str(g["lbs_fn_keys"]))
    for k, (shape, dtype) in ref.items():
        assert list(sd[k].shape) == shape and str(sd[k].dtype) == dtype, k
    # a state written by another module (here: perturbed copies) loads strictly and the kernels follow it
    m = m.to(cuda)
    mo = R.motion(B, 200).to(cuda)
    before = m.pose(torch.zeros(1, m.lbs_fn.num_verts, 3, device=cuda), mo)
    other = {k: v.clone() for k, v in sd.items()}
    other["lbs_fn.skin_weights"] = other["lbs_fn.skin_weights"].flip(1).contiguous()
    other["lbs_fn.skin_indices"] = other["lbs_fn.skin_indices"].flip(1).contiguous()
    m.load_state_dict(other, strict=True)
    after = m.pose(torch.zeros(1, m.lbs_fn.num_verts, 3, device=cuda), mo)
    assert torch.allclose(after, before, rtol=1e-5, atol=1e-4 * float(before.abs().max()))  # same sum, other slot order
    other["lbs_fn.joint_parents"] = torch.full_like(other["lbs_fn.joint_parents"], -1)
    m.load_state_dict(other, strict=True)
    flat = m.pose(torch.zeros(1, m.lbs_fn.num_verts, 3, device=cuda), mo)
    assert not torch.allclose(flat, before)  # the level order was rebuilt from the loaded parents


def _geom_decoder(cuda, train=False):
    from goliath_b200.hand_mvp import GeomDecoder
    from goliath_b200.lbs import LBSModule

    model, cfg, template, scales = R.tube_model(7)
    lbs = LBSModule(model, cfg, template[None], scales, global_scaling=[10.0, 10.0, 10.0])
    geo = R.TubeGeometry()
    dec = GeomDecoder(8, 2, 1024, 4096, lbs, geo, primposstart=1000)
    R.init_weights(dec.transdecoder, 11)
    R.init_weights(dec.alphadecoder, 12)
    geo.vt = geo.vt.to(cuda)
    return dec.to(cuda).train(train), geo


def test_geom_decoder_dict(cuda):
    g = np.load(GOLD)
    dec, geo = _geom_decoder(cuda)
    assert np.array_equal(dec.prim_vidx_img.cpu().numpy(), g["gd_vidx"])
    assert set(dict(dec.named_buffers())) >= {"prim_vidx_img", "prim_vtidx_img", "prim_bary_img"}
    assert not any(k.startswith("prim_") for k in dec.state_dict())
    pose = R.motion(B, 21).to(cuda)
    joint = torch.randn(B, 8, 64, 64, generator=torch.Generator().manual_seed(22)).to(cuda)
    p = dec(pose, joint, iteration=5000)
    assert sorted(p) == ["geom_lbs", "primalpha", "primpos", "primrot", "primscale"]
    for k in ("primpos", "primrot", "primscale", "geom_lbs"):
        _close(p[k], g["gd_" + k], "GeomDecoder " + k)
    assert p["primalpha"].shape == (B, 2, 1, 1024, 1024)
    _close(p["primalpha"].reshape(-1)[R.alpha_sample(p["primalpha"].numel()).to(cuda)], g["gd_alpha"], "primalpha")
    assert torch.isnan(p["primrot"][:, 2080]).any() and not torch.isnan(p["primrot"][:, :2080]).any()

    dec.train()
    pt = dec(pose[:1], joint[:1], iteration=0)  # iteration < primposstart: zero deltas
    for k in ("primpos", "primrot", "primscale"):
        _close(pt[k], g["gdt_" + k], "GeomDecoder training " + k)


def test_prim_base_frames_and_view_cos_with_negative_indices(cuda):
    from goliath_b200.hand_mvp import prim_base_frames, view_cos_uv

    g = np.load(GOLD)
    dec, geo = _geom_decoder(cuda)
    geom_lbs = torch.from_numpy(g["gd_geom_lbs"]).to(cuda)
    vidx = R.with_negative_indices(dec.prim_vidx_img)
    pos, rot = prim_base_frames(geom_lbs[:1], geo.vt, vidx, dec.prim_vtidx_img, dec.prim_bary_img)
    _close(pos, g["fr_posbase"], "primposbase")
    _close(rot, g["fr_rotbase"], "primrotbase")
    vc = view_cos_uv(geom_lbs, geo.vi.to(cuda), R.CAMPOS.to(cuda), vidx, dec.prim_bary_img)
    _close(vc, g["fr_view_cos_uv"], "view_cos_uv")
    assert (vc[:, 0, 0, :5] == 0).all() and (vc[:, 0, 3, 7] == 0).all()


# ------------------------------------------------------------------------------------------ large size
def _torch_pose(lbs, motion, verts):
    """LBSModule.pose restated in torch (fp64): per-joint chain, states_to_matrix, gather-and-sum skinning"""
    f = lbs.lbs_fn
    d = torch.float64
    params = torch.cat([motion.to(d), lbs.lbs_scale.to(d).reshape(1, -1).expand(motion.shape[0], -1)], 1)
    jp = (f.param_transform.transform.to(d) @ params.t()).t() + f.param_transform.transform_offsets.to(d)
    jp = jp.view(motion.shape[0], -1, 7)

    def qmul(q, r):
        x1, y1, z1, w1 = q.unbind(-1)
        x2, y2, z2, w2 = r.unbind(-1)
        return torch.stack([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                            w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2], -1)

    def qrot(q, v):
        u, w = q[..., :3], q[..., 3:]
        return v + 2 * (w * torch.cross(u, v, dim=-1) + torch.cross(u, torch.cross(u, v, dim=-1), dim=-1))

    h = jp[..., 3:6] * torch.tensor([-0.5, 0.5, 0.5], dtype=d, device=jp.device)
    c, s = torch.cos(h), torch.sin(h)
    qx = -s[..., 0] * c[..., 1] * c[..., 2] - c[..., 0] * s[..., 1] * s[..., 2]
    qy = c[..., 0] * s[..., 1] * c[..., 2] - s[..., 0] * c[..., 1] * s[..., 2]
    qz = c[..., 0] * c[..., 1] * s[..., 2] + s[..., 0] * s[..., 1] * c[..., 2]
    qw = c[..., 0] * c[..., 1] * c[..., 2] - s[..., 0] * s[..., 1] * s[..., 2]
    lr = qmul(f.joint_rotation.to(d)[None].expand_as(jp[..., :4]), torch.stack([qx, qy, qz, qw], -1))
    lt, ls = jp[..., :3] + f.joint_offset.to(d), torch.pow(2.0, jp[..., 6:7])
    st = []
    for j, p in enumerate(f.joint_parents.reshape(-1).tolist()):
        if p == -1:
            st.append(torch.cat([lt[:, j], lr[:, j], ls[:, j]], -1))
        else:
            ps = st[p]
            st.append(torch.cat([qrot(ps[:, 3:7], lt[:, j] * ps[:, 7:]) + ps[:, :3], qmul(ps[:, 3:7], lr[:, j]),
                                 ps[:, 7:] * ls[:, j]], -1))
    st = torch.stack(st, 1)
    bind = f.bind_state.to(d)
    bq = bind[..., 3:7] * torch.tensor([-1.0, -1, -1, 1], dtype=d, device=bind.device) / (bind[..., 3:7] ** 2).sum(-1, keepdim=True)
    bs = 1.0 / bind[..., 7:]
    bt = qrot(bq, -bind[..., :3]) * bs
    tr, ts = qmul(st[..., 3:7], bq.expand_as(st[..., 3:7])), st[..., 7:] * bs
    tt = qrot(st[..., 3:7], bt * st[..., 7:]) + st[..., :3]
    x, y, z, w = tr.unbind(-1)
    R_ = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                      2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                      2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1).view(*tr.shape[:2], 3, 3)
    M = torch.cat([R_ * ts[..., None], tt[..., None]], -1)
    vh = verts.to(d) + lbs.lbs_template_verts.to(d).reshape(1, -1, 3)
    Mk = M[:, f.skin_indices]                                   # [B, V, 8, 3, 4]
    out = (Mk[..., :3] @ vh[:, :, None, :, None]).squeeze(-1) + Mk[..., 3]
    out = (out * f.skin_weights.to(d)[None, :, :, None]).sum(2)
    return out * lbs.global_scaling.to(d)


def test_torch_restatement_pinned_to_fixture(cuda):
    g = np.load(GOLD)
    for idx, kind in enumerate(R.SKELETONS):
        m = _module(kind, cuda, idx)
        gen = torch.Generator().manual_seed(300 + idx)
        vu = (0.1 * torch.randn(1, m.lbs_fn.num_verts, 3, generator=gen)).to(cuda)
        _close(_torch_pose(m, R.motion(B, 200 + idx).to(cuda), vu), g[kind + "_pose1"], kind + " restatement", 3e-5)


def test_large_batch_against_restatement(cuda):
    from goliath_b200.lbs import LBSModule

    model, cfg, template, scales = R.skinned_model("tree24", 5, n_verts=100_000)
    m = LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0]).to(cuda)
    mo = R.motion(8, 6).to(cuda)
    vu = (0.1 * torch.randn(8, 100_000, 3, generator=torch.Generator().manual_seed(7))).to(cuda)
    _close(m.pose(vu, mo), _torch_pose(m, mo, vu).cpu().numpy(), "B=8, 100k vertices")


def test_graph_replay_and_deterministic_backward(cuda):
    dec, geo = _geom_decoder(cuda)
    from goliath_b200.hand_mvp import prim_base_frames, view_cos_uv

    lbs = dec.lbs_fn
    pose = R.motion(B, 21).to(cuda)
    campos = R.CAMPOS.to(cuda)
    vi = geo.vi.to(cuda)

    def front():
        geom = lbs.pose(torch.zeros_like(lbs.lbs_template_verts), pose)
        pos, rot = prim_base_frames(geom, geo.vt, dec.prim_vidx_img, dec.prim_vtidx_img, dec.prim_bary_img)
        return geom, pos, rot, view_cos_uv(geom, vi, campos, dec.prim_vidx_img, dec.prim_bary_img)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            eager = front()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = front()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(outs[:3], eager[:3]):  # geom_lbs, primposbase, primrotbase: bit for bit
        assert torch.equal(torch.nan_to_num(a, 7.0), torch.nan_to_num(b, 7.0))
    # the view cosine reads gb_vert_normals_fwd, whose face pass adds with atomics: equal up to the summation order
    assert torch.allclose(outs[3], eager[3], rtol=0, atol=1e-5)

    vu = torch.zeros(1, lbs.lbs_fn.num_verts, 3, device=cuda, requires_grad=True)
    w = torch.randn(B, lbs.lbs_fn.num_verts, 3, generator=torch.Generator().manual_seed(3)).to(cuda)
    grads = []
    for _ in range(3):
        (lbs.pose(vu, pose) * w).sum().backward()
        grads.append(vu.grad.clone())
        vu.grad = None
    assert all(torch.equal(grads[0], x) for x in grads[1:])
