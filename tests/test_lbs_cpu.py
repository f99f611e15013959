"""CPU: the skinning modules' buffers, bind state and refusals (goliath_b200/lbs.py), without a GPU."""
import numpy as np
import pytest
import torch

import lbs_recipe as R
from goliath_b200 import lbs


def _model(kind="tree24", seed=100):
    return R.skinned_model(kind, seed)


def test_buffers_follow_the_reference_layout():
    model, cfg, template, scales = _model()
    m = lbs.LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0])
    f = m.lbs_fn
    J, V = 24, 500
    assert f.joint_parents.shape == (J, 1) and f.joint_parents.dtype == torch.int64
    assert f.joint_parents[0, 0] == -1 and f.joint_parents[9, 0] == -1   # Parent 1000 > J -> root
    assert f.skin_indices.shape == (V, 8) and f.skin_indices.dtype == torch.int64
    assert f.mesh_faces.dtype == torch.int32 and f.bind_state.shape == (1, J, 8)
    assert f.joints_weights.shape == (J, V)
    offs = model["SkinnedModel"]["SkinningOffsets"]
    sw = model["SkinnedModel"]["SkinningWeights"]
    for v in (0, 17, V - 1):  # ragged offsets -> slot k holds entry offsets[v] + k, zero past the vertex's count
        n = offs[v + 1] - offs[v]
        assert f.skin_indices[v, :n].tolist() == [e[0] for e in sw[offs[v]:offs[v + 1]]]
        assert np.allclose(f.skin_weights[v, :n].numpy(), [e[1] for e in sw[offs[v]:offs[v + 1]]])
        assert (f.skin_weights[v, n:] == 0).all() and (f.skin_indices[v, n:] == 0).all()
    keys = list(m.state_dict())
    assert keys[:3] == ["lbs_scale", "lbs_template_verts", "global_scaling"]
    assert keys[-2:] == ["lbs_fn.param_transform.transform_offsets", "lbs_fn.param_transform.transform"]


def test_bind_state_is_the_zero_pose_chain():
    """bind_state = the joint chain at the parameter offsets; checked with a direct per-joint loop in fp64"""
    model, cfg, template, scales = _model("chain160", 101)
    f = lbs.LinearBlendSkinning(model, cfg)
    jp = torch.as_tensor(cfg["transform_offsets"], dtype=torch.float64).view(-1, 7)
    st = []
    for j, p in enumerate(f.joint_parents.reshape(-1).tolist()):
        lt = jp[j, :3] + f.joint_offset[j].double()
        lr = lbs._qmul(f.joint_rotation[j].double(), lbs._from_xyz(jp[j, 3:6]))
        ls = 2.0 ** jp[j, 6]
        if p == -1:
            st.append(torch.cat([lt, lr, ls[None]]))
        else:
            q, t, s = st[p][3:7], st[p][:3], st[p][7]
            st.append(torch.cat([lbs._qrot(q, lt * s) + t, lbs._qmul(q, lr), (s * ls)[None]]))
    ref = torch.stack(st)[None]
    assert torch.allclose(f.bind_state.double(), ref, rtol=1e-4, atol=1e-4 * float(ref.abs().max()))


def test_skeleton_levels():
    order, start = lbs.skeleton_levels([-1, 0, 0, 1, -1, 4, 3])
    assert start.tolist() == [0, 2, 5, 6, 7]
    assert sorted(order[:2].tolist()) == [0, 4] and sorted(order[2:5].tolist()) == [1, 2, 5]
    assert order[5:].tolist() == [3, 6]
    o, s = lbs.skeleton_levels([-1] + [0] * 300)
    assert s.tolist() == [0, 1, 301]


@pytest.mark.parametrize("bad", [[-1, 2, 0], [-1, 1], [-1, 0, -2], [0]])
def test_misordered_skeleton_is_refused(bad):
    model, cfg, template, scales = _model()
    bones = model["Skeleton"]["Bones"][:len(bad)]
    for b, p in zip(bones, bad):
        b["Parent"] = p
    model["Skeleton"]["Bones"] = bones
    cfg = dict(cfg, transform=cfg["transform"][:7 * len(bad)], transform_offsets=cfg["transform_offsets"][:, :7 * len(bad)])
    model["SkinnedModel"]["SkinningWeights"] = [[0, 1.0] for _ in model["SkinnedModel"]["SkinningWeights"]]
    with pytest.raises(ValueError, match="parent"):
        lbs.LinearBlendSkinning(model, cfg)


def test_too_many_joints_is_refused():
    from goliath_b200 import _lib

    assert _lib.lib().gb_lbs_max_joints() == lbs.MAX_JOINTS
    J = lbs.MAX_JOINTS + 1
    model = {"Skeleton": {"Bones": [{"Name": "j%d" % j, "Parent": j - 1, "PreRotation": [0, 0, 0, 1],
                                     "TranslationOffset": [0, 0, 0]} for j in range(J)]}}
    with pytest.raises(ValueError, match="at most"):
        lbs.LinearBlendSkinning(model, {"channel_names": [], "limits": [], "transform": np.zeros((7 * J, 1), np.float32),
                                        "transform_offsets": np.zeros((1, 7 * J), np.float32),
                                        "nr_scaling_params": 0, "nr_position_params": 1})


def test_cpu_module_and_grad_motion_are_refused():
    model, cfg, template, scales = _model()
    m = lbs.LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0])
    mo = R.motion(2, 1)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.pose(torch.zeros(1, 500, 3), mo)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.lbs_fn(mo, torch.zeros(2, 4))
    with pytest.raises(RuntimeError, match="requires grad"):
        m.pose(torch.zeros(1, 500, 3), mo.clone().requires_grad_())
    with pytest.raises(RuntimeError, match="requires grad"):
        m.lbs_fn(mo, torch.zeros(2, 4, requires_grad=True))
    with torch.no_grad():  # under no_grad nothing would be differentiated: only the device is refused
        with pytest.raises(RuntimeError, match="CUDA"):
            m.pose(torch.zeros(1, 500, 3), mo.clone().requires_grad_())


def test_init_primitives_keeps_torch_negative_indexing():
    from goliath_b200.hand_mvp import init_primitives

    geo = R.TubeGeometry()
    vidx, vtidx, bary = init_primitives(1024, 4096, geo)
    assert vidx.shape == (64, 64, 3) and bary.shape == (64, 64, 3)
    _, face, _ = geo.render_index_images(1024, impaint=True)
    assert face[8, 8] == -1
    assert vidx[0, 0].tolist() == geo.vi[-1].tolist() and vtidx[0, 0].tolist() == geo.vti[-1].tolist()
    assert vidx[32, 32].tolist() == geo.vi[geo.degenerate_face].tolist()
