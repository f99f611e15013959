"""Linear blend skinning of the tracked mesh (DESIGN.md row R8'): `ParameterTransform`, `LinearBlendSkinning` and
`LBSModule` of ca_code/utils/lbs.py with the reference's constructor arguments and persistent buffers (names, shapes,
dtypes), so a checkpoint holding the reference's `lbs_fn.*` buffers loads with strict=True.

The posing runs on csrc/lbs.cu: one launch computes the parameter transform, the joint chain (level by level of the
skeleton tree) and the skinning matrices, a second one skins the vertices, or, for `unpose`, applies the inverse of
each vertex's blended matrix (forward only).  Gradients flow to the vertices only;
pose and scale gradients are not implemented, so a `motion` / `scales` that requires grad is refused.  The bind state
is computed once on the host at construction, as the reference does."""
from typing import Any, Dict, Optional

import numpy as np
import torch
import torch.nn as nn
from torch.autograd import Function

from . import _lib

MAX_JOINTS = 1024  # gb_lbs_max_joints(): one CTA keeps every joint's state in shared memory
N_SLOTS = 8        # influences per vertex the skinning kernel reads


# ------------------------------------------------------------------------------------------ host-side setup
def _qmul(q, r):
    qx, qy, qz, qw = q.unbind(-1)
    rx, ry, rz, rw = r.unbind(-1)
    return torch.stack([qx * rw + qy * rz - qz * ry + qw * rx, -qx * rz + qy * rw + qz * rx + qw * ry,
                        qx * ry - qy * rx + qz * rw + qw * rz, -qx * rx - qy * ry - qz * rz + qw * rw], -1)


def _qrot(q, v):
    a = q[..., :3]
    av = torch.cross(a, v, dim=-1)
    return v + 2 * (av * q[..., 3:] + torch.cross(a, av, dim=-1))


def _from_xyz(r):
    rm = r * torch.tensor([-0.5, 0.5, 0.5], dtype=r.dtype)
    (c0, c1, c2), (s0, s1, s2) = torch.cos(rm).unbind(-1), torch.sin(rm).unbind(-1)
    return torch.stack([-s0 * (c1 * c2) - c0 * (s1 * s2), c0 * (s1 * c2) - s0 * (c1 * s2),
                        c0 * (c1 * s2) + s0 * (s1 * c2), c0 * (c1 * c2) - s0 * (s1 * s2)], -1)


def skeleton_levels(parents):
    """parents [J] (-1 = root) -> (order [J], level_start [L+1]) listing the joints level by level, roots first.
    Raises unless every parent index is -1 or below the joint's own index, which the reference's loop
    (lbs.py:364-383) needs as well."""
    p = [int(x) for x in np.asarray(parents).reshape(-1)]
    depth = []
    for j, pj in enumerate(p):
        if pj == -1:
            depth.append(0)
        elif 0 <= pj < j:
            depth.append(depth[pj] + 1)
        else:
            raise ValueError("skeleton joint %d has parent %d: parents must be -1 or a lower joint index" % (j, pj))
    depth = np.asarray(depth, dtype=np.int64)
    order = np.argsort(depth, kind="stable").astype(np.int32)
    level_start = np.searchsorted(depth[order], np.arange(int(depth.max()) + 2)).astype(np.int32)
    return order, level_start


def _solve_states_host(params, joint_offset, joint_rotation, parents):
    """solve_skeleton_state (lbs.py:340-385) on the host, one tree level at a time: params [N, 7J] -> [N, J, 8]."""
    jp = params.reshape(params.shape[0], -1, 7)
    lt = jp[..., 0:3] + joint_offset[None]
    lr = _qmul(joint_rotation[None].expand_as(jp[..., :4]), _from_xyz(jp[..., 3:6]))
    ls = torch.pow(torch.tensor([2.0], dtype=params.dtype), jp[..., 6:7])
    state = torch.cat([lt, lr, ls], -1)
    order, start = skeleton_levels(parents)
    p = torch.as_tensor(np.asarray(parents).reshape(-1), dtype=torch.long)
    for lo, hi in zip(start[1:-1], start[2:]):
        j = torch.as_tensor(order[lo:hi], dtype=torch.long)
        ps = state[:, p[j]]
        gr = _qmul(ps[..., 3:7], lr[:, j])
        gt = _qrot(ps[..., 3:7], lt[:, j] * ps[..., 7:8]) + ps[..., 0:3]
        state[:, j] = torch.cat([gt, gr, ps[..., 7:8] * ls[:, j]], -1)
    return state


# ------------------------------------------------------------------------------------------ modules
class ParameterTransform(nn.Module):
    """lbs.py:23-46: the [7J, P+S] pose-parameter -> joint-parameter map.  Its forward (a host-side matmul used to
    build the bind state) is fused into gb_lbs_skeleton_fwd on the device path."""

    def __init__(self, lbs_cfg_dict: Dict[str, Any]):
        super().__init__()
        self.channel_names = list(lbs_cfg_dict["channel_names"])
        self.limits = lbs_cfg_dict["limits"]
        self.nr_scaling_params = lbs_cfg_dict["nr_scaling_params"]
        self.nr_position_params = lbs_cfg_dict["nr_position_params"]
        self.nr_total_params = self.nr_scaling_params + self.nr_position_params
        self.register_buffer("transform_offsets", torch.FloatTensor(lbs_cfg_dict["transform_offsets"]))
        self.register_buffer("transform", torch.FloatTensor(lbs_cfg_dict["transform"]))

    def forward(self, pose: torch.Tensor) -> torch.Tensor:
        return self.transform.mm(pose.t()).t() + self.transform_offsets


class _Skin(Function):
    @staticmethod
    def forward(ctx, verts, mats, templ, skin_idx, skin_w, gscale):
        verts = verts.contiguous()
        _lib.check_input(verts, "verts_unposed")
        B, J = mats.shape[0], mats.shape[1]
        vb, V = verts.shape[0], verts.shape[1]
        if verts.shape[2:] != (3,) or vb not in (1, B) or skin_idx.shape != (V, N_SLOTS):
            raise RuntimeError("verts_unposed must be [1 or B, V, 3] with V = the skinned mesh's vertex count")
        out = torch.empty(B, V, 3, device=verts.device)
        _lib.kernels().gb_lbs_skin_fwd(B, V, J, vb, mats, verts, templ, skin_idx, skin_w, gscale, out)
        ctx.save_for_backward(mats, skin_idx, skin_w, gscale)
        ctx.vb = vb
        return out

    @staticmethod
    def backward(ctx, g_out):
        mats, skin_idx, skin_w, gscale = ctx.saved_tensors
        B, J = mats.shape[0], mats.shape[1]
        V = skin_idx.shape[0]
        g_out = g_out.contiguous()
        g_v = torch.empty(ctx.vb, V, 3, device=g_out.device)
        _lib.kernels().gb_lbs_skin_bwd(B, V, J, ctx.vb, mats, skin_idx, skin_w, gscale, g_out, g_v)
        return g_v, None, None, None, None, None


def _no_grad_input(t, name):
    if torch.is_grad_enabled() and t.requires_grad:
        raise RuntimeError("%s requires grad, but the skinning kernels give no pose or scale gradient" % name)


class LinearBlendSkinning(nn.Module):
    """lbs.py:49-337: buffers built from the model json / parameter config dicts exactly as the reference builds them
    (including `Parent > J` -> root and the ragged SkinningOffsets -> [V, num_max_skin_joints] tables)."""

    def __init__(self, model_json: Dict[str, Any], lbs_config_dict: Dict[str, Any], num_max_skin_joints: int = 8):
        super().__init__()
        if num_max_skin_joints != N_SLOTS:
            raise ValueError("the skinning kernel reads %d influences per vertex" % N_SLOTS)
        self.param_transform = ParameterTransform(lbs_config_dict)
        bones = model_json["Skeleton"]["Bones"]
        J = len(bones)
        if J > MAX_JOINTS:
            raise ValueError("%d joints: the skeleton kernel holds at most %d" % (J, MAX_JOINTS))
        self.joint_names = [b["Name"] for b in bones]
        joint_parents = torch.tensor([[-1 if b["Parent"] > J else b["Parent"]] for b in bones], dtype=torch.int64)
        joint_rotation = torch.FloatTensor([b["PreRotation"] for b in bones]).reshape(J, 4)
        joint_offset = torch.FloatTensor([b["TranslationOffset"] for b in bones]).reshape(J, 3)
        skeleton_levels(joint_parents)  # refuse a misordered skeleton before anything else is built

        skin = model_json["SkinnedModel"]
        mesh_vertices = torch.FloatTensor(skin["RestPositions"])
        mesh_normals = torch.FloatTensor(skin["RestVertexNormals"])
        weights = torch.FloatTensor([e[1] for e in skin["SkinningWeights"]])
        indices = torch.LongTensor([e[0] for e in skin["SkinningWeights"]])
        offsets = torch.LongTensor(skin["SkinningOffsets"])
        V = len(offsets) - 1
        skin_weights = torch.zeros(V, num_max_skin_joints, dtype=torch.float32)
        skin_indices = torch.zeros(V, num_max_skin_joints, dtype=torch.int64)
        for k in range(num_max_skin_joints):  # slot k of vertex v holds entry offsets[v] + k when it is in range
            left = offsets[:-1] + k
            m = left < offsets[1:]
            skin_weights[m, k] = weights[left[m]]
            skin_indices[m, k] = indices[left[m]]

        zero = torch.zeros(1, self.param_transform.nr_total_params, dtype=torch.float32)
        bind_state = _solve_states_host(self.param_transform(zero), joint_offset, joint_rotation, joint_parents)

        self.register_buffer("mesh_vertices", mesh_vertices)
        self.register_buffer("joint_parents", joint_parents)
        self.register_buffer("joint_rotation", joint_rotation)
        self.register_buffer("joint_offset", joint_offset)
        self.register_buffer("mesh_normals", mesh_normals)
        self.register_buffer("mesh_faces", torch.IntTensor(skin["Faces"]["Indices"]).view(-1, 3))
        self.register_buffer("mesh_texture_faces", torch.IntTensor(skin["Faces"]["TextureIndices"]).view(-1, 3))
        self.register_buffer("mesh_texture_coords", torch.FloatTensor(skin["TextureCoordinates"]).view(-1, 2))
        self.register_buffer("skin_weights", skin_weights)
        self.register_buffer("skin_indices", skin_indices)
        self.register_buffer("bind_state", bind_state)
        self.register_buffer("rest_vertices", mesh_vertices)
        joints_weights = torch.zeros(J, V, dtype=torch.float32)  # lbs.py:171-186
        joints_weights[skin_indices, torch.arange(V)[:, None].expand(-1, num_max_skin_joints)] = skin_weights
        self.register_buffer("joints_weights", joints_weights)
        self._derived = None

    @property
    def num_verts(self):
        return self.mesh_vertices.size(0)

    @property
    def num_joints(self):
        return self.joint_offset.size(0)

    @property
    def num_params(self):
        return self.skin_weights.shape[-1]

    def _kernel_tables(self):
        """int32 / contiguous copies of the buffers the kernels read and the level order, rebuilt whenever a buffer
        was replaced or written in place (load_state_dict, .to(), ...)."""
        srcs = (self.joint_parents, self.skin_indices, self.skin_weights, self.bind_state, self.joint_offset,
                self.joint_rotation, self.param_transform.transform, self.param_transform.transform_offsets)
        key = tuple((t.data_ptr(), t._version, t.device) for t in srcs)
        if self._derived is not None and self._derived[0] == key:
            return self._derived[1]
        dev = self.joint_parents.device
        if dev.type != "cuda":
            raise RuntimeError("LinearBlendSkinning runs on CUDA kernels only: move the module to a CUDA device")
        parents = self.joint_parents.reshape(-1)
        J = parents.numel()
        if J > MAX_JOINTS:
            raise ValueError("%d joints: the skeleton kernel holds at most %d" % (J, MAX_JOINTS))
        order, start = skeleton_levels(parents.cpu())
        c = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        tabs = dict(parents=parents.to(torch.int32).contiguous(),
                    order=torch.as_tensor(order, device=dev), level_start=torch.as_tensor(start, device=dev),
                    n_levels=len(start) - 1, skin_idx=self.skin_indices.to(torch.int32).contiguous(),
                    skin_w=c(self.skin_weights), bind=c(self.bind_state.reshape(J, 8)), joint_offset=c(self.joint_offset),
                    joint_rotation=c(self.joint_rotation), transform=c(self.param_transform.transform),
                    offsets=c(self.param_transform.transform_offsets.reshape(-1)))
        if tabs["offsets"].numel() != 7 * J or tabs["transform"].shape[0] != 7 * J:
            raise RuntimeError("transform must be [7J, P+S] and transform_offsets hold 7J values")
        self._derived = (key, tabs)
        return tabs

    def skeleton(self, poses: torch.Tensor, scales: torch.Tensor, return_states: bool = False):
        """ParameterTransform + solve_skeleton_state + states_to_matrix(bind_state, .) in one launch:
        poses [B,P], scales [B,S] (or a stride-0 expand of one row) -> mats [B,J,3,4] (and states [B,J,8])."""
        _no_grad_input(poses, "motion")
        _no_grad_input(scales, "scales")
        tabs = self._kernel_tables()
        poses = poses.contiguous()
        _lib.check_input(poses, "poses")
        if poses.device != tabs["parents"].device:
            raise RuntimeError("poses must be on the module's device")
        if scales.dim() == 1:
            scales = scales[None]
        if scales.stride(-1) != 1:
            scales = scales.contiguous()
        if scales.device != poses.device or scales.dtype != torch.float32:
            raise RuntimeError("scales must be float32 on the poses' device")
        B, P = poses.shape
        S = scales.shape[1]
        J = tabs["parents"].numel()
        if tabs["transform"].shape[1] != P + S or scales.shape[0] not in (1, B):
            raise RuntimeError("poses [B,P] and scales [B,S] must give P+S = transform.shape[1]")
        stride = scales.stride(0) if scales.shape[0] == B else 0  # 0: one row for every item (lbs_scale.expand)
        mats = torch.empty(B, J, 3, 4, device=poses.device)
        states = torch.empty(B, J, 8, device=poses.device) if return_states else None
        _lib.kernels().gb_lbs_skeleton_fwd(
            B, J, P, S, poses, scales, stride, tabs["transform"], tabs["offsets"], tabs["joint_offset"],
            tabs["joint_rotation"], tabs["parents"], tabs["order"], tabs["level_start"], tabs["n_levels"],
            tabs["bind"], mats, states)
        return (mats, states) if return_states else mats

    def skin(self, mats, verts, template=None, global_scaling=None):
        """global_scaling * skinning(mats, verts + template): verts [1 or B, V, 3], template [V,3] / [1,V,3] or None,
        global_scaling [3] or None.  Gradients flow to `verts`."""
        tabs = self._kernel_tables()
        return _Skin.apply(verts, mats, template, tabs["skin_idx"], tabs["skin_w"], global_scaling)

    def unskin(self, mats, verts, template=None, global_scaling=None):
        """The inverse of `skin`: (blended matrix)^-1 [verts / global_scaling; 1] - template, one launch (lbs.py:273-306
        with the scaling and template of lbs.py:733-739).  verts [1 or B, V, 3]; a vertex whose blended matrix is
        singular comes back NaN.  Forward only: a `verts` that requires grad is refused."""
        if torch.is_grad_enabled() and verts.requires_grad:
            raise RuntimeError("verts requires grad, but the unskinning kernel has no backward (call it under no_grad)")
        tabs = self._kernel_tables()
        verts = verts.contiguous()
        _lib.check_input(verts, "verts")
        B, J = mats.shape[0], mats.shape[1]
        vb, V = tuple(verts.shape[:2]) if verts.dim() == 3 else (0, 0)
        if verts.shape[2:] != (3,) or vb not in (1, B) or tabs["skin_idx"].shape != (V, N_SLOTS):
            raise RuntimeError("verts must be [1 or B, V, 3] with V = the skinned mesh's vertex count")
        out = torch.empty(B, V, 3, device=verts.device)
        _lib.kernels().gb_lbs_unskin_fwd(
            B, V, J, vb, mats, verts, template, tabs["skin_idx"], tabs["skin_w"], global_scaling, out)
        return out

    def unpose(self, poses: torch.Tensor, scales: torch.Tensor, verts: torch.Tensor):
        """lbs.py:256-271: poses [B,P], scales [B,S], posed verts [B,V,3] -> unposed verts [B,V,3]."""
        return self.unskin(self.skeleton(poses, scales), verts)

    def forward(self, poses: torch.Tensor, scales: torch.Tensor, verts_unposed: Optional[torch.Tensor] = None):
        """lbs.py:308-337: poses [B,P], scales [B,S], verts_unposed [1 or B, V, 3] (default: the rest mesh) -> [B,V,3]."""
        if verts_unposed is None:
            verts_unposed = self.mesh_vertices[None]
        return self.skin(self.skeleton(poses, scales), verts_unposed)


class LBSModule(nn.Module):
    """lbs.py:707-745: `lbs_fn` plus the skeleton scales, the template mesh and the global scaling."""

    def __init__(self, lbs_model_json, lbs_config_dict, lbs_template_verts, lbs_scale, global_scaling):
        super().__init__()
        self.lbs_fn = LinearBlendSkinning(lbs_model_json, lbs_config_dict)
        self.register_buffer("lbs_scale", torch.as_tensor(lbs_scale, dtype=torch.float32))
        self.register_buffer("lbs_template_verts", torch.as_tensor(lbs_template_verts, dtype=torch.float32))
        self.register_buffer("global_scaling", torch.as_tensor(global_scaling))

    def _gscale(self):
        g = self.global_scaling.to(torch.float32).reshape(-1)
        if g.numel() not in (1, 3):
            raise RuntimeError("global_scaling must hold 1 or 3 values")
        return g.expand(3).contiguous()

    def _template(self, template, V):
        """template as the kernel adds it ([V,3]), or None when it has a batch of its own and is added here."""
        if template.numel() == V * 3:
            _no_grad_input(template, "template")
            return template.reshape(V, 3).to(torch.float32).contiguous()
        return None

    def pose(self, verts_unposed: torch.Tensor, motion: torch.Tensor, template: Optional[torch.Tensor] = None):
        """global_scaling * lbs_fn(motion, lbs_scale, verts_unposed + template)  (lbs.py:725-731)."""
        if template is None:
            template = self.lbs_template_verts
        mats = self.lbs_fn.skeleton(motion, self.lbs_scale.reshape(1, -1).expand(motion.shape[0], -1))
        tpl = self._template(template, verts_unposed.shape[-2])
        if tpl is None:
            verts_unposed, tpl = verts_unposed + template, None
        return self.lbs_fn.skin(mats, verts_unposed, tpl, self._gscale())

    def unpose(self, verts: torch.Tensor, motion: torch.Tensor):
        """lbs_fn.unpose(motion, lbs_scale, verts / global_scaling) - lbs_template_verts  (lbs.py:733-739)."""
        mats = self.lbs_fn.skeleton(motion, self.lbs_scale.reshape(1, -1).expand(motion.shape[0], -1))
        tpl = self._template(self.lbs_template_verts, verts.shape[-2])
        out = self.lbs_fn.unskin(mats, verts, tpl, self._gscale())
        return out if tpl is not None else out - self.lbs_template_verts

    def template_pose(self, motion: torch.Tensor):
        """global_scaling * lbs_fn(motion, lbs_scale, lbs_template_verts)  (lbs.py:741-745)."""
        mats = self.lbs_fn.skeleton(motion, self.lbs_scale.reshape(1, -1).expand(motion.shape[0], -1))
        return self.lbs_fn.skin(mats, self.lbs_template_verts.reshape(1, -1, 3), None, self._gscale())
