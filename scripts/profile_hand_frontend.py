"""Time the hand-MVP front end: pose the mesh (LBSModule.pose), build the primitive base frames (make_postex +
compute_tbn) and the view cosine in UV (compute_view_cos + values_to_uv).

  ours   goliath_b200.lbs.LBSModule.pose + hand_mvp.prim_base_frames + hand_mvp.view_cos_uv, eager and replayed from a
         CUDA graph
  torch  the reference's formulation (ca_code/utils/lbs.py:340-429, quaternion.py:178-320, geom.py:308-397,515-520)
         restated below in plain torch ops and run on the same GPU

on a synthetic skeleton and a UV-gridded tube mesh whose sizes are printed, at B = 1 and B = 8.
Usage: python scripts/profile_hand_frontend.py [--iters N]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from goliath_b200 import _lib  # noqa: E402
from goliath_b200.hand_mvp import prim_base_frames, view_cos_uv  # noqa: E402
from goliath_b200.lbs import LBSModule  # noqa: E402

J, P, S = 40, 48, 8
NU, NV = 128, 96           # tube vertices around x along
UV, S_PRIM = 1024, 64      # texture size, primitives per side


def synthetic(seed=0):
    rng = np.random.default_rng(seed)
    parents = [-1] + [int(rng.integers(max(0, j - 4), j)) for j in range(1, J)]
    bones = [{"Name": "j%d" % j, "Parent": p, "PreRotation": (lambda q: (q / np.linalg.norm(q)).tolist())(rng.normal(size=4)),
              "TranslationOffset": rng.normal(size=3).tolist()} for j, p in enumerate(parents)]
    a, z = np.linspace(0, 2 * np.pi, NU), np.linspace(-6, 6, NV)
    verts = np.stack([3 * np.cos(a)[None].repeat(NV, 0), 3 * np.sin(a)[None].repeat(NV, 0), z[:, None].repeat(NU, 1)], -1)
    verts = verts.reshape(-1, 3).astype(np.float32)
    uu, vv = np.meshgrid(np.linspace(0, 1, NU), np.linspace(0, 1, NV))
    uvs = np.stack([uu, vv], -1).reshape(-1, 2).astype(np.float32)
    faces = np.asarray([t for r in range(NV - 1) for c in range(NU - 1) for i in [r * NU + c]
                        for t in ((i, i + 1, i + NU), (i + 1, i + NU + 1, i + NU))])
    # 8 influences per vertex, Gaussian falloff over the joints along the tube
    V = len(verts)
    counts = np.full(V, 8)
    sw = []
    for v in range(V):
        c = (v // NU) / (NV - 1) * (J - 1)
        ks = np.clip(np.round(c) + np.arange(-3, 5), 0, J - 1).astype(int)
        ks = np.unique(ks)
        ks = np.concatenate([ks, [k for k in range(J) if k not in ks][:8 - len(ks)]])
        w = np.exp(-((ks - c) ** 2) / 4.0)
        sw += [[int(k), float(x)] for k, x in zip(ks, w / w.sum())]
    model = {"Skeleton": {"Bones": bones},
             "SkinnedModel": {"RestPositions": verts.tolist(), "RestVertexNormals": verts.tolist(), "SkinningWeights": sw,
                              "SkinningOffsets": np.concatenate([[0], np.cumsum(counts)]).tolist(),
                              "Faces": {"Indices": faces.reshape(-1).tolist(), "TextureIndices": faces.reshape(-1).tolist()},
                              "TextureCoordinates": uvs.reshape(-1).tolist()}}
    transform = (rng.normal(size=(7 * J, P + S)) * (rng.uniform(size=(7 * J, P + S)) < 0.2) * 0.3).astype(np.float32)
    cfg = {"channel_names": list("abcdefg"), "limits": [], "transform": transform,
           "transform_offsets": np.zeros((1, 7 * J), np.float32), "nr_scaling_params": S, "nr_position_params": P}
    # per-primitive texel: centre of each of the 64 x 64 slab cells on the UV grid
    c = ((np.arange(S_PRIM) * (UV // S_PRIM) + UV // S_PRIM // 2) + 0.5) / UV
    fu, fv = np.meshgrid(c * (NU - 1), c * (NV - 1))
    ci, ri = np.floor(fu).astype(int), np.floor(fv).astype(int)
    lu, lv = fu - ci, fv - ri
    upper = lu + lv > 1
    face = 2 * (ri * (NU - 1) + ci) + upper
    bary = np.stack([np.where(upper, 1 - lv, 1 - lu - lv), np.where(upper, lu + lv - 1, lu), np.where(upper, 1 - lu, lv)], -1)
    return model, cfg, verts, faces, uvs, face, bary.astype(np.float32)


# ---------------------------------------------------------------- the reference's formulation, restated in torch
def q_mul(q, r):
    rows = [((1.0, 1.0, -1.0, 1.0), (3, 2, 1, 0)), ((-1.0, 1.0, 1.0, 1.0), (2, 3, 0, 1)),
            ((1.0, -1.0, 1.0, 1.0), (1, 0, 3, 2)), ((-1.0, -1.0, -1.0, 1.0), (0, 1, 2, 3))]
    return torch.stack([(q * torch.tensor([[list(s)]], dtype=q.dtype, device=q.device) * r[:, :, p]).sum(-1)
                        for s, p in rows], 2)


def q_rot(q, v):
    av = torch.cross(q[:, :, :3], v, dim=2)
    return v + 2 * (av * q[:, :, 3:4] + torch.cross(q[:, :, :3], av, dim=2))


def q_from_xyz(r):
    rm = r * torch.tensor([[[-0.5, 0.5, 0.5]]], dtype=r.dtype, device=r.device)
    c, s = torch.cos(rm), torch.sin(rm)
    return torch.stack([-s[..., 0] * (c[..., 1] * c[..., 2]) - c[..., 0] * (s[..., 1] * s[..., 2]),
                        c[..., 0] * (s[..., 1] * c[..., 2]) - s[..., 0] * (c[..., 1] * s[..., 2]),
                        c[..., 0] * (c[..., 1] * s[..., 2]) + s[..., 0] * (s[..., 1] * c[..., 2]),
                        c[..., 0] * (c[..., 1] * c[..., 2]) - s[..., 0] * (s[..., 1] * s[..., 2])], 2)


def torch_front(m, motion, campos, vi, vt, vidx, vtidx, bary):
    f = m.lbs_fn
    B = motion.shape[0]
    params = f.param_transform.transform.mm(torch.cat([motion, m.lbs_scale.expand(B, -1)], 1).t()).t()
    jp = (params + f.param_transform.transform_offsets).view(B, -1, 7)
    lt = jp[:, :, 0:3] + f.joint_offset[None]
    lr = q_mul(f.joint_rotation[None].expand(B, -1, -1), q_from_xyz(jp[:, :, 3:6]))
    ls = torch.pow(torch.tensor([2.0], device=motion.device), jp[:, :, 6:7])
    state = []
    for j, p in enumerate(f.joint_parents):
        if int(p) != -1:
            ps = state[p]
            gr = q_mul(ps[:, :, 3:7], lr[:, j:j + 1])
            gt = q_rot(ps[:, :, 3:7], lt[:, j:j + 1] * ps[:, :, 7:8]) + ps[:, :, 0:3]
            state.append(torch.cat((gt, gr, ps[:, :, 7:8] * ls[:, j:j + 1]), 2))
        else:
            state.append(torch.cat((lt[:, j], lr[:, j], ls[:, j]), 1).view(B, 1, 8))
    st = torch.cat(state, 1)
    bind = f.bind_state
    br = bind[:, :, 3:7] * torch.tensor([-1.0, -1, -1, 1], device=bind.device) / (bind[:, :, 3:7] ** 2).sum(2, keepdim=True)
    bs = bind[:, :, 7:8].reciprocal()
    bt = q_rot(br, -bind[:, :, 0:3]) * bs
    tr, ts = q_mul(st[:, :, 3:7], br.expand(B, -1, -1)), st[:, :, 7:8] * bs
    tt = q_rot(st[:, :, 3:7], bt * st[:, :, 7:8]) + st[:, :, 0:3]
    x, y, z, w = (tr[:, :, i] for i in range(4))
    mat = torch.stack((torch.stack((1 - 2 * (y * y + z * z), 2 * (x * y + z * w), 2 * (x * z - y * w)), 2) * ts,
                       torch.stack((2 * (x * y - z * w), 1 - 2 * (x * x + z * z), 2 * (y * z + x * w)), 2) * ts,
                       torch.stack((2 * (x * z + y * w), 2 * (y * z - x * w), 1 - 2 * (x * x + y * y)), 2) * ts, tt), 3)
    verts = torch.zeros_like(m.lbs_template_verts) + m.lbs_template_verts
    vs = torch.matmul(mat[:, f.skin_indices], torch.cat((verts, torch.ones_like(verts[:, :, :1])), 2)[:, :, None, :, None])
    geom = (vs * f.skin_weights[None, :, :, None, None]).sum(2).squeeze(3) * m.global_scaling
    post = (bary[None, :, :, 0, None] * geom[:, vidx[:, :, 0]] + bary[None, :, :, 1, None] * geom[:, vidx[:, :, 1]]
            + bary[None, :, :, 2, None] * geom[:, vidx[:, :, 2]]).permute(0, 3, 1, 2)
    v0, v1, v2 = geom[:, vidx[..., 0]], geom[:, vidx[..., 1]], geom[:, vidx[..., 2]]
    t0, t1, t2 = vt[vtidx[..., 0]], vt[vtidx[..., 1]], vt[vtidx[..., 2]]
    v01, v02, t01, t02 = v1 - v0, v2 - v0, t1 - t0, t2 - t0
    fdet = 1.0 / (t01[None, ..., 0] * t02[None, ..., 1] - t01[None, ..., 1] * t02[None, ..., 0])
    tan = F.normalize(fdet[..., None] * (v01 * t02[None, ..., 1:2] - v02 * t01[None, ..., 1:2]), dim=-1)
    nrm = F.normalize(torch.cross(v01, v02, dim=-1), dim=-1)
    bit = F.normalize(torch.cross(tan, nrm, dim=-1), dim=-1)
    rot = torch.stack((tan, bit, nrm), -2).reshape(B, -1, 3, 3).permute(0, 1, 3, 2).contiguous()
    pts = geom[:, vi]
    fn = torch.cross(pts[:, :, 1] - pts[:, :, 0], pts[:, :, 2] - pts[:, :, 0], dim=-1)
    fn = fn / fn.norm(dim=-1, keepdim=True).clamp(min=1e-5)
    fn = fn[:, :, None].expand(-1, -1, 3, -1).reshape(B, -1, 3)
    vn = torch.zeros_like(geom)
    for k in range(3):
        vn[..., k].scatter_add_(1, vi.reshape(1, -1).expand(B, -1), fn[..., k])
    vn = F.normalize(vn / vn.norm(dim=-1, keepdim=True).clamp(min=1e-5), dim=-1)
    vc = torch.einsum("bnd,bnd->bn", vn, F.normalize(geom - campos[:, None], dim=-1))[..., None]
    mask = torch.all(vidx != -1, dim=-1)
    flat = torch.sum(vc[:, vidx[mask]].permute(0, 3, 1, 2) * bary[mask], dim=-1)
    uv = torch.zeros(B, 1, S_PRIM, S_PRIM, device=geom.device, dtype=geom.dtype)
    uv[:, :, mask] = flat
    return geom, post.permute(0, 2, 3, 1).reshape(B, -1, 3), rot, uv


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    model, cfg, verts, faces, uvs, face, bary = synthetic()
    print("GPU: %s" % q)
    print("skeleton: %d joints, P=%d, S=%d; mesh: %d vertices, %d faces; %d x %d primitive texels"
          % (J, P, S, len(verts), len(faces), S_PRIM, S_PRIM))
    m = LBSModule(model, cfg, np.zeros((1, len(verts), 3), np.float32), np.zeros(S, np.float32), [10.0, 10.0, 10.0]).to(dev)
    vi = torch.as_tensor(faces, device=dev)
    vt = torch.as_tensor(uvs, device=dev)
    fidx = torch.as_tensor(face, device=dev)
    vidx64, bary_t = vi[fidx], torch.as_tensor(bary, device=dev)
    vidx, vtidx = vidx64.to(torch.int32), vidx64.to(torch.int32)
    vi32 = vi.to(torch.int32)
    L = _lib.lib()
    for B in (1, 8):
        motion = 0.3 * torch.randn(B, P, device=dev, generator=torch.Generator(device=dev).manual_seed(B))
        campos = torch.tensor([[40.0, 5.0, 3.0]], device=dev).expand(B, -1).contiguous()

        def ours():
            geom = m.pose(torch.zeros_like(m.lbs_template_verts), motion)
            pos, rot = prim_base_frames(geom, vt, vidx, vtidx, bary_t)
            return geom, pos, rot, view_cos_uv(geom, vi32, campos, vidx, bary_t)

        def ref():
            return torch_front(m, motion, campos, vi, vt, vidx64, vidx64, bary_t)

        with torch.no_grad():
            L.gb_launch_count_reset()
            ours()
            launches = L.gb_launch_count()
            t_ours, t_ref = timed(ours, args.iters), timed(ref, max(5, args.iters // 10))
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                ours()
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                ours()
            t_graph = timed(g.replay, args.iters)
        print("B=%d  ours eager %.3f ms, graph replay %.3f ms, %d gb launches / call;  torch formulation %.3f ms;"
              "" % (B, t_ours, t_graph, launches, t_ref))


if __name__ == "__main__":
    main()
