"""Seeded synthetic skinned models for the LBS / hand front-end tests and tests/golden/make_lbs_golden.py: the model
json and parameter config dicts in the reference asset loader's layout, a UV-gridded tube mesh with its index images,
and a weight recipe for the decoders.  Everything is rebuilt from seeds, so only outputs are stored in the fixture."""
import numpy as np
import torch

SKELETONS = ("tree24", "chain160", "star300")


def _parents(kind, rng):
    if kind == "tree24":    # two roots: joint 0 (-1) and joint 9, whose Parent is above J (the `Parent > J` rule)
        p = [-1] + [int(rng.integers(0, j)) for j in range(1, 24)]
        p[9] = 1000
        return p
    if kind == "chain160":  # 160 levels
        return [-1] + list(range(159))
    if kind == "star300":   # one root, one level of 300 children
        return [-1] + [0] * 300
    raise KeyError(kind)


def skinned_model(kind, seed, verts=None, faces=None, tex_faces=None, uvs=None, n_verts=500):
    """(model_json, lbs_config_dict, template [V,3], skeleton scales [S]) for skeleton `kind`."""
    rng = np.random.default_rng(seed)
    parents = _parents(kind, rng)
    J = len(parents)
    step = 0.3 if kind == "chain160" else 1.0     # keeps the 160-long chain's reach moderate
    bones = []
    for j, p in enumerate(parents):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        bones.append({"Name": "j%d" % j, "Parent": p, "PreRotation": q.tolist(),
                      "TranslationOffset": (rng.normal(size=3) * step).tolist()})
    if verts is None:
        verts = rng.normal(size=(n_verts, 3)) * 2.0
        faces = np.stack([np.arange(n_verts - 2), np.arange(1, n_verts - 1), np.arange(2, n_verts)], 1)
        tex_faces, uvs = faces, rng.uniform(size=(n_verts, 2))
    V = len(verts)
    counts = rng.integers(1, 9, size=V)           # 1..8 influences, ragged offsets
    offsets = np.concatenate([[0], np.cumsum(counts)])
    sw = []
    for v in range(V):
        idx = rng.choice(J, size=counts[v], replace=False)
        w = rng.uniform(0.1, 1.0, size=counts[v])
        sw += [[int(i), float(x)] for i, x in zip(idx, w / w.sum())]
    model = {"Skeleton": {"Bones": bones},
             "SkinnedModel": {"RestPositions": np.asarray(verts, np.float32).tolist(),
                              "RestVertexNormals": rng.normal(size=(V, 3)).astype(np.float32).tolist(),
                              "SkinningWeights": sw, "SkinningOffsets": offsets.tolist(),
                              "Faces": {"Indices": np.asarray(faces).reshape(-1).tolist(),
                                        "TextureIndices": np.asarray(tex_faces).reshape(-1).tolist()},
                              "TextureCoordinates": np.asarray(uvs, np.float32).reshape(-1).tolist()}}
    P, S = 12, 4
    transform = (rng.normal(size=(7 * J, P + S)) * (rng.uniform(size=(7 * J, P + S)) < 0.3)).astype(np.float32)
    transform[6::7] *= 0.05 if kind == "chain160" else 0.3   # scale channels: 2^s stays tame along the chain
    transform[0::7] *= step
    cfg = {"channel_names": ["tx", "ty", "tz", "rx", "ry", "rz", "sc"], "limits": [],
           "transform": transform, "transform_offsets": (rng.normal(size=(1, 7 * J)) * 0.1).astype(np.float32),
           "nr_scaling_params": S, "nr_position_params": P}
    template = (rng.normal(size=(V, 3)) * 0.1).astype(np.float32)
    scales = (rng.normal(size=S) * 0.2).astype(np.float32)
    return model, cfg, template, scales


def motion(B, seed, P=12):
    return torch.randn(B, P, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------ tube mesh
TUBE_NU, TUBE_NV = 40, 30   # vertices around x along


def tube():
    """A tube (radius 3, length 12) with a UV grid over [0.05, 0.95]^2; the UV seam is a column of its own.  Faces:
    the grid's triangles, then one face with a degenerate (collinear) UV triangle, then a copy of face 0 as the last
    face (the one a -1 face index selects)."""
    nu, nv = TUBE_NU, TUBE_NV
    a = np.linspace(0, 2 * np.pi, nu)             # the last column repeats the first position (the seam)
    z = np.linspace(-6, 6, nv)
    verts = np.stack([3 * np.cos(a)[None].repeat(nv, 0), 3 * np.sin(a)[None].repeat(nv, 0), z[:, None].repeat(nu, 1)],
                     -1).reshape(-1, 3)
    uu, vv = np.meshgrid(np.linspace(0.05, 0.95, nu), np.linspace(0.05, 0.95, nv))
    uvs = np.stack([uu, vv], -1).reshape(-1, 2)
    faces = []
    for r in range(nv - 1):
        for c in range(nu - 1):
            i = r * nu + c
            faces += [(i, i + 1, i + nu), (i + 1, i + nu + 1, i + nu)]
    faces = np.asarray(faces)
    tex = faces.copy()
    degenerate_face = len(faces)
    faces = np.concatenate([faces, faces[[nu + 3]], faces[[0]]])
    tex = np.concatenate([tex, [[tex[nu + 3, 0], tex[nu + 3, 0], tex[nu + 3, 1]]], tex[[0]]])
    return verts.astype(np.float32), faces, tex, uvs.astype(np.float32), degenerate_face


class TubeGeometry:
    """Holder with the part of the reference's GeometryModule that `init_primitives` reads: vi, vti, vt and
    render_index_images(uv_size, impaint=True), here rasterised analytically on the tube's UV grid."""

    def __init__(self, dtype=torch.float32):
        verts, faces, tex, uvs, self.degenerate_face = tube()
        self.vi = torch.as_tensor(faces, dtype=torch.int64)
        self.vti = torch.as_tensor(tex, dtype=torch.int64)
        self.vt = torch.as_tensor(uvs).to(dtype)

    def render_index_images(self, uv_size, flip_uv=False, impaint=False):
        nu, nv = TUBE_NU, TUBE_NV
        c = (np.arange(uv_size) + 0.5) / uv_size
        fu = (c[None, :] - 0.05) / 0.9 * (nu - 1)
        fv = (c[:, None] - 0.05) / 0.9 * (nv - 1)
        fu, fv = np.broadcast_to(fu, (uv_size, uv_size)), np.broadcast_to(fv, (uv_size, uv_size))
        covered = (fu >= 0) & (fu < nu - 1) & (fv >= 0) & (fv < nv - 1)
        ci, ri = np.clip(np.floor(fu), 0, nu - 2).astype(np.int64), np.clip(np.floor(fv), 0, nv - 2).astype(np.int64)
        lu, lv = np.clip(fu - ci, 0, 1), np.clip(fv - ri, 0, 1)
        upper = lu + lv > 1.0
        face = 2 * (ri * (nu - 1) + ci) + upper
        # lower triangle (i, i+1, i+nu): (1-u-v, u, v); upper (i+1, i+nu+1, i+nu): (1-v, u+v-1, 1-u)
        bary = np.stack([np.where(upper, 1 - lv, 1 - lu - lv), np.where(upper, lu + lv - 1, lu),
                         np.where(upper, 1 - lu, lv)], -1)
        face = np.where(covered, face, -1)
        face[uv_size // 2 + 8, uv_size // 2 + 8] = self.degenerate_face  # one texel sampled by init_primitives
        index = self.vi.numpy()[face]
        index[face < 0] = -1
        return (torch.as_tensor(index), torch.as_tensor(face), torch.as_tensor(bary.astype(np.float32)).to(self.vt.dtype))


def tube_model(seed):
    verts, faces, tex, uvs, _ = tube()
    return skinned_model("tree24", seed, verts=verts, faces=faces, tex_faces=tex, uvs=uvs)


CAMPOS = torch.tensor([[40.0, 5.0, 3.0], [-10.0, 30.0, -20.0]])


def with_negative_indices(vidx):
    """a copy of an [S,S,3] vertex index image with -1 entries: one corner of five texels, and one whole texel"""
    vidx = vidx.clone()
    vidx[0, :5, 0] = -1
    vidx[3, 7] = -1
    return vidx


def alpha_sample(n, k=8000):
    return torch.as_tensor(np.random.default_rng(23).integers(0, n, size=k))


# ------------------------------------------------------------------------------------------ decoder weights
def init_weights(module, seed):
    """Overwrite every parameter, in name order, from one generator: weight_v ~ N(0,1), weight_g = sqrt(fan-out)
    (1 + 0.1 N), bias ~ 0.1 N.  Works for the reference's modules and ours alike (same names and shapes)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(module.named_parameters()):
            r = torch.randn(p.shape, generator=g, dtype=torch.float32)
            if name.endswith("weight_g"):
                r = (1.0 + 0.1 * r) * float(np.sqrt(p.numel()))
            elif name.endswith("bias"):
                r = 0.1 * r
            p.copy_(r.to(p.dtype))
