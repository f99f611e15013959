"""Seeded assets, configuration and parameters of the hand avatar's frame (`hand_mvp.AutoEncoder`), shared by
tests/golden/make_hand_frame_golden.py, the CPU and GPU tests and scripts/profile_hand_frame.py.

The mesh is lbs_recipe's UV-gridded tube (radius 3, length 12, x10 in the posed frame) skinned by a 24-joint
skeleton with 12 pose parameters (n_pose_dims = 6).  Its four plain UV images come from lbs_recipe.TubeGeometry;
the barycentric image `render_index_images(1024, impaint=True)` returns is inpainted here in numpy with the
reference's rule (every uncovered texel within 100 texels copies its nearest covered texel), and its face image is
the plain one, as that call returns it.  The frame's inputs are frozen in the golden file."""
import numpy as np
import torch

import lbs_recipe as R

CAMERAS = ["401033", "400870", "410244", "402100"]   # unsorted on purpose: CalV5 sorts, LearnableBlur does not
IDENTITY = "400870"
BATCH_CAMERAS = [IDENTITY, "410244"]                 # the identity-calibration camera and a grey ("41...") camera
H, W = 64, 96                                        # render size of the fixture
MODES = ("eval", "train0", "train")                  # eval; training before primposstart; training after it
ITERATION = {"eval": None, "train0": 0, "train": 5000}


class Assets(dict):
    """the reference's asset object: attribute access and `"key" in assets`"""

    __getattr__ = dict.__getitem__


def inpaint_nearest(valid, image, threshold=100.0):
    """index_image_impaint's rule (ca_code/utils/geom.py:145-194) on a [S,S] validity mask: every invalid texel
    closer than `threshold` to a valid one takes the value of its nearest valid texel"""
    from scipy.spatial import cKDTree

    vij, iij = np.argwhere(valid), np.argwhere(~valid)
    dist, idx = cKDTree(vij).query(iij)
    keep = dist < threshold
    out = image.copy()
    src, dst = vij[idx[keep]], iij[keep]
    out[dst[:, 0], dst[:, 1]] = image[src[:, 0], src[:, 1]]
    return out


def assets():
    verts, faces, tex, uvs, _ = R.tube()
    model, cfg, _, scales = R.skinned_model("tree24", 7, verts=verts, faces=faces, tex_faces=tex, uvs=uvs)
    index, face, bary = (t.numpy().copy() for t in R.TubeGeometry().render_index_images(1024))
    # TubeGeometry plants its degenerate UV triangle at a texel init_primitives samples (a NaN frame, which the
    # front-end tests cover); the frame's fixture takes the neighbouring texel's face instead
    c = np.argwhere(face == R.tube()[4])[0]
    face[c[0], c[1]], bary[c[0], c[1]] = face[c[0], c[1] + 1], bary[c[0], c[1] + 1]
    index[c[0], c[1]] = faces[face[c[0], c[1]]]
    valid = index[..., 0] != -1
    return Assets(
        topology=Assets(vi=torch.as_tensor(faces), vt=torch.as_tensor(uvs), vti=torch.as_tensor(tex),
                        v2uv=torch.arange(len(verts))[:, None]),
        lbs_model_json=model, lbs_config_dict=cfg, template_mesh_unscaled=verts.astype(np.float32),
        skeleton_scales=scales, camera_ids=list(CAMERAS),
        index_image=torch.as_tensor(index), bary_image=torch.as_tensor(bary),
        face_index_image=torch.as_tensor(face), valid_mask=torch.as_tensor(valid[..., None]),
        face_index_image_impaint=torch.as_tensor(face),
        bary_image_impaint=torch.as_tensor(inpaint_nearest(valid, bary)))


def config(h=H, w=W):
    """hand_mvp_example.yml's model section at the fixture's size, with the synthetic skeleton's n_pose_dims"""
    return {"n_embs": 64, "image_height": h, "image_width": w, "cal": {"identity_camera": IDENTITY},
            "learn_blur": True, "n_pose_dims": 6}


def seeded_fill(module, seed=2025):
    """every parameter by name from one generator, rounded to fp32: weight_v ~ N(0, 2/fan), weight_g in [0.5, 1.5),
    the alpha slab's untied bias 150 + 50 N (an opacity of about one half per primitive crossed at dt = 1 / 2000),
    the calibration rows w = 1 + 0.1 N / b = 0.05 N, LearnableBlur's logits N(0, 1), every other parameter 0.05 N"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(module.named_parameters()):
            f64 = dict(generator=g, dtype=torch.float64)
            if name.endswith("weight_v"):
                v = torch.randn(p.shape, **f64) * (2.0 / max(1, p[0].numel())) ** 0.5
            elif name.endswith("weight_g"):
                v = 0.5 + torch.rand(p.shape, **f64)
            elif name.startswith("geomdecoder.alphadecoder.texbranch.6.bias"):
                v = 150.0 + 50.0 * torch.randn(p.shape, **f64)
            elif name.endswith("holder.params"):
                v = torch.cat([1.0 + 0.1 * torch.randn(p.shape[0], 3, **f64), 0.05 * torch.randn(p.shape[0], 3, **f64)],
                              1)
            elif name.endswith("weights_raw"):
                v = torch.randn(p.shape, **f64)
            else:
                v = 0.05 * torch.randn(p.shape, **f64)
            p.copy_(v.float().to(p.dtype))
    return module


def side_cameras(points, h=H, w=W):
    """K [B,3,3], Rt [B,3,4], campos [B,3] of cameras looking at each item's points across the tube's axis (image x
    along world z), camera b turned by 0.4 b radians about z, framing the points"""
    B = points.shape[0]
    c = points.mean(1)
    r = (points - c[:, None]).norm(dim=-1).max(1).values
    Rs, ts = [], []
    for b in range(B):
        a = 0.4 * b
        rz = torch.tensor([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]],
                          dtype=points.dtype)
        R0 = torch.tensor([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]], dtype=points.dtype) @ rz.T
        Rs.append(R0)
        ts.append(-(R0 @ c[b]) + torch.tensor([0.0, 0.0, 2.2], dtype=points.dtype) * r[b])
    Rm, t = torch.stack(Rs), torch.stack(ts)
    Rt = torch.cat([Rm, t[:, :, None]], 2)
    f = 0.55 * w * 2.2
    K = torch.tensor([[f, 0.0, w / 2.0], [0.0, f, h / 2.0], [0.0, 0.0, 1.0]], dtype=points.dtype).expand(B, 3, 3)
    campos = -(Rm.transpose(1, 2) @ t[:, :, None])[..., 0]
    return K.contiguous(), Rt, campos


def pose_inputs(batch=2, seed=7):
    g = torch.Generator().manual_seed(seed)
    return 0.05 * torch.randn(batch, 12, generator=g), torch.rand(batch, 1, 128, 128, generator=g)


def background(batch=2, h=H, w=W, seed=9):
    return 40.0 + 120.0 * torch.rand(batch, 3, h, w, generator=torch.Generator().manual_seed(seed))


def raydirs(campos, camrot, focal, princpt, h, w, volradius):
    """compute_raydirs on the integer pixel grid: the reference's torch formula (extensions/utils/utils.py:127-143)
    with the CUDA op's viewpos / volradius (utils_kernel.cu)"""
    viewpos = campos / volradius
    y, x = torch.meshgrid(torch.arange(h, dtype=campos.dtype), torch.arange(w, dtype=campos.dtype), indexing="ij")
    pix = torch.stack([x, y], -1)[None]
    raypos = viewpos[:, None, None, :].expand(-1, h, w, -1).contiguous()
    raydir = (pix - princpt[:, None, None, :]) / focal[:, None, None, :]
    raydir = torch.cat([raydir, torch.ones_like(raydir[..., :1])], -1)
    raydir = torch.sum(camrot[:, None, None, :, :] * raydir[..., :, None], dim=-2)
    raydir = raydir / torch.sqrt(torch.sum(raydir ** 2, dim=-1, keepdim=True))
    t1 = (-1.0 - viewpos[:, None, None, :]) / raydir
    t2 = (1.0 - viewpos[:, None, None, :]) / raydir
    tmin = torch.max(torch.min(t1[..., 0], t2[..., 0]),
                     torch.max(torch.min(t1[..., 1], t2[..., 1]), torch.min(t1[..., 2], t2[..., 2]))).clamp(min=0.0)
    tmax = torch.min(torch.max(t1[..., 0], t2[..., 0]),
                     torch.min(torch.max(t1[..., 1], t2[..., 1]), torch.max(t1[..., 2], t2[..., 2])))
    return raypos, raydir, torch.stack([tmin, tmax], -1)


def summarise(t):
    f = t.detach().double().reshape(-1).cpu()
    idx = torch.linspace(0, f.numel() - 1, 256, dtype=torch.float64).long()
    return np.concatenate([[f.mean().item(), f.std().item(), f.abs().max().item(), float(f.numel())], f[idx].numpy()])


def nrel_summary(a, b):
    """norm-wise relative difference of two summaries (statistics and samples, not the count)"""
    a, b = np.delete(a, 3), np.delete(b, 3)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


PRE_MODULES = ("poseencoder", "geomdecoder.transdecoder", "geomdecoder.alphadecoder", "rgbdecoder")
PRIM_KEYS = ("primpos", "primrot", "primscale", "primrgba")


def grad_param_names(model):
    """the first and last parameter (by name) of each decoder module"""
    names = sorted(n for n, _ in model.named_parameters())
    out = []
    for m in PRE_MODULES:
        sub = [n for n in names if n.startswith(m + ".")]
        out += sorted({sub[0], sub[-1]})
    return out


def functional_weights(shapes, seed=31):
    """the seeded linear functional on the per-primitive outputs: one fp64 N(0,1) weight per element"""
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(shapes[k], generator=g, dtype=torch.float64) for k in PRIM_KEYS}


def cotangents(rgb_shape, alpha_shape, seed=77):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(rgb_shape, generator=g, dtype=torch.float64),
            torch.randn(alpha_shape, generator=g, dtype=torch.float64))
