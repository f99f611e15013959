"""Seeded assets, configuration, parameters and inputs of the body avatar's frame (`mesh_vae.AutoEncoder`), shared by
tests/golden/make_body_frame_golden.py, the CPU and GPU tests and scripts/profile_body_frame.py, and plain-torch
restatements (any device, any dtype) of the frame's small pieces: geom.depth_discontuity_mask, CameraPixelBias,
CalV5 and LearnableBlur.

The mesh is the UV-gridded sheet of body_texture_restate.uv_mesh, skinned by a lbs_recipe skeleton with
n_pose_dims = P - 6; the UV index images are that sheet's, given as assets (this project does not rasterise them)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import body_texture_restate as bt
import lbs_recipe as R
import seams_restate as sr

CAMERAS = ["401033", "400870", "410244", "402100"]   # unsorted on purpose: CalV5 sorts, LearnableBlur does not
IDENTITY = "400870"
BATCH_CAMERAS = ["410244", "401033"]                 # a grey ("41...") and a colour camera
H, W, DS = 128, 96, 8                                # render size of the fixture
GLOBAL_SCALING = 1000.0                              # depth in the thousands, as the threshold 40 expects


class Assets(dict):
    """the reference's asset object: attribute access and `"key" in assets`"""

    __getattr__ = dict.__getitem__


def config(h=H, w=W, ds=DS):
    """mesh_vae_example.yml's model section, with n_pose_dims = P - 6 of the synthetic skeleton and the render size"""
    return {
        "encoder": {"n_embs": 1024},
        "encoder_face": {"n_embs": 256},
        "decoder": {"init_uv_size": 64, "n_init_channels": 64, "n_min_channels": 4, "n_pose_dims": 6,
                    "n_pose_enc_channels": 16, "n_embs": 1024, "n_embs_enc_channels": 32, "n_face_embs": 256,
                    "uv_size": 1024},
        "decoder_view": {"net_uv_size": 1024},
        "upscale_net": {"n_ftrs": 4},
        "shadow_net": {"uv_size": 2048, "shadow_size": 256, "n_dims": 4},
        "renderer": Assets(image_height=h, image_width=w, depth_disc_ksize=3),
        "cal": {"identity_camera": IDENTITY},
        "pixel_cal": {"image_height": h, "image_width": w, "ds_rate": ds},
        "learn_blur": True,
    }


def assets():
    from oracle.mesh_vae_oracle import synthetic_masks

    vi, verts0, idx_img, bary_img = bt.uv_mesh()
    V = verts0.shape[0]
    vt = verts0[:, :2].float()
    model, cfg, _, scales = R.skinned_model("tree24", 61, verts=verts0.numpy(), faces=vi.numpy(),
                                            tex_faces=vi.numpy(), uvs=vt.numpy())
    rng = np.random.default_rng(29)
    yy, xx = np.mgrid[0:1024, 0:1024]
    face_mask = ((yy >= 600) & (yy < 900) & (xx >= 100) & (xx < 400)).astype(np.float32)
    face_index = np.where(idx_img[..., 0].numpy() >= 0, rng.integers(0, vi.shape[0], (1024, 1024)), -1)
    a = Assets(
        topology=Assets(vi=vi, vt=vt, vti=vi.clone(), v2uv=torch.arange(V)[:, None]),
        lbs_model_json=model, lbs_config_dict=cfg,
        template_mesh=(verts0 - 0.5).float().numpy(), skeleton_scales=scales,
        global_scaling=np.full(3, GLOBAL_SCALING, np.float32),
        seam_data_1024=sr.synthetic_seams(1024), seam_data_2048=sr.synthetic_seams(2048, n_pairs=16000, seed=5),
        color_mean=(100.0 + 20.0 * rng.standard_normal((3, 512, 512))).astype(np.float32),
        mouth_eyes_mask_geom=(rng.random(V) < 0.2).astype(np.float32),
        face_mask=face_mask,
        ambient_occlusion_mean=(0.5 + 0.1 * rng.standard_normal((1, 512, 512))).astype(np.float32),
        camera_ids=list(CAMERAS),
        index_image=idx_img, bary_image=bary_img, face_index_image=torch.as_tensor(face_index, dtype=torch.int64),
        valid_mask=idx_img[..., :1] != -1,
        **synthetic_masks(n_pose_dims=6, size=64, seed=11))
    return a


def seeded_fill(module, seed=2024):
    """every parameter by name from one generator, rounded to fp32: weight_v ~ N(0, 2/fan), weight_g in [0.5, 1.5),
    the calibration rows w = 1 + 0.1 N / b = 0.05 N, LearnableBlur's logits N(0, 1), the pixel bias 0.05 N, every
    other parameter 0.05 N"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(module.named_parameters()):
            f64 = dict(generator=g, dtype=torch.float64)
            if name.endswith("weight_v"):
                v = torch.randn(p.shape, **f64) * (2.0 / max(1, p[0].numel())) ** 0.5
            elif name.endswith("weight_g"):
                v = 0.5 + torch.rand(p.shape, **f64)
            elif name.endswith("holder.params"):
                v = torch.cat([1.0 + 0.1 * torch.randn(p.shape[0], 3, **f64), 0.05 * torch.randn(p.shape[0], 3, **f64)], 1)
            elif name.endswith("weights_raw"):
                v = torch.randn(p.shape, **f64)
            else:
                v = 0.05 * torch.randn(p.shape, **f64)
            p.copy_(v.float().to(p.dtype))
    return module


def look_at(points, h, w):
    """K [B,3,3], Rt [B,3,4] and the camera position [B,3] of a camera on -z of each item's points, framing them"""
    c = points.mean(1)
    r = (points - c[:, None]).norm(dim=-1).max(1).values
    B = points.shape[0]
    t = torch.stack([-c[:, 0], -c[:, 1], -c[:, 2] + 2.5 * r], -1)
    Rt = torch.cat([torch.eye(3, dtype=points.dtype).expand(B, 3, 3), t[:, :, None]], 2)
    f = 0.9 * min(h, w)
    K = torch.tensor([[f, 0.0, w / 2.0], [0.0, f, h / 2.0], [0.0, 0.0, 1.0]], dtype=points.dtype).expand(B, 3, 3)
    return K.contiguous(), Rt, -t


def inputs(model, batch=2, h=H, w=W, seed=7):
    """pose [B,P], campos, registration_vertices [B,V,3], ambient_occlusion [B,1,256,256], K, Rt, camera_id (fp32,
    from seeds; the camera frames the template posed by `model.lbs_fn`, which runs here in torch on the CPU)"""
    g = torch.Generator().manual_seed(seed)
    P = model.lbs_fn.lbs_fn.param_transform.transform.shape[1] - model.lbs_fn.lbs_scale.shape[-1]
    pose = 0.3 * torch.randn(batch, P, generator=g)
    V = model.lbs_fn.lbs_template_verts.shape[0]
    delta = 0.01 * torch.randn(batch, V, 3, generator=g)
    with torch.no_grad():
        lbs = model.lbs_fn
        posed = lbs.lbs_fn(pose, lbs.lbs_scale.expand(batch, -1), delta + lbs.lbs_template_verts) * lbs.global_scaling
    reg = posed + 0.5 * torch.randn(batch, V, 3, generator=g)
    K, Rt, campos = look_at(posed, h, w)
    ao = ambient_occlusion(batch, seed + 1)
    cams = (BATCH_CAMERAS * math.ceil(batch / 2))[:batch]
    return {"pose": pose, "campos": campos, "registration_vertices": reg, "ambient_occlusion": ao, "K": K, "Rt": Rt,
            "camera_id": cams}


def ambient_occlusion(batch, seed=8):
    return torch.rand(batch, 1, 256, 256, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------ restatements
def depth_disc_mask(depth, threshold=40.0, pool_ksize=3):
    """geom.py:768-794 in depth's dtype; also returns the gradient norm"""
    k = torch.tensor([[[[-1, 0, 1], [-2, 0, 2], [-1, 0, 1]]], [[[-1, -2, -1], [0, 0, 0], [1, 2, 1]]]],
                     dtype=depth.dtype, device=depth.device)
    norm = torch.norm(F.conv2d(depth, k, bias=None, padding=1), dim=1)[:, None]
    m = F.avg_pool2d((norm > threshold).to(depth.dtype), pool_ksize, stride=1, padding=pool_ksize // 2) > 0.0
    return m, norm


def pixel_bias(rgb, bias, idx, h, w):
    """mesh_vae.py:65-69 then :339"""
    return rgb + F.interpolate(bias[idx], size=(h, w), mode="bilinear")


def gaussian_blur(img, k):
    """torchvision's gaussian_blur with its default sigma and reflect padding"""
    sigma = 0.3 * ((k - 1) * 0.5 - 1) + 0.8
    x = torch.linspace(-(k - 1) * 0.5, (k - 1) * 0.5, k, dtype=img.dtype, device=img.device)
    k1 = torch.exp(-0.5 * (x / sigma) ** 2)
    k1 = k1 / k1.sum()
    k2 = (k1[:, None] * k1[None, :]).expand(img.shape[1], 1, k, k)
    return F.conv2d(F.pad(img, [k // 2] * 4, mode="reflect"), k2, groups=img.shape[1])


def cal_v5(image, params, idxs, identity_idx, grey_idxs, training=False, gs=1.0, col=0.1):
    """color_cal.py:211-241 (the per-item loop and the training-mode scale hook)"""
    rows = params[idxs]
    outs, scales = [], []
    for i in range(idxs.shape[0]):
        n, img = int(idxs[i]), image[i:i + 1]
        if n == identity_idx:
            outs.append(img)
            scales.append(1.0)
            continue
        w, b = rows[i, :3], rows[i, 3:]
        if n in grey_idxs:
            outs.append((img * w[None, :, None, None]).sum(1, keepdim=True).expand(-1, 3, -1, -1) + b.sum())
        else:
            outs.append(img * w[None, :, None, None] + b[None, :, None, None])
        scales.append(gs if n in grey_idxs else col)
    if training and rows.requires_grad:
        s = torch.tensor(scales, dtype=rows.dtype, device=rows.device)
        rows.register_hook(lambda g: g * s[:, None])
    return torch.cat(outs)


def learn_blur(img, weights_raw, idxs):
    """dof_cal.py:44-56"""
    wts = torch.softmax(weights_raw[idxs], dim=-1).reshape(img.shape[0], 3, 1, 1, 1)
    return wts[:, 0] * img + wts[:, 1] * gaussian_blur(img, 3) + wts[:, 2] * gaussian_blur(img, 7)
