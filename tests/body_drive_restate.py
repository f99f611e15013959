"""Seeded assets, configuration and inputs of the drivable body avatar (`mesh_vae_drivable.AutoEncoder`), shared by
tests/golden/make_body_drive_golden.py, the CPU and GPU tests and scripts/profile_body_drive.py, and fp64 torch
restatements (any device, any dtype) of the three kernels of csrc/body_drive.cu.

Built on tests/body_frame_restate.py: the same sheet, skeleton, seams and cameras, with the drivable model's asset names
(`lbs_template_verts`, `lbs_scale`, `tex_mean`, `ao_mean`), a `mugsy_face_mask` and a `face_frontal_view`,
`pose_to_shadow = {n_pose_dims: P, uv_size: 2048}`, B = 2 with a grey and a colour camera and a 128 x 96 render.
The face decoder's geometry is N_FACE_VERTS vertices here (the real face model has 7306)."""
import numpy as np
import torch
import torch.nn.functional as F

import body_frame_restate as bf

H, W, DS = bf.H, bf.W, bf.DS
N_FACE_VERTS = 500
RENAMED = {"template_mesh": "lbs_template_verts", "skeleton_scales": "lbs_scale", "color_mean": "tex_mean",
           "ambient_occlusion_mean": "ao_mean"}
Assets = bf.Assets
seeded_fill = bf.seeded_fill


def assets():
    a = bf.assets()
    for old, new in RENAMED.items():
        a[new] = a.pop(old)
    yy, xx = np.mgrid[0:1024, 0:1024]
    r = np.hypot((yy - 540) / 400.0, (xx - 500) / 330.0)
    a["mugsy_face_mask"] = np.clip(3.0 * (1.0 - r), 0.0, 1.0).astype(np.float32)[..., None]   # soft-edged oval
    a["face_frontal_view"] = np.array([0.1, -0.2, 2.5], np.float32)
    return a


def config(h=H, w=W, ds=DS, n_face_verts=N_FACE_VERTS, n_pose_dims=12):
    """mesh_vae_drivable's model section on the mesh_vae_example.yml sizes, with noise_std given; n_pose_dims is the
    width P of lbs_motion (12 for the fixture's skeleton)"""
    c = bf.config(h, w, ds)
    c["encoder"] = {"n_embs": 1024, "noise_std": 1.0}
    c["encoder_face"] = {"n_embs": 256, "noise_std": 1.0, "n_vert_in": 3 * n_face_verts}
    c["decoder_face"] = {"n_latent": 256, "n_vert_out": 3 * n_face_verts}
    c["pose_to_shadow"] = {"n_pose_dims": n_pose_dims, "uv_size": 2048}
    return c


def inputs(model, batch=2, h=H, w=W, seed=7):
    """the drivable forward's arguments: lbs_motion, campos, geom, ao, K, Rt, _index, face_embs (fp32, seeded)"""
    i = bf.inputs(model, batch, h, w, seed)
    face_embs = torch.randn(batch, 256, generator=torch.Generator().manual_seed(seed + 2))
    return {"lbs_motion": i["pose"], "campos": i["campos"], "geom": i["registration_vertices"],
            "ao": i["ambient_occlusion"], "K": i["K"], "Rt": i["Rt"], "_index": {"camera": i["camera_id"]},
            "face_embs": face_embs}


# ------------------------------------------------------------------------------------------ restatements
def face_tex_tail(x, v, g, bias, face_bias):
    """face.py:58,78-82 for the last texmod layer: (tex_raw, tex)"""
    w = g * v / v.norm()
    raw = F.conv_transpose2d(x, w, None, stride=2, padding=1) + bias
    return raw, 255 * (raw + face_bias + 0.5)


def face_tex_cond(face_tex, mask):
    """mesh_vae_drivable.py:721-724"""
    t = F.interpolate(face_tex, mask.shape[-2:], mode="bilinear", align_corners=False)
    return (t / 255.0 - 0.5) * mask


def pose_shadow(x, beta, size):
    """shadow.py:466-470"""
    return F.interpolate(torch.sigmoid(x + beta), size=(size, size), mode="bilinear")
