"""Generate tests/golden/mesh_render_ref.npz by RUNNING the reference's `RenderLayer` (ca_code/utils/render_drtk.py)
on CPU in fp64.  drtk is a third-party package that is not installed, so `drtk` is put in sys.modules as the torch
restatement of the project's conventions (tests/mesh_render_restate.py: transform, rasterize deciding coverage in fp32
with the kernel's expression order, render, interpolate, and an identity edge_grad_estimator).  What the fixture pins
is what the reference itself decides around drtk: the (2 vt - 1) remap, the grid_sample mode / align_corners / zero
padding, the mask multiply, flip_uvs, the output keys and the image_size buffer; the edge term is not in it.

Scene: B = 2 cameras on the tube mesh of tests/lbs_recipe.py plus a quad that cuts through it, a 64 x 96 image and a
4-channel 64^2 texture; flip_uvs=True.  Stored: inputs, every output, and the gradients of verts and tex under a seeded
cotangent of `render`.

Needs /root/reference; the .npz is committed.   Usage: python tests/golden/make_mesh_render_golden.py
"""
import importlib
import os
import sys

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "mesh_render_ref.npz")
SRC = "/root/reference/ca_code/utils/render_drtk.py"
H, W = 64, 96


def scene():
    import lbs_recipe

    verts, faces, tex_faces, uvs, _ = lbs_recipe.tube()
    quad = np.array([[-8.0, -5.0, 2.0], [8.0, -4.0, -1.0], [7.0, 6.0, -2.0], [-7.0, 5.0, 1.0]], np.float32)
    quv = np.array([[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]], np.float32)
    V, T = len(verts), len(uvs)
    vi = np.concatenate([faces, np.array([[0, 1, 2], [0, 2, 3]]) + V]).astype(np.int64)
    vti = np.concatenate([tex_faces, np.array([[0, 1, 2], [0, 2, 3]]) + T]).astype(np.int64)
    verts = np.concatenate([verts, quad])
    vt = np.concatenate([uvs, quv])
    K = np.array([[[110.0, 0, 48.0], [0, 110.0, 32.0], [0, 0, 1]], [[95.0, 0, 50.0], [0, 97.0, 30.0], [0, 0, 1]]],
                 np.float32)
    Rt = np.zeros((2, 3, 4), np.float32)
    for b, (yaw, pitch, dist) in enumerate(((0.3, 1.2, 40.0), (-0.5, 1.7, 34.0))):
        cy, sy, cp, sp = np.cos(yaw), np.sin(yaw), np.cos(pitch), np.sin(pitch)
        Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
        Rx = np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
        Rt[b, :, :3] = Rx @ Ry
        Rt[b, :, 3] = [0.3 * b, -0.2, dist]
    rng = np.random.default_rng(2024)
    # quantised (exact in fp32, and they compress)
    tex = (np.round(rng.uniform(0, 1, size=(2, 4, 64, 64)) * 64) / 64).astype(np.float32)
    cot = (np.round(rng.standard_normal((2, 4, H, W)) * 16) / 16).astype(np.float32)
    return dict(verts=np.repeat(verts[None], 2, 0).astype(np.float32), vi=vi, vti=vti, vt_in=vt.astype(np.float32),
                K=K, Rt=Rt, tex=tex, cotangent=cot)


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, "/root/reference")
    import mesh_render_restate as mr

    sys.modules["drtk"] = mr.drtk_stub()
    RenderLayer = importlib.import_module("ca_code.utils.render_drtk").RenderLayer

    s = scene()
    d = lambda a: th.from_numpy(np.asarray(a)).double()
    layer = RenderLayer(H, W, th.from_numpy(s["vi"]), d(s["vt_in"]).clone(), th.from_numpy(s["vti"]), flip_uvs=True)
    verts = d(s["verts"]).requires_grad_()
    tex = d(s["tex"]).requires_grad_()
    out = layer(verts, tex, d(s["K"]), d(s["Rt"]))
    g_verts, g_tex = th.autograd.grad((out["render"] * d(s["cotangent"])).sum(), [verts, tex])
    res = dict(s, h=np.array(H), w=np.array(W), flip_uvs=np.array(True), keys=np.array(sorted(out)),
               sd_image_size=layer.state_dict()["image_size"].numpy(), g_verts=g_verts.numpy(), g_tex=g_tex.numpy())
    for k, v in out.items():
        res[k] = v.detach().numpy()
    cov = (res["index_img"] >= 0).mean()
    assert 0.1 < cov < 0.9, cov
    res = {k: v.astype(np.float32) if v.dtype == np.float64 else v for k, v in res.items()}
    np.savez_compressed(OUT, **res)
    print("wrote", OUT, os.path.getsize(OUT), "bytes; coverage %.2f" % cov)


if __name__ == "__main__":
    main()
