"""Generate tests/golden/body_frame_ref.npz by RUNNING the reference's own `mesh_vae.AutoEncoder` (__init__ and
forward) on CPU, in fp64 and again in fp32, at the mesh_vae_example.yml model configuration with a 128 x 96 render
(ds_rate 8):

  * `AutoEncoder`, `CameraPixelBias`, `Encoder`, `FaceEncoder`, `ConvDecoder`, `UNetViewDecoder` and `UpscaleNet` are
    sliced out of /root/reference/ca_code/models/mesh_vae.py by AST at run time (the module cannot be imported: drtk
    and pytorch3d are absent) and run on the reference's own LBSModule, SeamSampler, GeometryModule, CalV5,
    LearnableBlur, ShadowUNet, UNetWB and RenderLayer;
  * drtk is tests/mesh_render_restate.drtk_stub() (its edge-gradient estimator is the identity);
  * make_uv_vert_index / make_uv_barys / index_image_impaint return the given UV images, so the reference's geo_fn
    holds exactly the images the assets carry;
  * depth_discontuity_mask builds an fp32 Sobel kernel, so the fp64 run hands it the depth in fp32;
  * assets, configuration and inputs come from tests/body_frame_restate.py (the synthetic sheet skinned by a
    lbs_recipe skeleton, B = 2 with a grey and a colour camera), parameters from its seeded fill by name.
Nothing of the reference is copied and no weights are stored.

Frozen: the state-dict keys and shapes; the inputs (except the seeded AO map); statistics + 256 samples of every
output key and of the constructor's tex_mean / meye_mask, face_cond_mask and depth_disc_mask in full; the
gradients of a seeded cotangent on rgb and alpha for the first and last parameter (by name) of each submodule; and
for each of those the norm-wise error of the fp32 run against the fp64 one.  `shadow_map` is the shadow net's map
before forward_tex impaints it in place.

Needs /root/reference; the .npz is committed.   Usage: python tests/golden/make_body_frame_golden.py
"""
import ast
import copy
import json
import logging
import os
import sys
import typing
import warnings

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "body_frame_ref.npz")
SRC = "/root/reference/ca_code/models/mesh_vae.py"
CLASSES = ("CameraPixelBias", "AutoEncoder", "Encoder", "FaceEncoder", "ConvDecoder", "UNetViewDecoder", "UpscaleNet")
MODULES = ("encoder", "encoder_face", "decoder", "decoder_view", "shadow_net", "upscale_net", "cal", "learn_blur",
           "pixel_cal")


def summarise(t):
    f = t.detach().double().reshape(-1)
    idx = th.linspace(0, f.numel() - 1, 256, dtype=th.float64).long()
    return np.concatenate([[f.mean().item(), f.std().item(), f.abs().max().item(), float(f.numel())], f[idx].numpy()])


def nrel_summary(a, b):
    """norm-wise relative difference of two summaries (statistics and samples, not the count)"""
    a, b = np.delete(a, 3), np.delete(b, 3)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def grad_params(model):
    names = sorted(n for n, _ in model.named_parameters() if "logvar" not in n)
    out = []
    for m in MODULES:
        sub = [n for n in names if n.startswith(m + ".")]
        out += sorted({sub[0], sub[-1]})
    return out


def cotangents(preds, seed=77):
    g = th.Generator().manual_seed(seed)
    return th.randn(preds["rgb"].shape, generator=g, dtype=th.float64), th.randn(preds["alpha"].shape, generator=g,
                                                                                 dtype=th.float64)


def run(model, inp, dtype, names):
    model = model.to(dtype)
    captured = {}
    h = model.shadow_net.register_forward_hook(lambda m, a, o: captured.update(shadow_map=o["shadow_map"].clone()))
    cast = {k: (v.to(dtype) if th.is_tensor(v) and v.is_floating_point() else v) for k, v in inp.items()}
    preds = model(**cast)
    h.remove()
    preds = dict(preds)
    preds["shadow_map"] = captured["shadow_map"]
    wr, wa = cotangents(preds)
    params = dict(model.named_parameters())
    loss = (preds["rgb"] * wr.to(dtype)).sum() + (preds["alpha"] * wa.to(dtype)).sum()
    grads = th.autograd.grad(loss, [params[n] for n in names], allow_unused=True)
    return preds, dict(zip(names, grads))


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, "/root/reference")
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, HERE)
    warnings.filterwarnings("ignore")
    from make_lbs_golden import _stub
    from unittest.mock import MagicMock

    _stub()
    sys.modules.setdefault("turtle", MagicMock())
    import mesh_render_restate as mr

    sys.modules["drtk"] = mr.drtk_stub()
    import body_frame_restate as bf
    import torch.nn.functional as F
    from torchvision.transforms.functional import gaussian_blur

    import ca_code.nn.layers as la
    import ca_code.utils.geom as geom
    from ca_code.nn.blocks import ConvBlock, ConvDownBlock, UpConvBlockDeep, tile2d, weights_initializer
    from ca_code.nn.color_cal import CalV5
    from ca_code.nn.dof_cal import LearnableBlur
    from ca_code.nn.shadow import ShadowUNet
    from ca_code.nn.unet import UNetWB
    from ca_code.utils.lbs import LBSModule
    from ca_code.utils.render_drtk import RenderLayer
    from ca_code.utils.seams import SeamSampler

    a = bf.assets()
    geom.make_uv_vert_index = lambda vt, vi, vti, uv_shape, flip_uv=False: a.index_image.clone()
    geom.make_uv_barys = lambda vt, vti, uv_shape, flip_uv=False: (a.face_index_image.clone(), a.bary_image.clone())
    geom.index_image_impaint = lambda idx, bary=None, distance_threshold=100.0: idx if bary is None else (idx, bary)

    src = open(SRC).read()
    ns = {"th": th, "nn": th.nn, "np": np, "F": F, "la": la, "gaussian_blur": gaussian_blur, "ConvBlock": ConvBlock,
          "ConvDownBlock": ConvDownBlock, "UpConvBlockDeep": UpConvBlockDeep, "tile2d": tile2d,
          "weights_initializer": weights_initializer, "LearnableBlur": LearnableBlur,
          "GeometryModule": geom.GeometryModule, "compute_view_cos": geom.compute_view_cos,
          "depth_discontuity_mask": lambda depth: geom.depth_discontuity_mask(depth.float()),  # an fp32 kernel
          "ShadowUNet": ShadowUNet, "PoseToShadow": None,
          "UNetWB": UNetWB, "CalV5": CalV5, "LBSModule": LBSModule, "SeamSampler": SeamSampler,
          "RenderLayer": RenderLayer, "logger": logging.getLogger("mesh_vae"), **vars(typing)}
    for node in ast.parse(src).body:
        if isinstance(node, ast.ClassDef) and node.name in CLASSES:
            exec(ast.get_source_segment(src, node), ns)

    th.manual_seed(0)
    cfg = bf.config()
    model = ns["AutoEncoder"](**cfg, assets=a)
    bf.seeded_fill(model)
    model.eval()
    d = {"keys_json": np.frombuffer(json.dumps({k: list(v.shape) for k, v in model.state_dict().items()},
                                               sort_keys=True).encode(), dtype=np.uint8)}
    for k in ("tex_mean", "meye_mask"):
        d["buf_" + k] = summarise(getattr(model, k))
    d["buf_face_cond_mask"] = model.face_cond_mask.numpy()

    th.set_num_threads(os.cpu_count() or 1)
    inp = bf.inputs(model, batch=2)
    for k in ("pose", "campos", "registration_vertices", "K", "Rt"):
        d["in_" + k] = inp[k].numpy()
    names = grad_params(model)
    d["grad_names_json"] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)

    model32 = copy.deepcopy(model)
    p64, g64 = run(model, inp, th.float64, names)
    p32, g32 = run(model32, inp, th.float32, names)
    d["out_keys_json"] = np.frombuffer(json.dumps(list(p64)).encode(), dtype=np.uint8)
    d["depth_disc_mask"] = p64["depth_disc_mask"].numpy()
    d["depth_disc_mask_fp32"] = p32["depth_disc_mask"].numpy()
    for kind, P64, P32 in (("out", p64, p32), ("grad", g64, g32)):
        for k in P64:
            if P64[k] is None or P64[k].dtype == th.bool:
                continue
            s64, s32 = summarise(P64[k]), summarise(P32[k])
            d["%s_%s" % (kind, k)] = s64
            d["shape_%s_%s" % (kind, k)] = np.array(P64[k].shape)
            d["err32_%s_%s" % (kind, k)] = np.float64(nrel_summary(s32, s64))
            print("%-4s %-40s |max| %.3e  fp32 err %.2e" % (kind, k, s64[2], d["err32_%s_%s" % (kind, k)]))
    cover = float((p64["alpha"] > 0).double().mean())
    print("coverage %.2f, depth_disc_mask %d px (fp32 run: %d)" % (cover, int(p64["depth_disc_mask"].sum()),
                                                                    int(p32["depth_disc_mask"].sum())))
    np.savez_compressed(OUT, **d)
    print("-> %s (%.0f kB)" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
