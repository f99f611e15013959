"""Generate tests/golden/body_drive_ref.npz by RUNNING the reference's own drivable body avatar
(`mesh_vae_drivable.AutoEncoder`, __init__ and forward) on CPU, in fp64 and again in fp32, in eval mode and in
training mode with the encoders' noise_std = 0:

  * `AutoEncoder`, `CameraPixelBias`, `Encoder`, `FaceEncoder`, `ConvDecoder`, `UNetViewDecoder` and `UpscaleNet` are
    sliced out of /root/reference/ca_code/models/mesh_vae_drivable.py by AST at run time (the module cannot be
    imported: pytorch3d is absent), `FaceDecoderFrontal` is imported from ca_code/nn/face.py (with a stand-in for the
    absent `addict`) and `PoseToShadow` from ca_code.nn.shadow;
  * `RenderLayer` is render_drtk.RenderLayer over tests/mesh_render_restate.drtk_stub(), as in
    make_body_frame_golden.py (the project renders through its own RenderLayer, not pytorch3d);
  * the UV-image builders return the given images, as in make_body_frame_golden.py;
  * assets, configuration and inputs come from tests/body_drive_restate.py, parameters from its seeded fill by name.
Nothing of the reference is copied and no weights are stored.

Frozen: the state-dict keys and shapes; the inputs; the constructor's tex_mean / meye_mask (statistics + samples),
face_cond_mask and encoder_face.tex_cond_mask; per mode, statistics + 256 samples of every output (face_dec_preds
flattened as face_dec_preds.<key>), the gradients of a seeded cotangent on rgb (plus pose_shadow_map in training) for
the first and last parameter (by name) of each trained submodule, and the fp32 run's norm-wise error on each.
`shadow_map` is the map before forward_tex impaints it in place.

Needs /root/reference; the .npz is committed.   Usage: python tests/golden/make_body_drive_golden.py
"""
import ast
import copy
import json
import logging
import os
import sys
import types
import typing
import warnings

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "body_drive_ref.npz")
SRC = "/root/reference/ca_code/models/mesh_vae_drivable.py"
CLASSES = ("CameraPixelBias", "AutoEncoder", "Encoder", "FaceEncoder", "ConvDecoder", "UNetViewDecoder", "UpscaleNet")
MODULES = ("encoder", "encoder_face", "decoder", "decoder_view", "shadow_net", "pose_to_shadow", "upscale_net", "cal",
           "learn_blur", "pixel_cal")

sys.path.insert(0, HERE)
from make_body_frame_golden import nrel_summary, summarise  # noqa: E402


def grad_params(model):
    names = sorted(n for n, _ in model.named_parameters() if "logvar" not in n)
    out = []
    for m in MODULES:
        sub = [n for n in names if n.startswith(m + ".")]
        out += sorted({sub[0], sub[-1]})
    return out


def flatten(preds):
    out = {}
    for k, v in preds.items():
        if isinstance(v, dict):
            out.update({"%s.%s" % (k, kk): vv for kk, vv in v.items()})
        else:
            out[k] = v
    return out


def cotangents(preds, seed=77):
    g = th.Generator().manual_seed(seed)
    wr = th.randn(preds["rgb"].shape, generator=g, dtype=th.float64)
    ws = th.randn(preds["pose_shadow_map"].shape, generator=g, dtype=th.float64) if "pose_shadow_map" in preds else None
    return wr, ws


def run(model, inp, dtype, names):
    model = model.to(dtype)
    captured = {}
    shadow = model.shadow_net if model.training else model.pose_to_shadow
    h = shadow.register_forward_hook(lambda m, a, o: captured.update(shadow_map=o["shadow_map"].clone()))
    cast = {k: (v.to(dtype) if th.is_tensor(v) and v.is_floating_point() else v) for k, v in inp.items()}
    preds = model(**cast)
    h.remove()
    preds = dict(preds)
    preds["shadow_map"] = captured["shadow_map"]
    wr, ws = cotangents(preds)
    loss = (preds["rgb"] * wr.to(dtype)).sum()
    if ws is not None:
        loss = loss + (preds["pose_shadow_map"] * ws.to(dtype)).sum()
    params = dict(model.named_parameters())
    grads = th.autograd.grad(loss, [params[n] for n in names], allow_unused=True)
    return flatten(preds), dict(zip(names, grads))


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, "/root/reference")
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    warnings.filterwarnings("ignore")
    from make_lbs_golden import _stub
    from unittest.mock import MagicMock

    _stub()
    sys.modules.setdefault("turtle", MagicMock())
    sys.modules.setdefault("addict", types.SimpleNamespace(Dict=dict))
    import mesh_render_restate as mr

    sys.modules["drtk"] = mr.drtk_stub()
    import body_drive_restate as bd
    import torch.nn.functional as F
    from torchvision.transforms.functional import gaussian_blur

    import ca_code.nn.layers as la
    import ca_code.utils.geom as geom
    from ca_code.nn.blocks import ConvBlock, ConvDownBlock, UpConvBlockDeep, tile2d, weights_initializer
    from ca_code.nn.color_cal import CalV5
    from ca_code.nn.dof_cal import LearnableBlur
    from ca_code.nn.face import FaceDecoderFrontal
    from ca_code.nn.shadow import PoseToShadow, ShadowUNet
    from ca_code.nn.unet import UNetWB
    from ca_code.utils.lbs import LBSModule
    from ca_code.utils.render_drtk import RenderLayer
    from ca_code.utils.seams import SeamSampler

    a = bd.assets()
    geom.make_uv_vert_index = lambda vt, vi, vti, uv_shape, flip_uv=False: a.index_image.clone()
    geom.make_uv_barys = lambda vt, vti, uv_shape, flip_uv=False: (a.face_index_image.clone(), a.bary_image.clone())
    geom.index_image_impaint = lambda idx, bary=None, distance_threshold=100.0: idx if bary is None else (idx, bary)

    src = open(SRC).read()
    ns = {"th": th, "nn": th.nn, "np": np, "F": F, "la": la, "gaussian_blur": gaussian_blur, "ConvBlock": ConvBlock,
          "ConvDownBlock": ConvDownBlock, "UpConvBlockDeep": UpConvBlockDeep, "tile2d": tile2d,
          "weights_initializer": weights_initializer, "LearnableBlur": LearnableBlur,
          "GeometryModule": geom.GeometryModule, "compute_view_cos": geom.compute_view_cos,
          "ShadowUNet": ShadowUNet, "PoseToShadow": PoseToShadow, "FaceDecoderFrontal": FaceDecoderFrontal,
          "UNetWB": UNetWB, "CalV5": CalV5, "LBSModule": LBSModule, "SeamSampler": SeamSampler,
          "RenderLayer": RenderLayer, "logger": logging.getLogger("mesh_vae_drivable"), **vars(typing)}
    for node in ast.parse(src).body:
        if isinstance(node, ast.ClassDef) and node.name in CLASSES:
            exec(ast.get_source_segment(src, node), ns)

    th.manual_seed(0)
    model = ns["AutoEncoder"](**bd.config(), assets=a)
    bd.seeded_fill(model)
    model.eval()
    d = {"keys_json": np.frombuffer(json.dumps({k: list(v.shape) for k, v in model.state_dict().items()},
                                               sort_keys=True).encode(), dtype=np.uint8)}
    for k in ("tex_mean", "meye_mask"):
        d["buf_" + k] = summarise(getattr(model, k))
    d["buf_face_cond_mask"] = model.face_cond_mask.numpy()
    d["buf_tex_cond_mask"] = model.encoder_face.tex_cond_mask.numpy()
    d["buf_frontal_view"] = model.decoder_face.frontal_view.numpy()

    th.set_num_threads(os.cpu_count() or 1)
    inp = bd.inputs(model, batch=2)
    for k in ("lbs_motion", "campos", "geom", "ao", "K", "Rt", "face_embs"):
        d["in_" + k] = inp[k].numpy()
    names = grad_params(model)
    d["grad_names_json"] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)

    for mode in ("eval", "train"):
        m64 = copy.deepcopy(model).train(mode == "train")
        if mode == "train":
            m64.encoder.noise_std = m64.encoder_face.noise_std = 0.0
        m32 = copy.deepcopy(m64)
        i = dict(inp)
        if mode == "eval":
            i["ao"] = None        # the pose alone drives the shadow
        p64, g64 = run(m64, i, th.float64, names)
        p32, g32 = run(m32, i, th.float32, names)
        d["%s_out_keys_json" % mode] = np.frombuffer(json.dumps(list(p64)).encode(), dtype=np.uint8)
        used = []
        for kind, P64, P32 in (("out", p64, p32), ("grad", g64, g32)):
            for k in P64:
                if P64[k] is None:
                    continue
                if kind == "grad":
                    used.append(k)
                s64, s32 = summarise(P64[k]), summarise(P32[k])
                d["%s_%s_%s" % (mode, kind, k)] = s64
                d["%s_shape_%s_%s" % (mode, kind, k)] = np.array(P64[k].shape)
                d["%s_err32_%s_%s" % (mode, kind, k)] = np.float64(nrel_summary(s32, s64))
                print("%-5s %-4s %-44s |max| %.3e  fp32 err %.2e" % (mode, kind, k, s64[2],
                                                                     d["%s_err32_%s_%s" % (mode, kind, k)]))
        d["%s_grad_names_json" % mode] = np.frombuffer(json.dumps(used).encode(), dtype=np.uint8)
    np.savez_compressed(OUT, **d)
    print("-> %s (%.0f kB)" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
