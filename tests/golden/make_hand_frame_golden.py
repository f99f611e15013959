"""Generate tests/golden/hand_frame_ref.npz by RUNNING the reference's own `hand_mvp.AutoEncoder` (__init__ and
forward) on CPU, in fp64 and again in fp32, at hand_mvp_example.yml's model configuration (uv 1024, 4096 primitives
of 16 x 16 x 8, volradius 2000) with a 96 x 64 render, B = 2 (the identity-calibration camera and a grey camera):

  * `AutoEncoder`, `PoseEncoder`, `TransDecoder`, `DeconvContentDecoder`, `GeomDecoder`, `RGBSlabDecoder`,
    `init_primitives` and `axisangle_to_matrix` are sliced out of /root/reference/ca_code/models/hand_mvp.py, and
    `Raymarcher` out of ca_code/utils/render_raymarcher.py, by AST at run time (the modules cannot be imported:
    pytorch3d and the CUDA extensions are absent).  They run on the reference's own LBSModule, GeometryModule
    (make_uv_vert_index / make_uv_barys / index_image_impaint return the assets' images), CalV5 and LearnableBlur;
  * pytorch3d's RenderLayer is a stub holding its `image_size` buffer;
  * compute_raydirs is the reference's torch formula (tests/hand_frame_restate.raydirs);
  * mvpraymarch is the C oracle's forward (oracle/raymarch_oracle.c, fp32 as the reference's fast-math kernel); its
    rayrgba is returned as a leaf, so the gradients after the render are taken with respect to it;
  * assets, configuration and parameters come from tests/hand_frame_restate.py.

Three modes: eval with cal and blur; training with a background at iteration 0 (< primposstart: zero deltas) and at
iteration 5000.  Frozen: the state-dict keys and shapes; the inputs; per mode, statistics + 256 samples of every
output key, of the march's inputs (the compacted transforms and template, raypos / raydir / tminmax), of the
pre-render gradients (a seeded linear functional of primpos / primrot / primscale / primrgba, with respect to the
first and last parameter of poseencoder, transdecoder, alphadecoder and rgbdecoder) and of the post-render gradients
(seeded cotangents on rgb and alpha, with respect to rayrgba, cal.holder.params and learn_blur.weights_raw), and for
each the norm-wise error of the fp32 run against the fp64 one.  Nothing of the reference is copied and no weights
are stored.

Needs /root/reference and a built oracle; the .npz is committed.   Usage: python tests/golden/make_hand_frame_golden.py
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
OUT = os.path.join(HERE, "hand_frame_ref.npz")
SRC = "/root/reference/ca_code/models/hand_mvp.py"
SRC_RM = "/root/reference/ca_code/utils/render_raymarcher.py"
CLASSES = ("AutoEncoder", "PoseEncoder", "TransDecoder", "DeconvContentDecoder", "GeomDecoder", "RGBSlabDecoder",
           "init_primitives", "axisangle_to_matrix")


class _Oracle:
    """mvpraymarch on the C oracle's forward; records the march inputs and the rayrgba leaf of each call"""

    def __init__(self):
        import oracle

        oracle.lib()
        self.o, self.calls = oracle, []

    def __call__(self, raypos, raydir, stepsize, tminmax, primtransf, template, warp=None, rayterm=None,
                 with_shadow=False, **kw):
        assert warp is None and rayterm is None and not with_shadow and not kw
        n = lambda t: np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32))
        pos, rot, scale = primtransf
        rgba, _, _ = self.o.raymarch_fwd(n(raypos), n(raydir), float(stepsize), n(tminmax), n(pos), n(rot), n(scale),
                                         n(template))
        out = th.from_numpy(rgba).to(template.dtype).requires_grad_()
        self.calls.append({"raypos": raypos, "raydir": raydir, "tminmax": tminmax, "primpos": pos, "primrot": rot,
                           "primscale": scale, "template": template, "rayrgba": out})
        return out


class RenderLayer(th.nn.Module):
    """pytorch3d RenderLayer's state (render_pytorch3d.py:20-31): the persistent image_size buffer"""

    def __init__(self, h, w, vi, vt, vti, flip_uvs=False):
        super().__init__()
        self.register_buffer("image_size", th.as_tensor([h, w], dtype=th.int32))


def run(model, inp, dtype, hr, orc, names, iteration):
    model = model.to(dtype)
    cast = {k: (v.to(dtype) if th.is_tensor(v) and v.is_floating_point() else v) for k, v in inp.items()}
    orc.calls = []
    preds = model(**cast, iteration=iteration)
    call = orc.calls[-1]
    params = dict(model.named_parameters())
    w = hr.functional_weights({k: preds[k].shape for k in hr.PRIM_KEYS})
    f = sum((preds[k] * w[k].to(dtype)).sum() for k in hr.PRIM_KEYS)
    pre = th.autograd.grad(f, [params[n] for n in names], retain_graph=True, allow_unused=True)
    pre = {n: (g if g is not None else th.zeros_like(params[n])) for n, g in zip(names, pre)}
    wr, wa = hr.cotangents(preds["rgb"].shape, preds["alpha"].shape)
    extra = [k for k in ("cal.holder.params", "learn_blur.weights_raw") if k in params]
    gr = th.autograd.grad((preds["rgb"] * wr.to(dtype)).sum() + (preds["alpha"] * wa.to(dtype)).sum(),
                          [call["rayrgba"]] + [params[k] for k in extra], allow_unused=True)
    post = {"rayrgba": gr[0], **dict(zip(extra, gr[1:]))}
    march = {k: call[k] for k in ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "template")}
    return preds, pre, post, march


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
    import hand_frame_restate as hr
    import torch.nn.functional as F

    import ca_code.nn.layers as la
    import ca_code.utils.geom as geom
    from ca_code.nn.blocks import ConvBlock, tile2d
    from ca_code.nn.color_cal import CalV5
    from ca_code.nn.dof_cal import LearnableBlur
    from ca_code.utils.lbs import LBSModule

    a = hr.assets()
    geom.make_uv_vert_index = lambda vt, vi, vti, uv_shape, flip_uv=False: a.index_image.clone()
    geom.make_uv_barys = lambda vt, vti, uv_shape, flip_uv=False: (a.face_index_image.clone(), a.bary_image.clone())
    geom.index_image_impaint = (lambda idx, bary=None, distance_threshold=100.0:
                                idx if bary is None else (idx, a.bary_image_impaint.clone()))
    orc = _Oracle()
    ns = {"th": th, "torch": th, "nn": th.nn, "np": np, "F": F, "la": la, "ConvBlock": ConvBlock, "tile2d": tile2d,
          "CalV5": CalV5, "LearnableBlur": LearnableBlur, "LBSModule": LBSModule, "GeometryModule": geom.GeometryModule,
          "compute_tbn": geom.compute_tbn, "compute_view_cos": geom.compute_view_cos, "make_postex": geom.make_postex,
          "values_to_uv": geom.values_to_uv, "RenderLayer": RenderLayer, "mvpraymarch": orc,
          "logger": logging.getLogger("hand_mvp"), **vars(typing)}
    ns["compute_raydirs"] = lambda campos, camrot, focal, princpt, pix, volradius: hr.raydirs(
        campos, camrot, focal, princpt, pix.shape[1], pix.shape[2], volradius)
    src = open(SRC).read()
    for node in ast.parse(src).body:
        if isinstance(node, (ast.ClassDef, ast.FunctionDef)) and node.name in CLASSES:
            exec(ast.get_source_segment(src, node), ns)
    src = open(SRC_RM).read()
    for node in ast.parse(src).body:
        if isinstance(node, ast.ClassDef) and node.name == "Raymarcher":
            exec(ast.get_source_segment(src, node), ns)

    th.manual_seed(0)
    th.set_num_threads(os.cpu_count() or 1)
    model = ns["AutoEncoder"](**hr.config(), assets=a)
    hr.seeded_fill(model)
    d = {"keys_json": np.frombuffer(json.dumps({k: list(v.shape) for k, v in model.state_dict().items()},
                                               sort_keys=True).encode(), dtype=np.uint8)}
    print("%d state-dict keys, %d valid primitives" % (len(model.state_dict()), int(model.valid_prims.sum())))
    d["valid_prims"] = model.valid_prims.numpy()

    pose, ao = hr.pose_inputs()
    with th.no_grad():
        posed = model.lbs_fn.pose(th.zeros_like(model.lbs_fn.lbs_template_verts), pose)
    K, Rt, campos = hr.side_cameras(posed)
    inp = {"pose": pose, "campos": campos, "ambient_occlusion": ao, "K": K, "Rt": Rt,
           "camera_id": list(hr.BATCH_CAMERAS), "background": hr.background()}
    for k in ("pose", "campos", "ambient_occlusion", "K", "Rt", "background"):
        d["in_" + k] = inp[k].numpy()
    names = hr.grad_param_names(model)
    d["grad_names_json"] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)

    for mode in hr.MODES:
        m64 = copy.deepcopy(model).train(mode != "eval")
        m32 = copy.deepcopy(m64)
        it = hr.ITERATION[mode]
        r64 = run(m64, inp, th.float64, hr, orc, names, it)
        r32 = run(m32, inp, th.float32, hr, orc, names, it)
        d["%s_out_keys_json" % mode] = np.frombuffer(json.dumps(list(r64[0])).encode(), dtype=np.uint8)
        for kind, A64, A32 in zip(("out", "pre", "post", "march"), r64, r32):
            for k in A64:
                if not th.is_tensor(A64[k]) or A64[k].dtype == th.bool:
                    continue
                s64, s32 = hr.summarise(A64[k]), hr.summarise(A32[k])
                d["%s_%s_%s" % (mode, kind, k)] = s64
                d["%s_shape_%s_%s" % (mode, kind, k)] = np.array(A64[k].shape)
                d["%s_err32_%s_%s" % (mode, kind, k)] = np.float64(hr.nrel_summary(s32, s64))
                print("%-6s %-5s %-40s |max| %.3e  fp32 err %.2e" % (mode, kind, k, s64[2],
                                                                      d["%s_err32_%s_%s" % (mode, kind, k)]))
        alpha = r64[0]["alpha"]
        print("%s: coverage %.2f (alpha > 0.5: %.2f)" % (mode, float((alpha > 0).double().mean()),
                                                         float((alpha > 0.5).double().mean())))
    np.savez_compressed(OUT, **d)
    print("-> %s (%.0f kB)" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
