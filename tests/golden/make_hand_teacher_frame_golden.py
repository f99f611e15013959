"""Generate tests/golden/hand_teacher_frame_ref.npz by RUNNING the reference's own `hand_teacher_mvp.AutoEncoder`
(__init__, forward and the inherited `render`) on CPU, in fp64 and again in fp32, at the example configuration's size
(uv 1024, 4096 primitives of 16 x 16 x 8, volradius 2000), B = 2 (the identity-calibration camera and a grey camera):

  * `AutoEncoder`, `OLATRGBDecoder` and `build_cam_rot_mat` are sliced out of ca_code/models/hand_teacher_mvp.py by
    AST at run time, on top of hand_mvp.py's classes sliced as tests/golden/make_hand_frame_golden.py does (the same
    stubs, GeometryModule images, RenderLayer and `Raymarcher`);
  * mvpraymarch is the C oracle's forward (oracle/raymarch_oracle.c), with `with_shadow=True` for the decoder's deep
    shadow march and mvpraymarch's shadow normalisation; the render's rayrgba is returned as a leaf, so the gradients
    after the render are taken with respect to it;
  * compute_raydirs is the reference's torch formula on the pixel grid it is given; drtk's `transform` is
    make_hand_olat_golden's restatement; `.cuda()` is the identity;
  * compose_envmap is the reference's, run in fp32 (it builds its blur kernel in fp32) and cast back;
  * assets, configuration and parameters come from tests/hand_frame_restate.py, lights and the fixture's reductions
    (128^2 shadow images, chunks of 1, L = 2) from tests/hand_teacher_frame_restate.py.

Modes (hand_teacher_frame_restate.MODES): eval with cal and blur; `.train()` with a background at iteration 0 (zero
deltas, shadow warm-up) and 5000; `fresh`, the model as constructed (geometry in eval, relight in training) at
iteration 0; `env`, eval at 200 x 208 without cal and blur, one light with a [B,1,1] intensity and an `envbg`.
Frozen: the state-dict keys and shapes; the inputs; per mode the output keys in order, statistics + 256 samples of
every output, of the march's inputs and of the shadow-summary render (`render` with primrgb = 255 primshadow); in
the training modes the gradients of a seeded linear functional of primpos / primrot / primscale / primrgba / texolat
with respect to the first and last parameter of poseencoder, poseencoder2, transdecoder, alphadecoder and
relightdecoder, and the post-render gradients (seeded cotangents on rgb and alpha, with respect to rayrgba,
cal.holder.params and learn_blur.weights_raw); for each, the norm-wise error of the fp32 run against the fp64 one.
Nothing of the reference is copied and no weights are stored.

Needs /root/reference and a built oracle; the .npz is committed.
Usage: python tests/golden/make_hand_teacher_frame_golden.py
"""
import ast
import copy
import json
import logging
import os
import sys
import time
import typing
import warnings

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "hand_teacher_frame_ref.npz")
SRC = "/root/reference/ca_code/models/hand_mvp.py"
SRC_T = "/root/reference/ca_code/models/hand_teacher_mvp.py"
SRC_RM = "/root/reference/ca_code/utils/render_raymarcher.py"
CLASSES = ("AutoEncoder", "PoseEncoder", "TransDecoder", "DeconvContentDecoder", "GeomDecoder", "RGBSlabDecoder",
           "init_primitives", "axisangle_to_matrix")
CLASSES_T = ("AutoEncoder", "OLATRGBDecoder", "build_cam_rot_mat")
MARCH_KEYS = ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "template")


class _Oracle:
    """mvpraymarch on the C oracle's forward; records the march inputs and the rayrgba leaf of each render"""

    def __init__(self):
        import oracle

        oracle.lib()
        self.o, self.calls = oracle, []

    def __call__(self, raypos, raydir, stepsize, tminmax, primtransf, template, warp=None, rayterm=None,
                 with_shadow=False, **kw):
        assert warp is None and rayterm is None and not kw
        n = lambda t: np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32))
        pos, rot, scale = primtransf
        rgba, _, sh = self.o.raymarch_fwd(n(raypos), n(raydir), float(stepsize), n(tminmax), n(pos), n(rot), n(scale),
                                          n(template), with_shadow=with_shadow)
        if with_shadow:  # mvpraymarch.py:410-416, channels last
            shadow = sh[..., 0:1] / (sh[..., 1:] + np.float32(1e-5))
            return th.from_numpy(rgba).to(template.dtype), th.from_numpy(shadow).to(template.dtype)
        out = th.from_numpy(rgba).to(template.dtype).requires_grad_()
        self.calls.append({"raypos": raypos, "raydir": raydir, "tminmax": tminmax, "primpos": pos, "primrot": rot,
                           "primscale": scale, "template": template, "rayrgba": out})
        return out


class RenderLayer(th.nn.Module):
    """pytorch3d RenderLayer's state (render_pytorch3d.py:20-31): the persistent image_size buffer"""

    def __init__(self, h, w, vi, vt, vti, flip_uvs=False):
        super().__init__()
        self.register_buffer("image_size", th.as_tensor([h, w], dtype=th.int32))


def raydirs(campos, camrot, focal, princpt, pix, volradius):
    """compute_raydirs: the reference's torch formula (extensions/utils/utils.py:127-143) on the pixel grid `pix`
    [N,H,W,2], with the CUDA op's viewpos / volradius (utils_kernel.cu)"""
    N, h, w = pix.shape[:3]
    viewpos = campos / volradius
    raypos = viewpos[:, None, None, :].expand(-1, h, w, -1).contiguous()
    raydir = (pix.to(campos.dtype) - princpt[:, None, None, :]) / focal[:, None, None, :]
    raydir = th.cat([raydir, th.ones_like(raydir[..., :1])], -1)
    raydir = th.sum(camrot[:, None, None, :, :] * raydir[..., :, None], dim=-2)
    raydir = raydir / th.sqrt(th.sum(raydir ** 2, dim=-1, keepdim=True))
    t1 = (-1.0 - viewpos[:, None, None, :]) / raydir
    t2 = (1.0 - viewpos[:, None, None, :]) / raydir
    tmin = th.max(th.min(t1[..., 0], t2[..., 0]),
                  th.max(th.min(t1[..., 1], t2[..., 1]), th.min(t1[..., 2], t2[..., 2]))).clamp(min=0.0)
    tmax = th.min(th.max(t1[..., 0], t2[..., 0]),
                  th.min(th.max(t1[..., 1], t2[..., 1]), th.max(t1[..., 2], t2[..., 2])))
    return raypos, raydir, th.stack([tmin, tmax], -1)


def run(model, inp, dtype, ht, hr, orc, names, iteration, grads):
    """-> ({kind: {name: (summary, shape)}}, output keys); the tensors and their graph are freed on return"""
    th.set_default_dtype(dtype)  # build_cam_rot_mat allocates its matrix in the default dtype
    try:
        *res, keys = _run(model, inp, dtype, ht, hr, orc, names, iteration, grads)
    finally:
        th.set_default_dtype(th.float32)
    kinds = ("out", "pre", "post", "march", "shadow")
    return {kind: {k: (hr.summarise(t), tuple(t.shape)) for k, t in r.items()} for kind, r in zip(kinds, res)}, keys


def _run(model, inp, dtype, ht, hr, orc, names, iteration, grads):
    model = model.to(dtype)
    ht.reduce(model)
    cast = {k: (v.to(dtype) if th.is_tensor(v) and v.is_floating_point() else v) for k, v in inp.items()}
    orc.calls = []
    preds = model(**cast, iteration=iteration)
    call = orc.calls[-1]
    march = {k: call[k] for k in MARCH_KEYS}
    # HandMVPSummary's shadow image: render with primrgb = 255 primshadow, on a copy of preds
    with th.no_grad():
        sp = dict(preds)
        sp["primrgb"] = 255.0 * preds["primshadow"]
        srgb, salpha, _ = model.render(cast["K"], cast["Rt"], sp, with_shadow=False)
    shadow = {"rgb": srgb, "alpha": salpha, "primrgba": sp["primrgba"]}
    out = {k: v for k, v in preds.items() if th.is_tensor(v) and v.dtype != th.bool}
    if not grads:
        return out, {}, {}, march, shadow, list(preds)
    params = dict(model.named_parameters())
    w = ht.functional_weights({k: preds[k].shape for k in ht.PRIM_KEYS if k in preds})
    f = sum((preds[k] * w[k].to(dtype)).sum() for k in w)
    pre = th.autograd.grad(f, [params[n] for n in names], retain_graph=True, allow_unused=True)
    pre = {n: (g if g is not None else th.zeros_like(params[n])) for n, g in zip(names, pre)}
    wr, wa = hr.cotangents(preds["rgb"].shape, preds["alpha"].shape)
    extra = [k for k in ("cal.holder.params", "learn_blur.weights_raw") if k in params]
    gr = th.autograd.grad((preds["rgb"] * wr.to(dtype)).sum() + (preds["alpha"] * wa.to(dtype)).sum(),
                          [call["rayrgba"]] + [params[k] for k in extra], allow_unused=True)
    post = {"rayrgba": gr[0], **dict(zip(extra, gr[1:]))}
    return out, pre, post, march, shadow, list(preds)


def _slice(ns, path, names):
    src = open(path).read()
    for node in ast.parse(src).body:
        if isinstance(node, (ast.ClassDef, ast.FunctionDef)) and node.name in names:
            exec(ast.get_source_segment(src, node), ns)


def main():
    if not os.path.isfile(SRC_T):
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
    import hand_teacher_frame_restate as ht
    import torch.nn.functional as F
    from make_hand_olat_golden import transform

    import ca_code.nn.layers as la
    import ca_code.utils.geom as geom
    from ca_code.nn.blocks import ConvBlock, tile2d
    from ca_code.nn.color_cal import CalV5
    from ca_code.nn.dof_cal import LearnableBlur
    from ca_code.utils.envmap import compose_envmap as ref_compose
    from ca_code.utils.lbs import LBSModule

    th.Tensor.cuda = lambda self, *a, **k: self
    a = hr.assets()
    geom.make_uv_vert_index = lambda vt, vi, vti, uv_shape, flip_uv=False: a.index_image.clone()
    geom.make_uv_barys = lambda vt, vti, uv_shape, flip_uv=False: (a.face_index_image.clone(), a.bary_image.clone())
    geom.index_image_impaint = (lambda idx, bary=None, distance_threshold=100.0:
                                idx if bary is None else (idx, a.bary_image_impaint.clone()))
    orc = _Oracle()

    def compose_envmap(render, alpha, envbg, K, Rt):
        dt = th.get_default_dtype()
        th.set_default_dtype(th.float32)
        try:
            return ref_compose(render.float(), alpha.float(), envbg.float(), K.float(), Rt.float()).to(render.dtype)
        finally:
            th.set_default_dtype(dt)

    ns = {"th": th, "torch": th, "nn": th.nn, "np": np, "F": F, "la": la, "ConvBlock": ConvBlock, "tile2d": tile2d,
          "CalV5": CalV5, "LearnableBlur": LearnableBlur, "LBSModule": LBSModule, "GeometryModule": geom.GeometryModule,
          "compute_tbn": geom.compute_tbn, "compute_view_cos": geom.compute_view_cos, "make_postex": geom.make_postex,
          "values_to_uv": geom.values_to_uv, "RenderLayer": RenderLayer, "mvpraymarch": orc,
          "compute_raydirs": raydirs, "transform": transform, "compose_envmap": compose_envmap,
          "logger": logging.getLogger("hand_mvp"), **vars(typing)}
    _slice(ns, SRC, CLASSES)
    _slice(ns, SRC_RM, ("Raymarcher",))
    ns["BaseAE"] = ns["AutoEncoder"]
    _slice(ns, SRC_T, CLASSES_T)
    AE = ns["AutoEncoder"]
    assert AE is not ns["BaseAE"] and issubclass(AE, ns["BaseAE"])

    th.manual_seed(0)
    th.set_num_threads(os.cpu_count() or 1)
    model = hr.seeded_fill(AE(**hr.config(), assets=a))
    sd = model.state_dict()
    d = {"keys_json": np.frombuffer(json.dumps({k: list(v.shape) for k, v in sd.items()}, sort_keys=True).encode(),
                                    dtype=np.uint8)}
    print("%d state-dict keys, %d valid primitives" % (len(sd), int(model.valid_prims.sum())))
    d["valid_prims"] = model.valid_prims.numpy()
    env_model = AE(**ht.env_config(), assets=a)
    res = env_model.load_state_dict(sd, strict=False)
    assert not res.missing_keys and all(k.startswith(("cal.", "learn_blur.")) for k in res.unexpected_keys)
    env_model.eval()

    pose, _ = hr.pose_inputs()
    with th.no_grad():
        posed = model.lbs_fn.pose(th.zeros_like(model.lbs_fn.lbs_template_verts), pose)
    K, Rt, campos = hr.side_cameras(posed)
    light_pos, light_intensity = ht.lights(posed)
    inp = {"pose": pose, "campos": campos, "K": K, "Rt": Rt, "light_pos": light_pos,
           "light_intensity": light_intensity, "camera_id": list(hr.BATCH_CAMERAS), "background": hr.background()}
    Ke, Rte, campose = hr.side_cameras(posed, ht.ENV_H, ht.ENV_W)
    lpe, _ = ht.lights(posed, n=1, seed=12)
    env = {"pose": pose, "campos": campose, "K": Ke, "Rt": Rte, "light_pos": lpe,
           "light_intensity": th.ones(2, 1, 1), "camera_id": list(hr.BATCH_CAMERAS), "envbg": ht.envbg(),
           "index": [3, 4], "n_lights": th.ones(2, 1)}
    for k in ("pose", "campos", "K", "Rt", "light_pos", "light_intensity", "background"):
        d["in_" + k] = inp[k].float().numpy()
    for k in ("campos", "K", "Rt", "light_pos", "light_intensity", "envbg"):
        d["env_in_" + k] = env[k].float().numpy()
    names = ht.grad_param_names(model)
    d["grad_names_json"] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)

    for mode in ht.MODES:
        t0 = time.time()
        base, x = (env_model, env) if mode == "env" else (model, inp)
        it, grads = ht.ITERATION[mode], mode in ht.GRAD_MODES
        r64, keys = run(_copy_mode(base, mode), x, th.float64, ht, hr, orc, names, it, grads)
        r32, _ = run(_copy_mode(base, mode), x, th.float32, ht, hr, orc, names, it, grads)
        d["%s_out_keys_json" % mode] = np.frombuffer(json.dumps(keys).encode(), dtype=np.uint8)
        for kind in r64:
            for k, (s64, shape) in r64[kind].items():
                d["%s_%s_%s" % (mode, kind, k)] = s64
                d["%s_shape_%s_%s" % (mode, kind, k)] = np.array(shape)
                d["%s_err32_%s_%s" % (mode, kind, k)] = np.float64(hr.nrel_summary(r32[kind][k][0], s64))
                print("%-6s %-6s %-40s |max| %.3e  fp32 err %.2e" % (mode, kind, k, s64[2],
                                                                       d["%s_err32_%s_%s" % (mode, kind, k)]))
        print("%s: %.0f s" % (mode, time.time() - t0))
    np.savez_compressed(OUT, **d)
    print("-> %s (%.0f kB)" % (OUT, os.path.getsize(OUT) / 1024))


def _copy_mode(base, mode):
    """a copy of the model in the mode's training state; `fresh` keeps the constructor's"""
    m = copy.deepcopy(base)
    if mode in ("eval", "env"):
        m.eval()
    elif mode != "fresh":
        m.train()
    return m


if __name__ == "__main__":
    main()
