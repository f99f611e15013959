"""Generate tests/golden/head_frame_ref.npz by RUNNING the reference's own `rgca.AutoEncoder` on CPU, in fp64 and
again in fp32, at rgca_example.yml's model configuration with a decoder slab of tests/head_frame_restate.SLAB and a
208 x 256 render, B = 2 (a grey and a colour camera):

  * `AutoEncoder`, `Encoder`, `GeomDecoder` and `PrimDecoder` are sliced out of /root/reference/ca_code/models/rgca.py
    by AST at run time (the module cannot be imported: gsplat and the sgutils extension are absent).  PrimDecoder's
    hard-coded slab is scaled from 1024 to SLAB (its 1024 literals, untied-bias sizes and 8 x 8 seed grid divided by
    1024 / SLAB).  They run on the reference's own GeometryModule (make_uv_vert_index / make_uv_barys return the
    assets' UV images), CalV5, LearnableBlur, compose_envmap, dir2uv, mipmap_grid_sample and sh;
  * `render_gs` is the C splat oracle's forward (oracle/, fp32: project, bin + sort, blend rgb, blend depth); its rgb
    images are returned as leaves so the gradients after the render can be taken with respect to them;
  * `evaluate_gaussian` is the reference wrapper's normalisation followed by the C SG oracle's forward and backward
    (fp32, as the reference's CUDA extension);
  * compose_envmap builds its mirror-ball rays in fp32, so the fp64 run hands it envbg, K and Rt in fp32;
  * parameters come from head_frame_restate.seeded_fill, inputs from head_frame_restate.mode_inputs.

Three modes: eval with L = 460 zero-padded point lights; training with noise_std = 0, a background and
is_fully_lit_frame = [True, False]; eval environment map with preconv_envmap, envbg and lightrot, cal off, blur on.

Frozen: the state-dict keys and shapes; the light statements (rgca.py:175-193) executed in fp64 (C = 1 and 3); per
mode, statistics + 256 samples of every output key, the render's arguments (fx, fy, cx, cy, Rt of each call), the
pre-render gradients (a seeded linear functional of the per-Gaussian outputs, with respect to the first and last
parameter of encoder, geomdecoder and decoder), the post-render gradients (a seeded cotangent on rgb, with respect to
the rendered images, cal.holder.params and learn_blur.weights_raw), and for each the fp32 run's norm-wise error
against the fp64 run.  Nothing of the reference is copied and no weights are stored.

Needs /root/reference; the .npz is committed.   Usage: python tests/golden/make_head_frame_golden.py
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
OUT = os.path.join(HERE, "head_frame_ref.npz")
SRC = "/root/reference/ca_code/models/rgca.py"
CLASSES = ("AutoEncoder", "Encoder", "GeomDecoder", "PrimDecoder")


def scale_slab(seg, slab):
    """PrimDecoder's source at a slab of `slab` instead of 1024"""
    import re

    f = 1024 // slab
    seg = re.sub(r"ub=\((\d+), (\d+)\)", lambda m: "ub=(%d, %d)" % (int(m[1]) // f, int(m[2]) // f), seg)
    seg = seg.replace("1024", str(slab)).replace("8 * 8", "%d * %d" % (8 // f, 8 // f))
    return seg.replace("256, 8, 8)", "256, %d, %d)" % (8 // f, 8 // f)).replace("-1, -1, 8, 8)", "-1, -1, %d, %d)"
                                                                                  % (8 // f, 8 // f))


def light_statements(src):
    """the statements of AutoEncoder.forward from `light_intensity = ...expand` up to the encoder call"""
    tree = ast.parse(src)
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "AutoEncoder"][0]
    fwd = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "forward"][0]
    body = fwd.body
    i0 = [i for i, s in enumerate(body) if "expand" in ast.get_source_segment(src, s)][0]
    i1 = [i for i, s in enumerate(body) if "self.encoder" in ast.get_source_segment(src, s)][0]
    stmts = body[i0:i1]
    print("light statements: reference lines %d-%d" % (stmts[0].lineno, stmts[-1].end_lineno))
    return "\n".join(ast.get_source_segment(src, s) for s in stmts)


class _Oracle:
    """render_gs and evaluate_gaussian on the C oracles; records each render call"""

    def __init__(self):
        import oracle

        oracle.lib()
        self.o, self.calls = oracle, []

    def render(self, cam_img_w, cam_img_h, fx, fy, cx, cy, Rt, primpos, primqvec, primscale, opacity, colors,
               return_depth=True, **kw):
        n = lambda t: np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32))
        H, W, dt = cam_img_h, cam_img_w, primpos.dtype
        p = self.o.project_fwd(n(primpos.reshape(-1, 3)), n(primscale.reshape(-1, 3)), 1.0, n(primqvec.reshape(-1, 4)),
                               n(Rt), fx, fy, cx, cy, H, W, 16, 0.1)
        b = self.o.bin_and_sort(p["xys"], p["depths"], p["radii"], p["num_tiles_hit"], H, W, 16)
        op = n(opacity.reshape(-1)) * p["compensation"]
        blend = lambda c: self.o.rasterize_fwd(H, W, 16, b["gaussian_ids_sorted"], b["tile_bins"], p["xys"],
                                               p["conics"], np.ascontiguousarray(c, np.float32), op,
                                               np.zeros(3, np.float32))
        img, Ts, _ = blend(n(colors.reshape(-1, 3)))
        dimg = blend(np.repeat(p["depths"][:, None], 3, 1))[0]
        rgb = th.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1))).to(dt).requires_grad_()
        self.calls.append({"fx": fx, "fy": fy, "cx": cx, "cy": cy, "Rt": n(Rt), "render": rgb})
        return {"render": rgb, "final_T": th.from_numpy(np.asarray(Ts)).to(dt)[None],
                "depth": th.from_numpy(np.ascontiguousarray(dimg[..., 0])).to(dt)[None]}

    def evaluate_gaussian(self, lobe_dirs, lobe_sigmas, light_values, light_pts, prim_pts, n_lights, w_type=0,
                          normalize_lobe_dirs=True):
        import torch.nn.functional as F

        if normalize_lobe_dirs:
            lobe_dirs = F.normalize(lobe_dirs, dim=-1)
        o = self.o

        class SG(th.autograd.Function):
            @staticmethod
            def forward(ctx, dirs, sig, vals):
                n = lambda t: t.detach().cpu().numpy()
                ctx.a = (n(dirs), n(sig), n(vals), n(light_pts), n(prim_pts), n(n_lights))
                ctx.dt = dirs.dtype
                return th.from_numpy(o.sg_fwd(*ctx.a, w_type=w_type)).to(dirs.dtype)

            @staticmethod
            def backward(ctx, g):
                gd, gs, gl = o.sg_bwd(*ctx.a, g.detach().cpu().numpy(), w_type=w_type)
                f = lambda x: th.from_numpy(x).to(ctx.dt)
                return f(gd), f(gs).reshape(ctx.a[1].shape), f(gl)

        return SG.apply(lobe_dirs, lobe_sigmas, light_values)


def run(model, inp, dtype, hr, orc, names):
    """one forward of the reference frame in `dtype`: outputs, render calls, pre- and post-render gradients"""
    model = model.to(dtype)
    cast = {k: (v.to(dtype) if th.is_tensor(v) and v.is_floating_point() else
                [x.to(dtype) for x in v] if isinstance(v, list) and v and th.is_tensor(v[0]) else v)
            for k, v in inp.items()}
    orc.calls = []
    preds = model(**cast)
    params = dict(model.named_parameters())
    w = hr.functional_weights(preds)
    f = sum((preds[k] * w[k].to(dtype)).sum() for k in hr.PRIM_KEYS)
    pre = th.autograd.grad(f, [params[n] for n in names], retain_graph=True, allow_unused=True)
    pre = {n: (g if g is not None else th.zeros_like(params[n])) for n, g in zip(names, pre)}
    renders = th.stack([c["render"] for c in orc.calls])                       # [n_calls, 3, H, W]
    post_leaves = {"renders": [c["render"] for c in orc.calls]}
    targets = list(post_leaves["renders"])
    extra = [k for k in ("cal.holder.params", "learn_blur.weights_raw") if k in params]
    cot = hr.rgb_cotangent(preds["rgb"].shape).to(dtype)
    gr = th.autograd.grad((preds["rgb"] * cot).sum(), targets + [params[k] for k in extra], allow_unused=True)
    post = {"renders": th.stack([g if g is not None else th.zeros_like(r) for g, r in zip(gr, renders)])}
    post.update({k: g for k, g in zip(extra, gr[len(targets):])})
    args = {"intrinsics": np.array([[c["fx"], c["fy"], c["cx"], c["cy"]] for c in orc.calls]),
            "Rt": np.stack([c["Rt"] for c in orc.calls])}
    return preds, pre, post, args


def run_mode(ns, hr, a, mode, d):
    orc = _Oracle()
    ns["render_gs"], ns["evaluate_gaussian"] = orc.render, orc.evaluate_gaussian
    th.manual_seed(0)
    cfg = hr.mode_config(mode)
    cfg["decoder"].pop("slabsize", None)
    model = ns["AutoEncoder"](**cfg, assets=a)
    hr.seeded_fill(model)
    model.train(mode == "train")
    inp = hr.mode_inputs(mode)
    names = hr.grad_param_names(model)
    model32 = copy.deepcopy(model)
    th.manual_seed(1)
    p64, pre64, post64, args = run(model, inp, th.float64, hr, orc, names)
    th.manual_seed(1)
    p32, pre32, post32, _ = run(model32, inp, th.float32, hr, orc, names)
    d["%s_out_keys_json" % mode] = np.frombuffer(json.dumps(sorted(p64)).encode(), dtype=np.uint8)
    d["%s_grad_names_json" % mode] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
    d["%s_args_intrinsics" % mode], d["%s_args_Rt" % mode] = args["intrinsics"], args["Rt"]
    for kind, A64, A32 in (("out", p64, p32), ("pre", pre64, pre32), ("post", post64, post32)):
        for k in A64:
            if not th.is_tensor(A64[k]) or (kind == "out" and k in hr.RANDOM_KEYS):
                continue
            s64, s32 = hr.summarise(A64[k]), hr.summarise(A32[k])
            d["%s_%s_%s" % (mode, kind, k)] = s64
            d["%s_shape_%s_%s" % (mode, kind, k)] = np.array(A64[k].shape)
            d["%s_err32_%s_%s" % (mode, kind, k)] = np.float64(hr.nrel_summary(s32, s64))
            print("%-6s %-4s %-32s |max| %.3e  fp32 err %.2e" % (mode, kind, k, s64[2],
                                                                  d["%s_err32_%s_%s" % (mode, kind, k)]))
    print("%s: coverage %.2f" % (mode, float((p64["alpha"] > 0).double().mean())))


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, "/root/reference")
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    warnings.filterwarnings("ignore")
    from make_lbs_golden import _stub

    _stub()
    import head_frame_restate as hr
    import torch.nn.functional as F

    import ca_code.nn.layers as la
    from ca_code.utils.envmap import compose_envmap, dir2uv
    from ca_code.utils.mipmap_sampler import mipmap_grid_sample
    import ca_code.utils.geom as geom
    import ca_code.utils.sh as sh
    from ca_code.nn.color_cal import CalV5
    from ca_code.nn.dof_cal import LearnableBlur
    from ca_code.nn.layers import make_conv_trans, make_linear

    a = hr.assets()
    geom.make_uv_vert_index = lambda vt, vi, vti, uv_shape, flip_uv=False: th.as_tensor(a.index_image)
    geom.make_uv_barys = lambda vt, vti, uv_shape, flip_uv=False: (th.as_tensor(a.face_index_image),
                                                                    th.as_tensor(a.bary_image))
    src = open(SRC).read()
    ns = {"th": th, "nn": th.nn, "np": np, "F": F, "la": la, "sh": sh, "math": __import__("math"),
          "make_conv_trans": make_conv_trans, "make_linear": make_linear, "CalV5": CalV5,
          "LearnableBlur": LearnableBlur, "GeometryModule": geom.GeometryModule,
          # envmap_to_mirrorball builds its rays in fp32, so the fp64 run hands it the cameras in fp32
          "compose_envmap": lambda render, alpha, envbg, K, Rt: compose_envmap(render, alpha, envbg.float(), K.float(),
                                                                               Rt.float()),
          "dir2uv": dir2uv, "mipmap_grid_sample": mipmap_grid_sample,
          "logger": logging.getLogger("rgca"), "primscale_range": (0.1, 20.0), **vars(typing)}
    for node in ast.parse(src).body:
        if isinstance(node, ast.ClassDef) and node.name in CLASSES:
            seg = ast.get_source_segment(src, node)
            if node.name == "PrimDecoder":
                seg = scale_slab(seg, hr.SLAB)
            exec(seg, ns)
    cfg = hr.config()
    cfg["decoder"].pop("slabsize", None)
    th.manual_seed(0)
    model = ns["AutoEncoder"](**cfg, assets=a)
    d = {"keys_json": np.frombuffer(json.dumps({k: list(v.shape) for k, v in model.state_dict().items()},
                                               sort_keys=True).encode(), dtype=np.uint8)}
    print("%d state-dict keys" % len(model.state_dict()))

    text = light_statements(src)
    for tag, C in (("c1", 1), ("c3", 3)):
        inp = hr.inputs(C=C)
        g = th.Generator().manual_seed(7 + C)
        lightrot = th.stack([hr.rotation(th.randn(3, generator=g, dtype=th.float64), 0.5 + b) for b in range(2)])
        lightrot = lightrot.float().double()        # the kernel's fp32 input
        loc = {k: inp[k].to(th.float64) for k in ("head_pose", "campos", "Rt", "light_pos", "light_intensity")}
        loc.update(lightrot=lightrot, self=type("S", (), {"n_diff_sh": 8})(), th=th, F=F, sh=sh)
        exec(text, loc)
        for k in ("head_pose", "campos", "Rt", "light_pos", "light_intensity"):
            d["%s_in_%s" % (tag, k)] = inp[k].numpy()
        d["%s_in_lightrot" % tag] = lightrot.float().numpy()
        for k in ("headrel_Rt", "headrel_campos", "headrel_light_pos", "headrel_light_sh", "lightrot"):
            d["%s_out_%s" % (tag, k)] = loc[k].numpy()
        print("%s: |headrel_light_sh| max %.3e" % (tag, float(loc["headrel_light_sh"].abs().max())))
    for mode in hr.MODES:
        run_mode(ns, hr, a, mode, d)
    np.savez_compressed(OUT, **d)
    print("-> %s (%.0f kB)" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
