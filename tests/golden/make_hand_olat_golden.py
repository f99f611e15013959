"""Generate tests/golden/hand_olat_ref.npz by RUNNING the reference's `OLATRGBDecoder` and `build_cam_rot_mat`
(ca_code/models/hand_teacher_mvp.py:28-46,159-554) on CPU in fp64, sliced out of the file's AST at run time as
make_hand_mvp_golden.py does (the module itself cannot be imported: drtk / torchvision extras are absent).  Only
three things are supplied around the reference's code:

  * `.cuda()` is the identity;
  * drtk's `transform` is the restatement v_cam = camrot (v - campos), pix = focal (x/z, y/z) + princpt, z kept;
  * the raymarcher runs `oracle.raymarch_fwd(with_shadow=True)` (fp32, the CPU oracle of the reference kernel) with
    the reference `Raymarcher`'s position scaling and `mvpraymarch`'s shadow normalisation, and `compute_raydirs` is
    `oracle.raydirs_fwd`.

Reduced size: primsize (8, 8, 4), 8 x 8 primitives, uv 64, 48^2 shadow images, B = 2, L = 7 (chunks of 5 + 2),
U-Net width 8 and 4 joint channels.  Stored for the warm-up (iteration 0) and the sigmoid branch (iteration 5000),
in training mode: inputs, the state dict, the light cameras and U-Net input of every chunk, primrgb, primshadow,
texolat, and the gradients of every parameter and of joint_feat under fixed upstream gradients of primrgb and
texolat.  Also: build_cam_rot_mat on lights on and off the y axis, the state-dict layout at the default size, and
the norm-wise error of the same reference code run in fp32 on the same inputs (`fp32_err`).

To keep the file small: parameters and the larger inputs are quantised (multiples of 1/256, 1/64 or 1/16, exact in
fp32), so they compress; image-shaped results (U-Net inputs, primrgb, primshadow, texolat and the untied-bias
gradients of the 64^2 and 32^2 layers) are stored on the texel lattice `lattice()` (every 9th row and column: 9 is
prime to the primitive size 8, so the 8 x 8 samples hit every primitive row and column and every in-primitive
offset (y', x') once).

Needs /root/reference and a built oracle; the .npz is committed.   Usage: python tests/golden/make_hand_olat_golden.py
"""
import ast
import copy
import json
import os
import sys
import warnings
from unittest.mock import MagicMock

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hand_olat_ref.npz")
SRC = "/root/reference/ca_code/models/hand_teacher_mvp.py"

B, L, S, VOLRADIUS = 2, 7, 48, 100.0
PRIMSIZE, NPX, NPY, UV = (8, 8, 4), 8, 8, 64
ENC, NINIT = [8] * 5, 4


def _top(tree, src, name):
    for node in tree.body:
        if isinstance(node, (ast.ClassDef, ast.FunctionDef)) and node.name == name:
            return ast.get_source_segment(src, node)
    raise KeyError(name)


def transform(v, campos, camrot, focal, princpt):
    vc = th.einsum("nij,npj->npi", camrot, v - campos[:, None])
    z = vc[..., 2:3]
    pix = th.einsum("nij,npj->npi", focal, vc[..., :2] / z) + princpt[:, None]
    return th.cat([pix, z], dim=-1)


def lattice(t):
    """every 9th texel row and column of an image-shaped array [..., H, W] with H, W >= 32; others unchanged"""
    return t[..., ::9, ::9] if t.ndim >= 2 and min(t.shape[-2:]) >= 32 else t


def upstream_grads(rgb_shape, texolat_shape):
    """Fixed upstream gradients of primrgb and texolat (numpy's legacy generator: the same numbers everywhere)."""
    rs = np.random.RandomState(77)
    return (th.from_numpy(rs.standard_normal(rgb_shape)), th.from_numpy(rs.standard_normal(texolat_shape)))


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, "/root/reference")
    sys.path.insert(0, ROOT)
    warnings.filterwarnings("ignore")
    sys.modules.setdefault("turtle", MagicMock())  # blocks.py imports it by accident; tkinter is absent here
    import ca_code.nn.layers as la

    import oracle

    th.Tensor.cuda = lambda self, *a, **k: self
    cams = []

    def compute_raydirs(viewpos, viewrot, focal, princpt, pixelcoords, volradius):
        cams.append((viewpos.clone(), viewrot.clone(), focal.clone(), princpt.clone()))
        n = lambda t: t.detach().numpy().astype(np.float32)
        out = oracle.raydirs_fwd(n(viewpos), n(viewrot), n(focal), n(princpt), n(pixelcoords), volradius)
        return tuple(th.from_numpy(o).to(th.get_default_dtype()) for o in out)

    class Raymarcher:
        def __init__(self, volradius, dt=1.0):
            self.volume_radius = volradius
            self.dt = dt / volradius

        def __call__(self, raypos, raydir, tminmax, decout, with_shadow=False):
            n = lambda t: t.detach().numpy().astype(np.float32)
            _, _, sh = oracle.raymarch_fwd(n(raypos), n(raydir), self.dt, n(tminmax),
                                           n(decout["primpos"] / self.volume_radius), n(decout["primrot"]),
                                           n(decout["primscale"]), n(decout["primrgba"]), None, with_shadow=True)
            shadow = sh[..., 0:1] / (sh[..., 1:] + np.float32(1e-5))
            return None, None, None, th.from_numpy(shadow).to(th.get_default_dtype())

    src = open(SRC).read()
    tree = ast.parse(src)
    ns = {"th": th, "nn": th.nn, "F": th.nn.functional, "la": la, "transform": transform,
          "compute_raydirs": compute_raydirs, "Optional": type(None).__class__, "logging": None}
    from typing import Optional
    ns["Optional"] = Optional
    exec(_top(tree, src, "build_cam_rot_mat"), ns)
    exec(_top(tree, src, "OLATRGBDecoder"), ns)
    Dec, build_cam_rot_mat = ns["OLATRGBDecoder"], ns["build_cam_rot_mat"]

    d = {}
    # state-dict layout at the default size (float32 to keep the 1024^2 untied biases small)
    big = Dec(1024, (16, 16, 8), 64, 64, Raymarcher(2000.0), 2000.0)
    d["layout_default"] = np.array(json.dumps([[k, list(v.shape)] for k, v in big.state_dict().items()]))
    del big

    th.set_default_dtype(th.float64)
    th.manual_seed(8123)
    f32 = lambda t: t.float().double()  # inputs representable in fp32, so the GPU side sees the same values

    # build_cam_rot_mat, lights off and on the y axis (the reference nudges a copy here)
    cpos = f32(th.randn(6, 3) * 300.0)
    cpos[1, 0] = cpos[1, 2] = 0.0
    cpos[4, 0], cpos[4, 2] = 0.0, 0.0
    ctr = f32(th.randn(6, 3) * 10.0)
    d["rot_campos"], d["rot_center"] = cpos.clone(), ctr
    d["rot_mat"] = build_cam_rot_mat(cpos.clone(), ctr)
    d["rot_mat_origin"] = build_cam_rot_mat(cpos.clone())

    rm = Raymarcher(VOLRADIUS)
    dec = Dec(UV, PRIMSIZE, NPX, NPY, rm, VOLRADIUS, n_init_channels=NINIT, n_enc_dims=ENC, shadow_img_size=S)
    for m in dec.modules():
        if hasattr(m, "weight_g"):
            m.weight_g.data.mul_(1.0 + 0.3 * th.randn_like(m.weight_g))
        if getattr(m, "bias", None) is not None:
            m.bias.data.normal_(0, 0.3)
    for n, p in dec.named_parameters():
        step = 256.0 if n.endswith("weight_v") else 64.0
        p.data = th.round(p.data * step) / step
    K = NPX * NPY
    q, _ = th.linalg.qr(th.randn(B, K, 3, 3))
    inp = {
        "campos": f32(th.randn(B, 3) * 300.0),
        "primpos": f32(th.randn(B, K, 3) * 22.0),
        "primrot": f32(q),
        "primscale": f32(8.0 + 6.0 * th.rand(B, K, 3)),
        "primalpha": th.round(th.randn(B, PRIMSIZE[2], 1, UV, UV).abs() * 64.0) / 16.0,
        "valid_prims": (th.rand(K) > 0.15).double(),
        "joint_feat": f32(th.randn(B, NINIT, UV // 16, UV // 16)),
        "light_pos": f32(th.nn.functional.normalize(th.randn(B, L, 3), dim=-1) * 400.0),
        "light_intensity": f32(th.rand(B, L, 3) * 2.0 + 0.1),
    }
    for k, v in inp.items():
        d["in_" + k] = v
    d["state_dict"] = np.array(json.dumps(sorted(dec.state_dict())))
    for k, v in dec.state_dict().items():
        d["sd_" + k] = v

    x_in = []

    def run(dec, inp):
        """both branches in training mode -> {name: result}; image-shaped results on the lattice"""
        r = {}
        hook = dec.enc_layers[0].register_forward_pre_hook(lambda mod, args: x_in.append(args[0].detach().clone()))
        dec.train()
        params = list(dec.named_parameters())
        for tag, it in (("warm", 0), ("sig", 5000)):
            cams.clear()
            x_in.clear()
            jf = inp["joint_feat"].clone().requires_grad_(True)
            out = dec(inp["campos"], None, None, inp["primpos"], inp["primrot"], inp["primscale"], inp["primalpha"],
                      inp["valid_prims"], jf, inp["light_pos"].clone(), inp["light_intensity"], it)
            w_rgb, w_tex = (w.to(th.get_default_dtype()) for w in upstream_grads(out["primrgb"].shape,
                                                                                  out["texolat"].shape))
            loss = (out["primrgb"] * w_rgb).sum() + (out["texolat"] * w_tex).sum()
            grads = th.autograd.grad(loss, [jf] + [p for _, p in params])
            r.update({tag + "_primrgb": lattice(out["primrgb"]), tag + "_texolat": lattice(out["texolat"]),
                      tag + "_g_joint_feat": grads[0]})
            for (n, _), g in zip(params, grads[1:]):
                r[tag + "_g_" + n] = lattice(g)
            # the features and primshadow do not depend on the branch: stored once
            assert len(x_in) == 2 and len(cams) == 2
            if tag == "warm":
                r["primshadow"] = lattice(out["primshadow"])
            assert th.equal(r["primshadow"], lattice(out["primshadow"]))
            for c, x in enumerate(x_in):
                if tag == "warm":
                    r["x%d" % c] = lattice(x)
                assert th.equal(r["x%d" % c], lattice(x))
            for c, (vp, vr, fc, pp) in enumerate(cams):
                r.update({"cam%d_pos" % c: vp, "cam%d_rot" % c: vr, "cam%d_focal" % c: fc, "cam%d_princpt" % c: pp})
        hook.remove()
        return r

    ref = run(dec, inp)
    d.update(ref)
    # The same reference code evaluated in fp32 on the same inputs and shadows: how far plain fp32 arithmetic of
    # this computation lands from fp64.  The U-Net gradients are long sums with cancellation, and their fp32 error
    # is several 1e-4 (norm-wise); the GPU parity test holds each result to a small multiple of this figure.
    th.set_default_dtype(th.float32)
    r32 = run(copy.deepcopy(dec).float(), {k: v.float() for k, v in inp.items()})
    d["fp32_err"] = np.array(json.dumps({k: float(((r32[k].double() - v).norm() / v.norm()).item())
                                         for k, v in ref.items() if v.norm() > 0}))

    out = {}
    for k, v in d.items():
        out[k] = v.detach().float().numpy() if isinstance(v, th.Tensor) else v
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
