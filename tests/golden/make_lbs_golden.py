"""Generate tests/golden/lbs_ref.npz by RUNNING the reference's own code on CPU in fp64:

  * LinearBlendSkinning / LBSModule imported from ca_code.utils.lbs (the bind state recomputed in fp64);
  * compute_tbn, make_postex, compute_view_cos and values_to_uv imported from ca_code.utils.geom (pytorch3d stubbed);
  * hand_mvp's GeomDecoder class, init_primitives and axisangle_to_matrix sliced out of the file's AST at run time, as
    make_hand_mvp_golden.py does; TransDecoder / DeconvContentDecoder likewise.
Inputs come from tests/lbs_recipe.py (seeded); only outputs (float32) are stored.

Needs /root/reference; the .npz is committed.   Usage: python tests/golden/make_lbs_golden.py
"""
import json
import os
import sys
import warnings
from unittest.mock import MagicMock

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "lbs_ref.npz")
SRC = "/root/reference/ca_code/models/hand_mvp.py"
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import lbs_recipe as R  # noqa: E402
from make_hand_mvp_golden import _slice  # noqa: E402

B = 2


def _stub():
    for name in ("pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh", "pytorch3d.renderer.mesh.rasterize_meshes",
                 "pytorch3d.structures", "sklearn", "sklearn.neighbors"):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = MagicMock()


def _lbs64(model, cfg, template, scales):
    """template [V,3] (what template_pose expects) or [1,V,3] (what hand_mvp.AutoEncoder passes)"""
    from ca_code.utils.lbs import LBSModule, solve_skeleton_state

    m = LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0])
    ref_state = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.double()
    f = m.lbs_fn
    zero = th.zeros(1, f.param_transform.nr_total_params, dtype=th.float64)
    f.bind_state = solve_skeleton_state(f.param_transform(zero), f.joint_offset, f.joint_rotation, f.joint_parents)
    return m, ref_state


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, "/root/reference")
    warnings.filterwarnings("ignore")
    _stub()
    sys.modules.setdefault("turtle", MagicMock())
    import ca_code.nn.layers as la
    from ca_code.nn.blocks import ConvBlock, tile2d
    from ca_code.utils import geom
    from ca_code.utils.lbs import LBSModule, solve_skeleton_state, states_to_matrix

    d = {}
    # (1) skeletons: matrices, states, skinning (batch-1 and batch-B vertices) with the autograd gradient
    for i, kind in enumerate(R.SKELETONS):
        model, cfg, template, scales = R.skinned_model(kind, 100 + i)
        m, ref_state = _lbs64(model, cfg, template, scales)
        mo = R.motion(B, 200 + i).double()
        f = m.lbs_fn
        params = f.param_transform(th.cat([mo, m.lbs_scale.expand(B, -1)], 1))
        states = solve_skeleton_state(params, f.joint_offset, f.joint_rotation, f.joint_parents)
        d[kind + "_states"] = states
        d[kind + "_mats"] = states_to_matrix(f.bind_state, states)
        d[kind + "_bind"] = f.bind_state
        V = f.num_verts
        g = th.Generator().manual_seed(300 + i)
        for vb in (1, B):
            vu = (0.1 * th.randn(vb, V, 3, generator=g)).double().requires_grad_()
            out = m.pose(vu, mo)
            w = th.randn(out.shape, generator=g).double()
            (gv,) = th.autograd.grad((out * w).sum(), [vu])
            d["%s_pose%d" % (kind, vb)], d["%s_gv%d" % (kind, vb)] = out, gv
        if kind == "tree24":
            d[kind + "_template_pose"] = m.template_pose(mo)
        if kind == "tree24":
            d["state_keys"] = np.array(json.dumps({k: [list(v.shape), str(v.dtype)] for k, v in ref_state.items()}))
            d["lbs_fn_keys"] = np.array(json.dumps(list(m.lbs_fn.state_dict().keys())))

    # (2) hand GeomDecoder at full size (uv 1024, 4096 primitives) on the tube mesh, eval and training warm start
    src = open(SRC).read()
    import ast

    tree = ast.parse(src)
    ns = {"th": th, "nn": th.nn, "la": la, "ConvBlock": ConvBlock, "tile2d": tile2d, "Tuple": tuple,
          "F": th.nn.functional, "make_postex": geom.make_postex, "compute_tbn": geom.compute_tbn}
    for name in ("TransDecoder", "DeconvContentDecoder", "GeomDecoder"):
        exec(_slice(tree, src, cls=name), ns)
    for fn in ("axisangle_to_matrix", "init_primitives"):
        exec(_slice(tree, src, func=fn), ns)

    model, cfg, template, scales = R.tube_model(7)
    lbs, _ = _lbs64(model, cfg, template[None], scales)
    geo = R.TubeGeometry(dtype=th.float64)
    th.manual_seed(0)
    dec = ns["GeomDecoder"](8, 2, 1024, 4096, lbs, geo, primposstart=1000).double()
    R.init_weights(dec.transdecoder, 11)
    R.init_weights(dec.alphadecoder, 12)
    pose = R.motion(B, 21).double()
    joint = th.randn(B, 8, 64, 64, generator=th.Generator().manual_seed(22)).double()
    dec.eval()
    with th.no_grad():
        p = dec(pose, joint, iteration=5000)
        dec.train()
        pt = dec(pose[:1], joint[:1], iteration=0)
    for k in ("primpos", "primrot", "primscale", "geom_lbs"):
        d["gd_" + k] = p[k]
    d["gdt_primpos"], d["gdt_primrot"], d["gdt_primscale"] = pt["primpos"], pt["primrot"], pt["primscale"]
    d["gd_alpha"] = p["primalpha"].reshape(-1)[R.alpha_sample(p["primalpha"].numel())]
    d["gd_vidx"] = dec.prim_vidx_img

    # (3) prim base frames and view cosine on the posed tube, with -1 vertex indices in a copy of the index image
    geom_lbs = p["geom_lbs"]
    vidx = R.with_negative_indices(dec.prim_vidx_img)
    g0 = geom_lbs[:1]  # frames of item 0 only (the fixture's size); the view cosine at B = 2
    postex = geom.make_postex(g0, vidx, dec.prim_bary_img).permute(0, 2, 3, 1).reshape(1, -1, 3)
    tbn = geom.compute_tbn(g0, geo.vt, vidx, dec.prim_vtidx_img)
    d["fr_posbase"] = postex
    d["fr_rotbase"] = th.stack(tbn, dim=-2).reshape(1, -1, 3, 3).permute(0, 1, 3, 2)
    vc = geom.compute_view_cos(geom_lbs, geo.vi.long(), R.CAMPOS.double())
    d["fr_view_cos_uv"] = geom.values_to_uv(vc[..., None], vidx, dec.prim_bary_img)

    out = {}
    for k, v in d.items():
        if isinstance(v, th.Tensor):
            v = v.detach().numpy()
            out[k] = v.astype(np.float32) if v.dtype == np.float64 else v.astype(np.int32)
        else:
            out[k] = v
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
    nan = np.isnan(out["gd_primrot"]).any(axis=(2, 3))
    print("NaN primitives:", np.argwhere(nan).tolist()[:4], "alpha > 0:", float((d["gd_alpha"] > 0).double().mean()))


if __name__ == "__main__":
    main()
