"""Generate tests/golden/body_encoder_ref.npz by RUNNING the reference's own code on CPU:

  * `Encoder` / `FaceEncoder` are sliced out of /root/reference/ca_code/models/mesh_vae.py by AST at run time (the
    module cannot be imported: drtk / pytorch3d are absent) and built on the reference's own
    `ca_code.nn.blocks.ConvDownBlock` and `ca_code.nn.layers` — nothing is copied into this repository — at the
    mesh_vae_example.yml sizes (n_embs 1024, face 256), with a seeded mask and a seeded UV position map;
  * `LBSModule.unpose` / `LinearBlendSkinning.unskinning` are imported from ca_code.utils.lbs and run in fp64 on the
    synthetic skeleton of tests/lbs_recipe.py.
The restatement tests/body_encoder_restate.py gets the same seeded parameters and inputs; the script asserts that the
two agree and freezes (a) the reference's state-dict keys and shapes, (b) the eval() outputs at B = 1 and 2, (c) the
gradients of a seeded linear functional w.r.t. a few named parameters, (d) the unposed vertices with the condition
number of each vertex's blended matrix.

Needs /root/reference; the .npz is committed.   Usage: python tests/golden/make_body_encoder_golden.py
"""
import ast
import json
import os
import sys
import warnings
from typing import Dict
from unittest.mock import MagicMock

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "body_encoder_ref.npz")
SRC = "/root/reference/ca_code/models/mesh_vae.py"
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import body_encoder_restate as br  # noqa: E402
import lbs_recipe as R  # noqa: E402
from make_lbs_golden import _lbs64, _stub  # noqa: E402

N_EMBS, N_FACE_EMBS = 1024, 256   # mesh_vae_example.yml
KEYS = ("embs", "embs_mu", "embs_logvar")


def functional(preds, prefix, seed):
    """the seeded linear functional whose parameter gradients the fixture keeps"""
    g = th.Generator().manual_seed(seed)
    return sum((preds[prefix + k] * th.randn(preds[prefix + k].shape, generator=g)).sum() for k in KEYS[1:])


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, "/root/reference")
    warnings.filterwarnings("ignore")
    _stub()
    sys.modules.setdefault("turtle", MagicMock())
    import ca_code.nn.layers as la
    from ca_code.nn.blocks import ConvDownBlock

    src = open(SRC).read()
    ns = {"th": th, "nn": th.nn, "np": np, "la": la, "F": th.nn.functional, "ConvDownBlock": ConvDownBlock, "Dict": Dict}
    for node in ast.parse(src).body:
        if isinstance(node, ast.ClassDef) and node.name in ("Encoder", "FaceEncoder"):
            exec(ast.get_source_segment(src, node), ns)

    mask = br.synthetic_mask()
    d = {}
    th.set_num_threads(os.cpu_count() or 1)
    for name, prefix, ref, ours in (
            ("encoder", "", ns["Encoder"](n_embs=N_EMBS, mask=mask), br.Encoder(n_embs=N_EMBS, mask=mask)),
            ("encoder_face", "face_", ns["FaceEncoder"](mask=mask, n_embs=N_FACE_EMBS),
             br.FaceEncoder(mask=mask, n_embs=N_FACE_EMBS))):
        keys_ref = {k: [list(v.shape), str(v.dtype)] for k, v in ref.state_dict().items()}
        keys_ours = {k: [list(v.shape), str(v.dtype)] for k, v in ours.state_dict().items()}
        assert keys_ref == keys_ours, set(map(str, keys_ref.items())) ^ set(map(str, keys_ours.items()))
        d[name + "_keys_json"] = np.frombuffer(json.dumps(keys_ref, sort_keys=True).encode(), dtype=np.uint8)
        br.seeded_fill(ref)
        ours.load_state_dict(ref.state_dict())     # the reference's own state dict loads, buffers included
        ref.eval(), ours.eval()
        for B in (1, 2):
            uv = br.seeded_uv(B)
            r, o = ref(uv), ours(uv)
            for k in KEYS:
                err = (r[prefix + k] - o[prefix + k]).abs().max().item() / r[prefix + k].abs().max().item()
                assert err < 2e-5, (name, k, err)
                d["%s_B%d_%s" % (name, B, k)] = r[prefix + k].detach().numpy()
            print("%-13s B=%d  |embs_mu| max %.3f  |embs_logvar| max %.3f" % (
                name, B, r[prefix + "embs_mu"].abs().max(), r[prefix + "embs_logvar"].abs().max()))
            if B == 2:
                pr = dict(ref.named_parameters())
                po = dict(ours.named_parameters())
                sub = "encoder." if prefix else ""
                gr = th.autograd.grad(functional(r, prefix, 5), [pr[sub + n] for n in br.GRAD_PARAMS])
                go = th.autograd.grad(functional(o, prefix, 5), [po[sub + n] for n in br.GRAD_PARAMS])
                for n, a, b in zip(br.GRAD_PARAMS, gr, go):
                    err = (a - b).norm().item() / a.norm().item()
                    assert err < 1e-4, (name, n, err)
                    d["%s_grad_%s" % (name, n)] = a.numpy()

    # unpose on the tree24 skeleton, fp64: registered vertices = a posed random mesh plus noise
    model, cfg, template, scales = R.skinned_model("tree24", 100)
    m, _ = _lbs64(model, cfg, template, scales)
    from ca_code.utils.lbs import solve_skeleton_state, states_to_matrix

    f = m.lbs_fn
    for B in (1, 3):
        mo = R.motion(B, 400 + B).double()
        g = th.Generator().manual_seed(500 + B)
        vu = (0.1 * th.randn(B, f.num_verts, 3, generator=g)).double()
        reg = (m.pose(vu, mo) + 0.01 * th.randn(B, f.num_verts, 3, generator=g).double()).float().double()
        out = m.unpose(reg, mo)
        back = m.pose(out, mo)
        assert (back - reg).abs().max() < 1e-8 * reg.abs().max(), "the reference's unpose does not invert its pose"
        states = solve_skeleton_state(f.param_transform(th.cat([mo, m.lbs_scale.expand(B, -1)], 1)), f.joint_offset,
                                      f.joint_rotation, f.joint_parents)
        mats = states_to_matrix(f.bind_state, states)
        ours = br.unskinning(mats, f.skin_indices, f.skin_weights, reg / m.global_scaling) - m.lbs_template_verts
        assert (ours - out).abs().max() < 1e-9 * out.abs().max().clamp_min(1.0), (ours - out).abs().max()
        d["unpose_B%d_in" % B] = reg.float().numpy()
        d["unpose_B%d_out" % B] = out.float().numpy()
        d["unpose_B%d_cond" % B] = th.linalg.cond(br.blended(mats, f.skin_indices, f.skin_weights)[..., :3]).float().numpy()
        print("unpose B=%d: |out| max %.2f, cond of the blended matrices: mean %.1f, max %.1f" % (
            B, out.abs().max(), d["unpose_B%d_cond" % B].mean(), d["unpose_B%d_cond" % B].max()))

    np.savez_compressed(OUT, **d)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
