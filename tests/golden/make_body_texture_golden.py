"""Generate tests/golden/body_texture_ref.npz by RUNNING the reference's own texture branch of the body avatar on CPU in
fp64, at the mesh_vae_example.yml configuration (decoder_view.net_uv_size 1024, upscale_net.n_ftrs 4, shadow_net
uv_size 2048 / shadow_size 256 / n_dims 4, interp_mode "bilinear", biases False), B = 2:

  `UNetWB` and `ShadowUNet` are imported from the reference's ca_code.nn (turtle stubbed, as make_mesh_vae_golden.py
  does); `UNetViewDecoder`, `UpscaleNet` and `AutoEncoder.forward_tex` are sliced out of mesh_vae.py's AST at run time,
  and forward_tex is bound to a module holding the reference's `SeamSampler` on seams_restate.synthetic_seams(1024)
  and (2048).  The view cosine runs on the reference's compute_view_cos / values_to_uv over the UV-gridded mesh of
  tests/body_texture_restate.uv_mesh, whose index image has uncovered texels.  Nothing of the reference is copied.

Frozen: the state-dict keys and shapes and parameter counts of the five modules, the initialisation properties of the
reference's ShadowUNet and UNetWB, statistics + 256 evenly spaced samples of every output, and of the gradients of a
fixed random cotangent of tex_rec with respect to forward_tex's three inputs, to tex_mean_rec through the whole
branch, and to every parameter.  The torch restatement (tests/body_texture_restate.py) is checked against the
reference here and against the fixture in tests/test_body_texture_cpu.py.

Needs /root/reference; the .npz is committed.   Usage: python tests/golden/make_body_texture_golden.py
"""
import ast
import json
import os
import sys
import textwrap
import types
import warnings
from unittest.mock import MagicMock

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "body_texture_ref.npz")
SRC = "/root/reference/ca_code/models/mesh_vae.py"


def summarise(t):
    f = t.detach().double().reshape(-1)
    idx = th.linspace(0, f.numel() - 1, 256, dtype=th.float64).long()
    return np.concatenate([[f.mean().item(), f.std().item(), f.abs().max().item(), float(f.numel())], f[idx].numpy()])


def keys_of(m):
    return {k: list(v.shape) for k, v in m.state_dict().items()}


def main():
    if not os.path.isfile(SRC):
        sys.exit("needs /root/reference (build container only)")
    sys.path.insert(0, "/root/reference")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    warnings.filterwarnings("ignore")
    for name in ("turtle", "pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.mesh",
                 "pytorch3d.renderer.mesh.rasterize_meshes", "pytorch3d.structures"):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = MagicMock()
    th.set_default_dtype(th.float64)
    import ca_code.nn.layers as la
    import torch.nn.functional as F
    from ca_code.nn.shadow import ShadowUNet
    from ca_code.nn.unet import UNetWB
    from ca_code.utils.geom import compute_view_cos, values_to_uv
    from ca_code.utils.seams import SeamSampler

    import body_texture_restate as bt

    src = open(SRC).read()
    tree = ast.parse(src)
    seg = {n.name: ast.get_source_segment(src, n) for n in tree.body if isinstance(n, ast.ClassDef)}
    ns = {"th": th, "nn": th.nn, "np": np, "la": la, "F": F, "UNetWB": UNetWB, "compute_view_cos": compute_view_cos}
    exec(seg["UNetViewDecoder"], ns)
    exec(seg["UpscaleNet"], ns)
    ae = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "AutoEncoder")
    ft_src = next(ast.get_source_segment(src, f) for f in ae.body if isinstance(f, ast.FunctionDef)
                  and f.name == "forward_tex")
    exec(textwrap.dedent(ft_src), ns)

    inp = bt.seeded_inputs()
    vi, _, idx_img, bary_img = bt.uv_mesh()
    s1k, s2k = ({k: v.double() if v.is_floating_point() else v for k, v in s.items()} for s in bt.seams())
    th.manual_seed(0)

    # ---- the reference modules, built as AutoEncoder builds them (mesh_vae.py:154-174)
    geo_fn = types.SimpleNamespace(vi=vi, to_uv=lambda v: values_to_uv(v, idx_img, bary_img))
    view_ref = ns["UNetViewDecoder"](geo_fn, net_uv_size=bt.UV, seam_sampler=None, n_init_ftrs=8)
    shadow_ref = ShadowUNet(uv_size=bt.UV2K, ao_mean=inp["ao_mean"], shadow_size=bt.SHADOW, n_dims=4,
                            interp_mode="bilinear", biases=False)
    comp_ref = th.nn.Module()
    comp_ref.upscale_net = ns["UpscaleNet"](in_channels=6, size=1024, upscale_factor=2, out_channels=3, n_ftrs=4)
    comp_ref.seam_sampler = SeamSampler(s1k)
    comp_ref.seam_sampler_2k = SeamSampler(s2k)
    comp_ref.register_buffer("tex_mean", inp["tex_mean"].clone())
    comp_ref.tex_std = bt.TEX_STD
    forward_tex = types.MethodType(ns["forward_tex"], comp_ref)
    unet_ref = UNetWB(4, 3, size=bt.UV)

    d = {}
    mods = {"unet": unet_ref, "shadow": shadow_ref, "view": view_ref, "upscale": comp_ref.upscale_net,
            "composer": comp_ref}
    for k, m in mods.items():
        d["keys_" + k] = np.frombuffer(json.dumps(keys_of(m), sort_keys=True).encode(), dtype=np.uint8)
        d["n_params_" + k] = np.int64(sum(p.numel() for p in m.parameters()))
    assert int(d["n_params_unet"]) == 19_879_839

    # ---- initialisation of the reference classes
    props = []
    for name, m in sorted(shadow_ref.named_modules()):
        if hasattr(m, "weight_v"):
            v, g = m.weight_v.detach(), m.weight_g.detach()
            fan_in = v[0].numel()
            props.append([float(v.abs().max()) * fan_in ** 0.5, float((g - v.norm()).abs().max() / v.norm()),
                          float(m.bias.abs().max()) if m.bias is not None else 0.0,
                          float(v.std()) * (3 * fan_in) ** 0.5])
    d["shadow_init"] = np.array(props)  # per layer: max|v| sqrt(fan_in), |g - ||v||| / ||v||, max|bias|, std-derived bound
    props = []
    for name, m in sorted(unet_ref.named_modules()):
        if hasattr(m, "weight_v"):
            w = m.weight.detach() if hasattr(m, "weight") else None
            v = m.weight_v.detach()
            props.append([float((w - v).abs().max() / v.abs().max()), float(m.bias.abs().max())])
    d["unet_init"] = np.array(props)

    # ---- seeded parameters on both sides; the restatement must load the reference's state dicts strictly
    seeds = {"shadow": 101, "view": 102, "upscale": 103}
    ours = {"shadow": bt.ShadowUNet(bt.UV2K, inp["ao_mean"], bt.SHADOW, n_dims=4, biases=False),
            "view": bt.UNetViewDecoder(vi, idx_img, bary_img, bt.UV),
            "upscale": bt.UpscaleNet(6, 3, 4)}
    for k in seeds:
        bt.seeded_fill(mods[k], seeds[k])
        ours[k].load_state_dict(mods[k].state_dict(), strict=True)
    ts1 = bt.sr.TorchSeamSampler(*(s1k[k] for k in ("dst_ij", "src_ij", "uvs", "weights")))
    ts2 = bt.sr.TorchSeamSampler(*(s2k[k] for k in ("dst_ij", "src_ij", "uvs", "weights")))
    comp_ours = bt.TextureComposer(ts1, ts2, inp["tex_mean"].clone())
    comp_ours.upscale_net = ours["upscale"]
    th.set_num_threads(os.cpu_count() or 1)

    def branch(view, shadow, ft, standalone_upscale):
        tmr = inp["tex_mean_rec"].clone().requires_grad_()
        vo = view(geom_rec=inp["geom_rec"], tex_mean_rec=tmr, camera_pos=inp["camera_pos"])
        so = shadow(inp["ao_map"])
        tvr = vo["tex_view_rec"].detach().requires_grad_()
        smap = so["shadow_map"].detach().requires_grad_()
        tmr2 = tmr.detach().requires_grad_()
        tex_rec = ft(tmr2, tvr, smap.clone())   # the reference impaints its shadow_map argument in place
        up = standalone_upscale(th.cat([tmr2, tvr], 1).detach())
        out = {"tex_view_rec": vo["tex_view_rec"], "cond_view": vo["cond_view"], "shadow_map": so["shadow_map"],
               "ao_map": so["ao_map"], "shadow_map_lowres": so["shadow_map_lowres"], "tex_rec": tex_rec,
               "upscale": up}
        gen = th.Generator().manual_seed(77)
        w = th.randn(tex_rec.shape, generator=gen)
        g_tmr2, g_tvr, g_smap = th.autograd.grad((tex_rec * w).sum(), [tmr2, tvr, smap], retain_graph=True)
        grads = {"ft_tex_mean_rec": g_tmr2, "ft_tex_view_rec": g_tvr, "ft_shadow_map": g_smap}
        # the whole branch: forward_tex's input gradients pushed through the view decoder and the shadow net
        params = ([("view." + n, p) for n, p in view.named_parameters()]
                  + [("shadow." + n, p) for n, p in shadow.named_parameters()])
        ft_params = [("composer.upscale_net." + n, p) for n, p in ft_upscale(ft).named_parameters()]
        gp = th.autograd.grad((tex_rec * w).sum(), [p for _, p in ft_params])
        gr = th.autograd.grad([vo["tex_view_rec"], so["shadow_map"]], [tmr] + [p for _, p in params],
                              grad_outputs=[g_tvr, g_smap], allow_unused=True)
        grads["tex_mean_rec"] = gr[0] + g_tmr2
        for (n, _), g in zip(params + ft_params, list(gr[1:]) + list(gp)):
            grads["p." + n] = g
        return out, grads

    def ft_upscale(ft):
        return ft.__self__.upscale_net if isinstance(ft, types.MethodType) else ft.upscale_net

    r_out, r_grads = branch(view_ref, shadow_ref, forward_tex, comp_ref.upscale_net)
    o_out, o_grads = branch(ours["view"], ours["shadow"], comp_ours, ours["upscale"])
    for kind, R, O in (("out", r_out, o_out), ("g", r_grads, o_grads)):
        for k in R:
            err = float((R[k] - O[k]).abs().max() / R[k].abs().max().clamp_min(1e-300))
            assert R[k].shape == O[k].shape and err < 1e-12, (kind, k, err)
            d[kind + "_" + k] = summarise(R[k])
            d["shape_" + kind + "_" + k] = np.array(R[k].shape)
        print("%s: %d tensors, restatement == reference to 1e-12" % (kind, len(R)))
    np.savez_compressed(OUT, **d)
    print("-> %s (%.0f kB)" % (OUT, os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
