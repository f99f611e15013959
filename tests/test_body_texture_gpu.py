"""GPU checks of the body avatar's texture branch (DESIGN.md row R9': csrc/body_tex.cu, goliath_b200/{unet,shadow,
mesh_vae}.py): the 2048^2 composite kernel against its fp64 torch formula at B = 1 and 4, each module against the fp64
restatement (tests/body_texture_restate.py) with seeded parameters loaded strictly, the whole branch against the
reference's fixture (tests/golden/body_texture_ref.npz), bitwise-repeatable TextureComposer gradients, and a
sync-free forward and backward with a graph replay equal to eager."""
import os
import types

import numpy as np
import pytest
import torch

import body_texture_restate as bt
from test_body_texture_cpu import _summary, restated_branch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "body_texture_ref.npz")


def _nrel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _maxrel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _no_tf32():
    class Ctx:
        def __enter__(self):
            self.s = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

        def __exit__(self, *a):
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.s

    return Ctx()


@pytest.mark.parametrize("B", [1, 4])
def test_compose_kernel_vs_fp64(cuda, B):
    from goliath_b200.mesh_vae import _TexCompose

    g = torch.Generator(device=cuda).manual_seed(B)
    H = 1024
    r = lambda *s: torch.randn(*s, device=cuda, generator=g)
    args = dict(t1=r(B, 3, H, H), h=r(B, 4, H, H), v=r(12, 4, 1, 1), g=0.5 + torch.rand(12, 1, 1, 1, device=cuda,
                generator=g), bias=0.1 * r(12, H, H), tex_mean=100 + 20 * r(1, 3, 2 * H, 2 * H),
                s3=torch.rand(B, 1, 2 * H, 2 * H, device=cuda, generator=g))
    w = r(B, 3, 2 * H, 2 * H)
    names = ("t1", "h", "v", "g", "bias", "s3")

    def run(fn, dtype):
        a = {k: t.to(dtype).requires_grad_(k in names) for k, t in args.items()}
        out = fn(a)
        return out.detach(), dict(zip(names, torch.autograd.grad((out * w.to(dtype)).sum(), [a[k] for k in names])))

    ref = lambda a: bt.compose(a["t1"], a["h"], a["v"], a["g"], a["bias"], bt.TEX_STD, a["tex_mean"], a["s3"])
    with _no_tf32():
        o64, g64 = run(ref, torch.float64)
        _, g32 = run(ref, torch.float32)
    ours = lambda a: _TexCompose.apply(a["t1"], a["h"], a["v"], a["g"], a["bias"], a["tex_mean"], a["s3"], bt.TEX_STD)
    out, gr = run(ours, torch.float32)
    _, gr2 = run(ours, torch.float32)
    assert _maxrel(out, o64) <= 1e-5
    for n in names:
        bound = max(1e-4, 4 * _nrel(g32[n], g64[n]))
        assert _nrel(gr[n], g64[n]) <= bound, (n, _nrel(gr[n], g64[n]), bound)
        assert torch.equal(gr[n], gr2[n]), n


def _check_grads(ours, ref64, ref32):
    out, g = ours
    o64, g64 = ref64
    _, g32 = ref32
    for k in o64:
        assert _maxrel(out[k], o64[k]) <= 1e-4, k
    assert set(g) == set(g64)
    bad = [(n, _nrel(g[n], g64[n]), max(1e-4, 4 * _nrel(g32[n], g64[n]))) for n in g64
           if _nrel(g[n], g64[n]) > max(1e-4, 4 * _nrel(g32[n], g64[n]))]
    assert not bad, bad


def _grads(module, inputs, outs, dtype, seed=3):
    module = module.to(dtype)
    xs = [x.to(dtype).requires_grad_(x.is_floating_point()) for x in inputs]
    res = module(*xs)
    res = res if isinstance(res, dict) else {"out": res}
    res = {k: res[k] for k in outs}
    gen = torch.Generator(device=xs[0].device).manual_seed(seed)
    loss = sum((v * torch.randn(v.shape, device=v.device, generator=gen).to(dtype)).sum() for v in res.values())
    leaves = [("x%d" % i, x) for i, x in enumerate(xs) if x.requires_grad] + list(module.named_parameters())
    gr = torch.autograd.grad(loss, [t for _, t in leaves], allow_unused=True)
    return {k: v.detach() for k, v in res.items()}, {n: t for (n, _), t in zip(leaves, gr) if t is not None}


def _vs_oracle(ours, ref, inputs, outs, ref_inputs=None):
    ref_inputs = inputs if ref_inputs is None else ref_inputs
    ours.load_state_dict(ref.state_dict(), strict=True)
    with _no_tf32():
        r64 = _grads(ref, ref_inputs, outs, torch.float64)
        r32 = _grads(ref, ref_inputs, outs, torch.float32)
    _check_grads(_grads(ours, inputs, outs, torch.float32), r64, r32)


def test_unet_vs_oracle(cuda):
    from goliath_b200.unet import UNetWB

    ref = bt.seeded_fill(bt.UNetWB(4, 3, 1024), 11).to(cuda)
    x = torch.randn(2, 4, 1024, 1024, device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))
    _vs_oracle(UNetWB(4, 3, 1024).to(cuda), ref, [x], ["out"])


@pytest.mark.parametrize("biases", [False, True])
def test_shadow_unet_vs_oracle(cuda, biases):
    from goliath_b200.shadow import ShadowUNet

    inp = bt.seeded_inputs(batch=2)
    ref = bt.seeded_fill(bt.ShadowUNet(2048, inp["ao_mean"], 256, n_dims=4, biases=biases), 12).to(cuda)
    ours = ShadowUNet(2048, inp["ao_mean"].float(), 256, n_dims=4, biases=biases).to(cuda)
    _vs_oracle(ours, ref, [inp["ao_map"].to(cuda)], ["shadow_map", "shadow_map_lowres"])


def test_upscale_net_vs_oracle(cuda):
    from goliath_b200.mesh_vae import UpscaleNet

    ref = bt.seeded_fill(bt.UpscaleNet(6, 3, 4), 13).to(cuda)
    x = torch.randn(2, 6, 1024, 1024, device=cuda, generator=torch.Generator(device=cuda).manual_seed(2))
    _vs_oracle(UpscaleNet(6, 3, 4).to(cuda), ref, [x], ["out"])


def test_view_decoder_vs_oracle(cuda):
    from goliath_b200.mesh_vae import UNetViewDecoder

    inp = bt.seeded_inputs(batch=2)
    vi, _, idx, bary = bt.uv_mesh()
    ref = bt.seeded_fill(bt.UNetViewDecoder(vi.to(cuda), idx.to(cuda), bary.to(cuda), 1024), 14).to(cuda)
    geo = _geo(cuda)
    ours = UNetViewDecoder(geo, 1024, None).to(cuda)
    args = [inp["geom_rec"].to(cuda).float(), inp["tex_mean_rec"].to(cuda).float(), inp["camera_pos"].to(cuda)]
    # the view cosine is under no_grad on both sides: geom_rec and camera_pos get no gradient
    _vs_oracle(ours, ref, [args[0].detach(), args[1], args[2]], ["tex_view_rec", "cond_view"])


def _geo(cuda):
    """duck-typed geo_fn, as the reference's UNetViewDecoder takes it (a submodule would add its buffers' keys)"""
    vi, _, idx, bary = bt.uv_mesh()
    return types.SimpleNamespace(vi=vi.to(cuda, torch.int32), index_image=idx.to(cuda), bary_image=bary.to(cuda))


def _our_branch(cuda):
    from goliath_b200.mesh_vae import TextureComposer, UNetViewDecoder
    from goliath_b200.seams import SeamSampler
    from goliath_b200.shadow import ShadowUNet

    inp, shadow_r, view_r, comp_r = restated_branch()
    s1k, s2k = bt.seams()
    view = UNetViewDecoder(_geo(cuda), 1024, None)
    view.load_state_dict(view_r.state_dict(), strict=True)
    shadow = ShadowUNet(2048, inp["ao_mean"].float(), 256, n_dims=4, biases=False)
    shadow.load_state_dict(shadow_r.state_dict(), strict=True)
    comp = TextureComposer(SeamSampler(s1k), SeamSampler(s2k), inp["tex_mean"].float())
    comp.upscale_net.load_state_dict(comp_r.upscale_net.state_dict(), strict=True)
    mods = [m.float().to(cuda) for m in (view, shadow, comp)]
    return {k: v.float().to(cuda) for k, v in inp.items()}, mods


def test_branch_vs_reference_fixture(cuda):
    gold = dict(np.load(GOLD))
    inp, (view, shadow, comp) = _our_branch(cuda)
    tmr = inp["tex_mean_rec"].clone().requires_grad_()
    vo = view(inp["geom_rec"], tmr, inp["camera_pos"])
    so = shadow(inp["ao_map"])
    tvr = vo["tex_view_rec"].detach().requires_grad_()
    smap = so["shadow_map"].detach().requires_grad_()
    tmr2 = tmr.detach().requires_grad_()
    tex_rec = comp(tmr2, tvr, smap)
    out = {"tex_view_rec": vo["tex_view_rec"], "cond_view": vo["cond_view"], "shadow_map": so["shadow_map"],
           "ao_map": so["ao_map"], "shadow_map_lowres": so["shadow_map_lowres"], "tex_rec": tex_rec,
           "upscale": comp.upscale_net(torch.cat([tmr2, tvr], 1).detach())}
    w = torch.randn(tex_rec.shape, generator=torch.Generator().manual_seed(77), dtype=torch.float64).float().to(cuda)
    g = dict(zip(["ft_tex_mean_rec", "ft_tex_view_rec", "ft_shadow_map"],
                 torch.autograd.grad((tex_rec * w).sum(), [tmr2, tvr, smap], retain_graph=True)))
    ups = list(comp.upscale_net.named_parameters())
    for (n, _), gp in zip(ups, torch.autograd.grad((tex_rec * w).sum(), [p for _, p in ups])):
        g["p.composer.upscale_net." + n] = gp
    params = [("view." + n, p) for n, p in view.named_parameters()] + [("shadow." + n, p)
                                                                        for n, p in shadow.named_parameters()]
    gr = torch.autograd.grad([vo["tex_view_rec"], so["shadow_map"]], [tmr] + [p for _, p in params],
                             grad_outputs=[g["ft_tex_view_rec"], g["ft_shadow_map"]])
    g["tex_mean_rec"] = gr[0] + g["ft_tex_mean_rec"]
    for (n, _), gp in zip(params, gr[1:]):
        g["p." + n] = gp
    # a sampled fp32 parameter gradient is a sum over up to 2 x 1024^2 terms through the U-Net, so single samples
    # carry ~1e-3 of the tensor's largest entry; the norm-wise gradient checks against the fp64 oracle are above
    bad = []
    for kind, d, tol in (("out", out, 1e-4), ("g", g, 1e-2)):
        for k, t in d.items():
            r = gold["%s_%s" % (kind, k)]
            assert list(t.shape) == gold["shape_%s_%s" % (kind, k)].tolist(), k
            got = _summary(t.cpu())
            got, exp = np.concatenate([got[:3], got[4:]]), np.concatenate([r[:3], r[4:]])
            err = np.abs(got - exp).max() / r[2]
            if err > tol:
                bad.append((kind, k, err))
    assert not bad, bad


def test_composer_repeatable_sync_free_and_graphed(cuda):
    from goliath_b200.graph import Graphed

    inp, (view, shadow, comp) = _our_branch(cuda)
    with torch.no_grad():
        tvr = view(inp["geom_rec"], inp["tex_mean_rec"], inp["camera_pos"])["tex_view_rec"]
        smap = shadow(inp["ao_map"])["shadow_map"]
    w = torch.randn(2, 3, 2048, 2048, device=cuda, generator=torch.Generator(device=cuda).manual_seed(5))
    leaves = [inp["tex_mean_rec"].clone().requires_grad_(), tvr.clone().requires_grad_(),
              smap.clone().requires_grad_()]
    ob = comp.upscale_net.out_block
    wrt = leaves + [ob.weight_v, ob.weight_g, ob.bias, comp.upscale_net.conv_block[0].bias]

    def step():
        return torch.autograd.grad((comp(*leaves) * w).sum(), wrt)

    first = step()                               # builds the seam tables
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        second = step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # every gradient the composite kernel and the seam gathers produce is bitwise repeatable (conv_block's weight
    # gradient comes from the stride-1 kernel's atomic reduction and is left out)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    with torch.no_grad():
        args = [t.detach() for t in leaves]
        eager = comp(*args).clone()
        gr = Graphed(lambda: comp(*args))
        assert torch.equal(gr(), eager)
