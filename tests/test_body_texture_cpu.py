"""CPU checks of the body avatar's texture branch (DESIGN.md row R9'): the checkpoint layout of the reference's
`UNetWB`, `ShadowUNet`, `UNetViewDecoder`, `UpscaleNet` and AutoEncoder's forward_tex subset against
tests/golden/body_texture_ref.npz, strict loading of the restatement's state dicts, ShadowUNet's initialisation, the
torch restatement (tests/body_texture_restate.py) against the reference's fp64 run, and the refusal of CPU tensors and
mismatched sizes."""
import json
import os
import types

import numpy as np
import pytest
import torch

import body_texture_restate as bt

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "body_texture_ref.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _samplers():
    from goliath_b200.seams import SeamSampler

    s1k, s2k = bt.seams()
    return SeamSampler(s1k), SeamSampler(s2k)


def _ours(inp=None):
    from goliath_b200.mesh_vae import TextureComposer, UNetViewDecoder, UpscaleNet
    from goliath_b200.shadow import ShadowUNet
    from goliath_b200.unet import UNetWB

    inp = inp or bt.seeded_inputs(batch=1)
    vi, _, idx, bary = bt.uv_mesh(n=4, size=8)
    geo = types.SimpleNamespace(vi=vi.int(), index_image=idx, bary_image=bary)
    s1, s2 = _samplers()
    return {"unet": UNetWB(4, 3, 1024),
            "shadow": ShadowUNet(2048, inp["ao_mean"].float(), 256, n_dims=4, interp_mode="bilinear", biases=False),
            "view": UNetViewDecoder(geo, 1024, None),
            "upscale": UpscaleNet(6, 3, 4),
            "composer": TextureComposer(s1, s2, inp["tex_mean"].float())}


def test_checkpoint_layout_matches_the_reference(gold):
    for k, m in _ours().items():
        keys = json.loads(bytes(gold["keys_" + k]).decode())
        assert {n: list(v.shape) for n, v in m.state_dict().items()} == keys, k
        assert sum(p.numel() for p in m.parameters()) == int(gold["n_params_" + k]), k
    assert int(gold["n_params_unet"]) == 19_879_839
    assert "faces" not in _ours()["view"].state_dict()


def test_restatement_state_dicts_load_strictly():
    inp = bt.seeded_inputs(batch=1)
    ours = _ours(inp)
    vi, _, idx, bary = bt.uv_mesh(n=4, size=8)
    refs = {"unet": bt.UNetWB(4, 3, 1024), "shadow": bt.ShadowUNet(2048, inp["ao_mean"], 256, n_dims=4, biases=False),
            "view": bt.UNetViewDecoder(vi, idx, bary, 1024), "upscale": bt.UpscaleNet(6, 3, 4)}
    for k, ref in refs.items():
        bt.seeded_fill(ref, 5)
        m = ours[k].double()
        m.load_state_dict(ref.state_dict(), strict=True)
        for n, v in ref.state_dict().items():
            assert torch.equal(m.state_dict()[n], v), (k, n)


def test_init_properties(gold):
    """ShadowUNet: weight_v keeps nn.Conv2d's default init, weight_g = ||weight_v||_F, biases zero — as the reference's
    weights_initializer leaves a weight-normalised layer; UNetWB: the effective weight equals weight_v, biases zero"""
    torch.manual_seed(0)
    ours = _ours()
    rows = []
    for _, m in sorted(ours["shadow"].named_modules()):
        if hasattr(m, "weight_v"):
            v, g = m.weight_v.detach().double(), m.weight_g.detach().double()
            fan_in = v[0].numel()
            rows.append([float(v.abs().max()) * fan_in ** 0.5, float((g - v.norm()).abs().max() / v.norm()),
                         float(m.bias.abs().max()), float(v.std()) * (3 * fan_in) ** 0.5])
    rows, ref = np.array(rows), gold["shadow_init"]
    assert rows.shape == ref.shape == (9, 4)
    for r in (rows, ref):
        assert np.all(r[:, 0] <= 1.0) and np.all(r[:, 0] > 0.5)     # uniform(-1/sqrt(fan_in), 1/sqrt(fan_in))
        assert np.all(r[:, 1] <= 1e-6) and np.all(r[:, 2] == 0.0)
    # the spread of each layer's sample agrees with the reference's to sampling noise
    assert np.all(np.abs(rows[:, 3] - ref[:, 3]) < 0.35)
    u = gold["unet_init"]
    assert u.shape == (11, 2) and np.all(u[:, 0] < 1e-6) and np.all(u[:, 1] == 0.0)
    for _, m in sorted(ours["unet"].named_modules()):
        if hasattr(m, "weight_v"):
            assert torch.allclose(m.weight.detach(), m.weight_v, rtol=1e-5, atol=1e-7)
            assert float(m.bias.abs().max()) == 0.0


def _summary(t):
    f = t.detach().double().reshape(-1)
    return np.concatenate([[f.mean().item(), f.std().item(), f.abs().max().item(), float(f.numel())],
                           f[torch.linspace(0, f.numel() - 1, 256, dtype=torch.float64).long()].numpy()])


def restated_branch(device="cpu", dtype=torch.float64, batch=bt.B):
    """the restatement's whole branch with the fixture's seeds: outputs and gradients, named as in the fixture"""
    inp = {k: v.to(device, dtype) for k, v in bt.seeded_inputs(batch=batch).items()}
    vi, _, idx, bary = bt.uv_mesh()
    s1k, s2k = bt.seams()
    ts = [bt.sr.TorchSeamSampler(*(s[k].to(device) for k in ("dst_ij", "src_ij", "uvs", "weights"))) for s in (s1k, s2k)]
    shadow = bt.seeded_fill(bt.ShadowUNet(2048, inp["ao_mean"].cpu(), 256, n_dims=4, biases=False).double(), 101)
    view = bt.seeded_fill(bt.UNetViewDecoder(vi.to(device), idx.to(device), bary.to(device), 1024).double(), 102)
    comp = bt.TextureComposer(ts[0], ts[1], inp["tex_mean"])
    bt.seeded_fill(comp.upscale_net.double(), 103)
    for m in (shadow, view, comp):
        m.to(device, dtype)
    return inp, shadow, view, comp


def test_restatement_matches_the_reference_fixture(gold):
    inp, shadow, view, comp = restated_branch()
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
    w = torch.randn(tex_rec.shape, generator=torch.Generator().manual_seed(77), dtype=torch.float64)
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
    assert {"g_" + k for k in g} == {k for k in gold if k.startswith("g_")}
    for kind, d in (("out", out), ("g", g)):
        for k, t in d.items():
            assert list(t.shape) == gold["shape_%s_%s" % (kind, k)].tolist(), k
            np.testing.assert_allclose(_summary(t), gold["%s_%s" % (kind, k)], rtol=1e-12, atol=1e-12 * gold[
                "%s_%s" % (kind, k)][2], err_msg=k)
    # the fixture covers uncovered texels (view cosine 0) and both signs of the view cosine
    vc = vo["cond_view"][:, 0]
    assert float((vc == 0).double().mean()) > 0.03 and float(vc.min()) < 0 < float(vc.max())


def test_cpu_tensors_and_mismatched_sizes_raise():
    from goliath_b200.mesh_vae import TextureComposer
    from goliath_b200.seams import SeamSampler

    ours = _ours()
    with pytest.raises(RuntimeError):
        ours["unet"](torch.zeros(1, 4, 1024, 1024))
    with pytest.raises(RuntimeError):
        ours["shadow"](torch.zeros(1, 1, 256, 256))
    with pytest.raises(RuntimeError):
        ours["upscale"](torch.zeros(1, 6, 1024, 1024))
    with pytest.raises(RuntimeError):
        ours["view"](torch.zeros(1, 16, 3), torch.zeros(1, 3, 1024, 1024), torch.zeros(1, 3))
    comp = ours["composer"]
    with pytest.raises(RuntimeError):
        comp(torch.zeros(1, 3, 1024, 1024), torch.zeros(1, 3, 1024, 1024), torch.zeros(1, 1, 2048, 2048))
    # tex_mean must be twice tex_mean_rec's size, and the samplers built for the sizes they receive; these checks
    # come before any device work, so they run on the meta device here
    meta = lambda *s: torch.empty(*s, device="meta")
    for tm, ts, sm in (((1, 3, 512, 512), (1, 3, 1024, 1024), (1, 1, 1024, 1024)),
                       ((1, 3, 1024, 1024), (1, 3, 1024, 1024), (1, 1, 1024, 1024))):
        c = TextureComposer(SeamSampler(bt.sr.synthetic_seams(tm[2] // 2, n_pairs=20)),
                            SeamSampler(bt.sr.synthetic_seams(tm[2], n_pairs=20)), torch.zeros(tm))
        with pytest.raises(RuntimeError, match="twice|built for"):
            c._check(meta(*ts), meta(*ts), meta(*sm))
    small = TextureComposer(SeamSampler(bt.sr.synthetic_seams(32, n_pairs=20)),
                            SeamSampler(bt.sr.synthetic_seams(2048, n_pairs=20)), torch.zeros(1, 3, 2048, 2048))
    with pytest.raises(RuntimeError, match="built for"):
        small._check(meta(1, 3, 1024, 1024), meta(1, 3, 1024, 1024), meta(1, 1, 2048, 2048))
    with pytest.raises(TypeError):
        TextureComposer(None, None, torch.zeros(1, 3, 2048, 2048))
