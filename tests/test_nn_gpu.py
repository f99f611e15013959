"""GPU parity of the fused deconv layer (csrc/deconv_wnub.cu, rows R1/R8) and LinearWN against vectors produced by
IMPORTING the reference's own layers (tests/golden/nn_layers_ref.npz <- tests/golden/make_layers_golden.py)."""
import os

import numpy as np
import pytest
import torch

from util import assert_close, t2n

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nn_layers_ref.npz")


def test_deconv_tower_vs_reference_layers(cuda):
    from goliath_b200 import nn as gnn

    g = np.load(GOLD)
    f = lambda k: torch.from_numpy(g[k]).float().to(cuda)
    l1 = gnn.make_conv_trans(5, 11, 4, 2, 1, "wn", torch.nn.LeakyReLU(0.2), ub=(12, 20))
    l2 = gnn.make_conv_trans(11, 7, 4, 2, 1, "wn", ub=(24, 40))
    net = torch.nn.Sequential(*l1, *l2).to(cuda)
    assert len(net) == 3 and isinstance(net[1], gnn.FusedLeakyReLU), "LeakyReLU is fused into the layer, indices kept"
    # the reference's Sequential state-dict names ([deconv, LeakyReLU, deconv] -> 0.*, 2.*) load directly
    sd = {"0.weight_v": f("dc_p0"), "0.weight_g": f("dc_p1"), "0.bias": f("dc_p2"),
          "2.weight_v": f("dc_p3"), "2.weight_g": f("dc_p4"), "2.bias": f("dc_p5")}
    net.load_state_dict(sd)
    x = f("dc_x").requires_grad_()
    y = net(x)
    assert_close(t2n(y), g["dc_y"], rtol=1e-4, atol=1e-5 * np.abs(g["dc_y"]).max(), what="deconv tower output")
    (y * f("dc_w")).sum().backward()
    assert_close(t2n(x.grad), g["dc_gx"], rtol=2e-4, atol=2e-5 * np.abs(g["dc_gx"]).max(), what="grad input")
    params = [net[0].weight_v, net[0].weight_g, net[0].bias, net[2].weight_v, net[2].weight_g, net[2].bias]
    for i, p in enumerate(params):
        r = g["dc_gp%d" % i]
        assert_close(t2n(p.grad), r, rtol=5e-4, atol=5e-5 * np.abs(r).max(), what="grad param %d" % i)


@pytest.mark.parametrize("shape", [(1, 16, 125, 64, 48), (2, 264, 40, 8, 8), (1, 3, 5, 17, 33)])
def test_deconv_kernel_vs_torch(cuda, shape):
    """Odd sizes, partial channel blocks, partial tiles; oracle = torch fp64 conv_transpose2d on the CPU."""
    from goliath_b200 import nn as gnn

    B, Cin, Cout, Hi, Wi = shape
    gen = torch.Generator().manual_seed(Cin * 7 + Cout)
    layer = gnn.ConvTranspose2dWNUB(Cin, Cout, 2 * Hi, 2 * Wi)
    with torch.no_grad():
        layer.weight_v.copy_(torch.randn(layer.weight_v.shape, generator=gen) * 0.1)
        layer.weight_g.copy_(torch.rand(layer.weight_g.shape, generator=gen) + 0.5)
        layer.bias.copy_(torch.randn(layer.bias.shape, generator=gen))
    x = torch.randn(B, Cin, Hi, Wi, generator=gen)
    w = (layer.weight_g * layer.weight_v / layer.weight_v.norm()).double()
    ref = torch.nn.functional.leaky_relu(
        torch.nn.functional.conv_transpose2d(x.double(), w, None, 2, 1) + layer.bias.double()[None], 0.2)
    y = layer.to(cuda)(x.to(cuda), slope=0.2)
    assert_close(t2n(y), ref.detach().numpy(), rtol=1e-4, atol=1e-5 * float(ref.abs().max()), what="deconv %s" % (shape,))


@pytest.mark.parametrize("shape,slope", [((1, 16, 125, 64, 48), None), ((1, 16, 125, 64, 48), 0.2), ((2, 32, 16, 32, 64), 0.2),
                                         ((1, 8, 12, 24, 36), 0.2), ((1, 20, 6, 16, 32), None), ((1, 3, 5, 17, 33), 0.2),
                                         ((2, 264, 40, 8, 8), 0.2)])
def test_deconv_backward_vs_torch(cuda, shape, slope):
    """Every gradient of the fused layer (input, weight_v, weight_g, untied bias) against torch autograd of the reference
    formula in fp64 (layers.py:200-204,380-396): the wide backward kernels (Cin <= 32, Wi % 4 == 0, >= 32 x 16: full and
    partial tiles, one and two channel blocks, batch 2, with and without the fused LeakyReLU, incl. the B == 1 aliasing of
    the bias gradient) and the narrow ones."""
    from goliath_b200 import nn as gnn

    B, Cin, Cout, Hi, Wi = shape
    gen = torch.Generator().manual_seed(Cin * 11 + Cout + Wi)
    layer = gnn.ConvTranspose2dWNUB(Cin, Cout, 2 * Hi, 2 * Wi)
    with torch.no_grad():
        layer.weight_v.copy_(torch.randn(layer.weight_v.shape, generator=gen) * 0.1)
        layer.weight_g.copy_(torch.rand(layer.weight_g.shape, generator=gen) + 0.5)
        layer.bias.copy_(torch.randn(layer.bias.shape, generator=gen))
    x = torch.randn(B, Cin, Hi, Wi, generator=gen)
    go = torch.randn(B, Cout, 2 * Hi, 2 * Wi, generator=gen)
    # reference
    v = layer.weight_v.detach().double().requires_grad_()
    g = layer.weight_g.detach().double().requires_grad_()
    bias = layer.bias.detach().double().requires_grad_()
    xr = x.double().requires_grad_()
    y = torch.nn.functional.conv_transpose2d(xr, g * v / v.norm(), None, 2, 1) + bias[None]
    if slope is not None:
        y = torch.nn.functional.leaky_relu(y, slope)
    y.backward(go.double())
    # ours
    layer = layer.to(cuda)
    xc = x.to(cuda).requires_grad_()
    yc = layer(xc, slope=slope)
    yc.backward(go.to(cuda))
    assert_close(t2n(yc), y.detach().numpy(), rtol=1e-4, atol=1e-5 * float(y.abs().max()), what="forward")
    for name, got, want in (("x", xc.grad, xr.grad), ("weight_v", layer.weight_v.grad, v.grad),
                            ("weight_g", layer.weight_g.grad, g.grad), ("bias", layer.bias.grad, bias.grad)):
        want = want.numpy()
        assert_close(t2n(got), want, rtol=2e-4, atol=2e-5 * float(np.abs(want).max()), what="grad %s %s" % (name, shape))


def test_linear_wn_vs_reference(cuda):
    from goliath_b200 import nn as gnn

    g = np.load(GOLD)
    f = lambda k: torch.from_numpy(g[k]).float().to(cuda)
    lin = gnn.LinearWN(9, 13).to(cuda)
    lin.load_state_dict({"weight_v": f("li_v"), "weight_g": f("li_g"), "bias": f("li_b")})
    x = f("li_x").requires_grad_()
    y = lin(x)
    assert_close(t2n(y), g["li_y"], rtol=1e-4, atol=1e-5, what="LinearWN")
    (y * f("li_w")).sum().backward()
    assert_close(t2n(x.grad), g["li_gx"], rtol=2e-4, atol=1e-5, what="LinearWN grad x")
    assert_close(t2n(lin.weight_v.grad), g["li_gv"], rtol=5e-4, atol=1e-5, what="LinearWN grad v")
    assert_close(t2n(lin.weight_g.grad), g["li_gg"], rtol=5e-4, atol=1e-5, what="LinearWN grad g")


def test_prim_decoder_end_to_end_small(cuda):
    """goliath_b200.rgca.PrimDecoder at slabsize 128 against the same computation done with torch fp64 ops on the
    CPU from the same parameters (towers = conv_transpose2d + untied bias + LeakyReLU, heads = pinned torch oracle)."""
    from goliath_b200.rgca import PrimDecoder
    from oracle import heads_oracle as ho

    class Geo:  # stand-in for ca_code.utils.geom.GeometryModule: UV position / normal maps
        def __init__(self, pos, nml): self.pos, self.nml = pos, nml
        def to_uv(self, x): return x
        def vn(self, g): return self.nml

    th = torch
    gen = th.Generator().manual_seed(9)
    S, B = 128, 1
    pos = 100 * th.randn(B, 3, S, S, generator=gen)
    nml = th.randn(B, 3, S, S, generator=gen)
    dec = PrimDecoder(16, Geo(pos.to(cuda), nml.to(cuda)), 255 * th.rand(3, S, S, generator=gen), slabsize=S).to(cuda)
    with th.no_grad():
        for n_, p in dec.named_parameters():
            if n_.endswith("bias"):
                p.normal_(0, 0.1)
    keys = list(dec.state_dict().keys())
    assert "vnocond_mod.12.weight_v" in keys and "vcond_mod.0.bias" in keys and "encmod.0.weight_g" in keys and "albedo" in keys
    embs = th.randn(B, 16, generator=gen)
    campos = th.tensor([[0.0, 0.0, 1000.0]])
    light_sh = th.randn(B, 3, 81, generator=gen)
    li_pos = 1100 * th.nn.functional.normalize(th.randn(B, 4, 3, generator=gen), dim=-1)
    li_int = th.rand(B, 4, 3, generator=gen) + 0.5
    nl = th.tensor([4], dtype=th.int32)
    out = dec(embs.to(cuda), pos.to(cuda), campos.to(cuda), li_int.to(cuda), li_pos.to(cuda), light_sh.to(cuda), nl.to(cuda))
    # torch fp64 restatement from the same parameters
    sd = {k: v.detach().double().cpu() for k, v in dec.state_dict().items()}
    def lin(x, pre): 
        w = sd[pre + ".weight_g"] * sd[pre + ".weight_v"] / sd[pre + ".weight_v"].norm()
        return th.nn.functional.leaky_relu(th.nn.functional.linear(x, w, sd[pre + ".bias"]), 0.2)
    def tower(x, pre):
        for i in range(7):
            p = "%s.%d" % (pre, 2 * i)
            w = sd[p + ".weight_g"] * sd[p + ".weight_v"] / sd[p + ".weight_v"].norm()
            x = th.nn.functional.conv_transpose2d(x, w, None, 2, 1) + sd[p + ".bias"][None]
            if i < 6:
                x = th.nn.functional.leaky_relu(x, 0.2)
        return x
    x = lin(embs.double(), "encmod.0").view(-1, 256, 1, 1)
    f1 = tower(x, "vnocond_mod")
    v = lin(th.nn.functional.normalize(campos.double(), dim=1), "viewmod.0")[:, :, None, None]
    f2 = tower(th.cat([x, v], 1), "vcond_mod")
    ref = ho.gaussian_heads(f1, f2, pos.double(), th.nn.functional.normalize(nml.double(), dim=1), sd["albedo"], light_sh.double(), campos.double())
    for k in ("primpos", "primqvec", "primscale", "opacity", "sigma", "spec_nml", "diff_color"):
        r = ref[k].numpy()
        assert_close(t2n(out[k]), r, rtol=2e-4, atol=2e-5 * np.abs(r).max(), frac=0.999, what="PrimDecoder " + k)
    assert out["color"].shape == (B, S * S, 3) and bool((out["color"] >= 0).all())
    out["color"].sum().backward()
    assert dec.vnocond_mod[0].weight_v.grad is not None and th.isfinite(dec.vnocond_mod[12].bias.grad).all()


@pytest.mark.parametrize("plan,size", [([(64, 32), (32, 16), (16, 8)], (16, 12)), ([(264, 256), (256, 128)], (8, 8)),
                                       ([(32, 48), (48, 16)], (40, 24)),
                                       # large enough for the pair-phase mode (one CTA, both column parities), first
                                       # layer -> NHWC pair stores, second -> NCHW float2 stores with Cout = 21 (padded N)
                                       ([(32, 32), (32, 21)], (96, 200)),
                                       # Npad = 256 over enough tiles to keep the whole N dimension in one CTA: the
                                       # widest accumulator (16 wgmma column blocks per warpgroup)
                                       ([(32, 256)], (64, 64))])
def test_tensor_core_tower_matches_simt(cuda, plan, size):
    """csrc/deconv_tc.cu (wgmma + TMA, 3xTF32) against the SIMT kernel on the same parameters: multi-layer
    NHWC hi/lo chaining, channel padding (264 -> 288, 48 -> 64), partial tiles, and the SIMT tail for Cout % 16 != 0."""
    from goliath_b200 import nn as gnn

    gen = torch.Generator().manual_seed(len(plan) * 100 + plan[0][0])
    H, W = size
    layers, h, w = [], H, W
    for i, (a, b) in enumerate(plan):
        act = torch.nn.LeakyReLU(0.2) if i < len(plan) - 1 else None
        layers += gnn.make_conv_trans(a, b, 4, 2, 1, "wn", act, ub=(2 * h, 2 * w))
        h, w = 2 * h, 2 * w
    tower = torch.nn.Sequential(*layers)
    with torch.no_grad():
        for m in tower:
            if isinstance(m, gnn.ConvTranspose2dWNUB):
                m.weight_v.copy_(torch.randn(m.weight_v.shape, generator=gen) * 0.1)
                m.weight_g.copy_(torch.rand(m.weight_g.shape, generator=gen) + 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=gen) * 0.3)
    tower = tower.to(cuda)
    x = torch.randn(2, plan[0][0], H, W, generator=gen).to(cuda)
    with torch.no_grad():
        ref = tower(x)
        out = gnn.tower_forward_tc(tower, x)
    torch.cuda.synchronize()
    r = t2n(ref)
    assert_close(t2n(out), r, rtol=1e-4, atol=2e-5 * np.abs(r).max(), what="tensor-core tower vs SIMT")
