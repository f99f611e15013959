"""GPU parity of the stride-2 weight-normalised convolution (Conv2dWNUB(.., 4, 2, 1), csrc/deconv_wnub.cu) and of the
RGCA Encoder / GeomDecoder mirrors (goliath_b200.rgca) against the reference's own layers and classes
(tests/golden/encoder_ref.npz <- tests/golden/make_encoder_golden.py) and against torch fp64 autograd on the CPU."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import assert_close, t2n

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "encoder_ref.npz")


def _recipe():
    spec = importlib.util.spec_from_file_location("make_encoder_golden", os.path.join(HERE, "golden", "make_encoder_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_conv_chain_vs_reference_layers(cuda):
    from goliath_b200 import nn as gnn

    g = np.load(GOLD)
    f = lambda k: torch.from_numpy(g[k]).float().to(cuda)
    l1 = gnn.Conv2dWNUB(5, 11, 10, 18, 4, 2, 1)
    l1.fused_slope = 0.2
    net = torch.nn.Sequential(l1, gnn.FusedLeakyReLU(), gnn.Conv2dWNUB(11, 7, 5, 9, 4, 2, 1)).to(cuda)
    net.load_state_dict({"0.weight_v": f("cv_p0"), "0.weight_g": f("cv_p1"), "0.bias": f("cv_p2"),
                         "2.weight_v": f("cv_p3"), "2.weight_g": f("cv_p4"), "2.bias": f("cv_p5")})
    x = f("cv_x").requires_grad_()
    y = net(x)
    assert_close(t2n(y), g["cv_y"], rtol=1e-4, atol=1e-5 * np.abs(g["cv_y"]).max(), what="conv chain output")
    (y * f("cv_w")).sum().backward()
    assert_close(t2n(x.grad), g["cv_gx"], rtol=2e-4, atol=2e-5 * np.abs(g["cv_gx"]).max(), what="grad input")
    params = [net[0].weight_v, net[0].weight_g, net[0].bias, net[2].weight_v, net[2].weight_g, net[2].bias]
    for i, p in enumerate(params):
        r = g["cv_gp%d" % i]
        assert_close(t2n(p.grad), r, rtol=5e-4, atol=5e-5 * np.abs(r).max(), what="grad param %d" % i)


# (B, Cin, Cout, Ho, Wo, slope, bias, input needs grad)
ENCODER_LAYERS = [(1, 3, 32, 512, 512), (1, 32, 32, 256, 256), (1, 32, 64, 128, 128), (1, 64, 64, 64, 64),
                  (1, 64, 128, 32, 32), (1, 128, 128, 16, 16), (1, 128, 256, 8, 8), (1, 256, 256, 4, 4)]
CASES = ([s + (0.2, True, s[1] != 3) for s in ENCODER_LAYERS] + [
    (2, 32, 64, 128, 128, 0.2, True, True),     # batch 2 (the wide forward at this size)
    (2, 5, 7, 17, 33, 0.2, True, True),         # partial tiles and channel blocks, odd output size
    (4, 6, 40, 72, 100, 0.2, True, True),       # partial tiles / channel blocks of the wide forward and weight kernels
    (1, 32, 32, 64, 64, None, True, True),      # no activation, B == 1: gz and the bias gradient alias gout
    (2, 16, 24, 40, 48, None, True, True),      # no activation, batch 2
    (2, 16, 24, 40, 48, 0.2, False, True),      # bias=False
    (1, 3, 32, 64, 96, None, False, False),     # bias=False, no activation, input without requires_grad
])


@pytest.mark.parametrize("B,Cin,Cout,Ho,Wo,slope,has_bias,need_gx", CASES)
def test_conv4x4s2_vs_torch(cuda, B, Cin, Cout, Ho, Wo, slope, has_bias, need_gx):
    """Forward and every gradient of the fused stride-2 layer against torch fp64 conv2d autograd on the CPU of the
    reference formula (layers.py:200-204,303-327)."""
    from goliath_b200 import nn as gnn

    gen = torch.Generator().manual_seed(Cin * 13 + Cout + Wo)
    layer = gnn.Conv2dWNUB(Cin, Cout, Ho, Wo, 4, 2, 1, bias=has_bias)
    with torch.no_grad():
        layer.weight_v.copy_(torch.randn(layer.weight_v.shape, generator=gen) * 0.1)
        layer.weight_g.copy_(torch.rand(layer.weight_g.shape, generator=gen) + 0.5)
        if has_bias:
            layer.bias.copy_(torch.randn(layer.bias.shape, generator=gen))
    x = torch.randn(B, Cin, 2 * Ho, 2 * Wo, generator=gen)
    go = torch.randn(B, Cout, Ho, Wo, generator=gen)
    v = layer.weight_v.detach().double().requires_grad_()
    g = layer.weight_g.detach().double().requires_grad_()
    xr = x.double().requires_grad_(need_gx)
    y = F.conv2d(xr, g * v / v.norm(), None, 2, 1)
    if has_bias:
        bias = layer.bias.detach().double().requires_grad_()
        y = y + bias[None]
    if slope is not None:
        y = F.leaky_relu(y, slope)
    y.backward(go.double())
    layer = layer.to(cuda)
    xc = x.to(cuda).requires_grad_(need_gx)
    yc = layer(xc, slope=slope)
    yc.backward(go.to(cuda))
    what = "(%d, %d, %d, %d, %d)" % (B, Cin, Cout, Ho, Wo)
    assert_close(t2n(yc), y.detach().numpy(), rtol=1e-4, atol=1e-5 * float(y.abs().max()), what="forward " + what)
    checks = [("weight_v", layer.weight_v.grad, v.grad), ("weight_g", layer.weight_g.grad, g.grad)]
    if has_bias:
        checks.append(("bias", layer.bias.grad, bias.grad))
    if need_gx:
        checks.append(("x", xc.grad, xr.grad))
    else:
        assert xc.grad is None
    for name, got, want in checks:
        want = want.numpy()
        assert_close(t2n(got), want, rtol=2e-4, atol=2e-5 * float(np.abs(want).max()), what="grad %s %s" % (name, what))


def _encoder_from_recipe(cuda, n_embs, n_verts, batch):
    from goliath_b200.rgca import Encoder

    enc = Encoder(n_embs, n_verts)
    sd, geom, color = _recipe().encoder_recipe([(k, tuple(v.shape)) for k, v in enc.state_dict().items()],
                                               n_verts=n_verts, batch=batch)
    enc.load_state_dict(sd)
    return enc.to(cuda), sd, geom, color


def test_encoder_eval_vs_reference(cuda):
    rec = _recipe()
    enc, _, geom, color = _encoder_from_recipe(cuda, rec.N_EMBS, rec.N_VERTS, rec.B_FULL)
    enc.eval()
    g = np.load(GOLD)
    with torch.no_grad():
        out = enc(geom.to(cuda), color.to(cuda))
    assert set(out) == {"embs", "embs_mu", "embs_logvar"}
    for k, r in (("embs_mu", g["enc_mu"]), ("embs_logvar", g["enc_logvar"])):
        assert_close(t2n(out[k]), r, rtol=1e-4, atol=1e-4 * np.abs(r).max(), what="Encoder " + k)
    assert torch.equal(out["embs"], out["embs_mu"]) and out["embs"].data_ptr() != out["embs_mu"].data_ptr()


def test_encoder_training_noise(cuda):
    """rgca.py:312-315: embs = mu + exp(logvar) * randn_like(mu) * noise_std (exp(logvar), not exp(logvar / 2))."""
    enc, _, geom, color = _encoder_from_recipe(cuda, 32, 16, 2)
    enc.noise_std = 0.7
    with torch.no_grad():
        enc.logvar.bias.fill_(3.0)  # exp(logvar) far from 1 and from exp(logvar / 2)
    enc.train()
    torch.cuda.manual_seed(123)
    with torch.no_grad():
        out = enc(geom.to(cuda), color.to(cuda))
    torch.cuda.manual_seed(123)
    noise = torch.randn_like(out["embs_mu"])
    want = out["embs_mu"] + torch.exp(out["embs_logvar"]) * noise * 0.7
    assert_close(t2n(out["embs"]), t2n(want), rtol=1e-6, atol=1e-6, what="training embs")
    assert float((out["embs"] - out["embs_mu"]).abs().max()) > 1.0


def test_encoder_backward_vs_torch(cuda):
    """Every parameter gradient of the full Encoder and the gradient w.r.t. the geometry input at B = 2, against torch
    fp64 CPU autograd of a functional restatement of rgca.py:303-310 from the same parameters."""
    enc, sd, geom, color = _encoder_from_recipe(cuda, 64, 24, 2)
    enc.eval()
    gen = torch.Generator().manual_seed(77)
    w_mu, w_lv = torch.randn(2, 64, generator=gen), torch.randn(2, 64, generator=gen)
    gc = geom.to(cuda).requires_grad_()
    out = enc(gc, color.to(cuda))
    ((out["embs_mu"] * w_mu.to(cuda)).sum() + (out["embs_logvar"] * w_lv.to(cuda)).sum()).backward()

    p = {k: v.double().requires_grad_() for k, v in sd.items()}
    wn = lambda pre: p[pre + ".weight_g"] * p[pre + ".weight_v"] / p[pre + ".weight_v"].norm()
    lin = lambda x, pre: F.linear(x, wn(pre), p[pre + ".bias"])
    gr = geom.double().requires_grad_()
    geomout = F.leaky_relu(lin(gr.view(2, -1), "geommod.0"), 0.2)
    h = color.double() / 255.0 - 0.5
    for i in range(8):
        pre = "texmod.%d" % (2 * i)
        h = F.leaky_relu(F.conv2d(h, wn(pre), None, 2, 1) + p[pre + ".bias"][None], 0.2)
    enc_out = F.leaky_relu(lin(torch.cat([geomout, h.view(-1, 256 * 4 * 4)], 1), "jointmod.0"), 0.2)
    mu, lv = lin(enc_out, "mean") * 0.1, lin(enc_out, "logvar") * 0.01
    ((mu * w_mu.double()).sum() + (lv * w_lv.double()).sum()).backward()
    assert_close(t2n(out["embs_mu"]), mu.detach().numpy(), rtol=1e-4, atol=1e-4 * float(mu.abs().max()), what="mu")
    named = dict(enc.named_parameters())
    assert set(named) == set(p)
    # a pre-activation within fp32 rounding of zero takes the other LeakyReLU branch than in fp64, so a few of the
    # 8.4 M first-layer bias gradients legitimately differ by the slope factor; the norm-wise bound still holds
    for k, ref in list(p.items()) + [("geom", gr)]:
        got = gc.grad if k == "geom" else named[k].grad
        want = ref.grad.numpy()
        assert_close(t2n(got), want, rtol=5e-4, atol=5e-5 * float(np.abs(want).max()), frac=1 - 1e-5, what="grad " + k)


def test_geom_decoder_vs_reference(cuda):
    from goliath_b200.rgca import GeomDecoder

    g = np.load(GOLD)
    names = json.loads(str(g["gd_names"]))
    gd = GeomDecoder(16, torch.zeros(12, 3), 2.5).to(cuda)
    gd.load_state_dict({k: torch.from_numpy(g["gd_p_" + k]).float() for k in names})
    with torch.no_grad():
        out = gd(torch.from_numpy(g["gd_embs"]).float().to(cuda))
    assert set(out) == {"face_geom"}
    r = g["gd_geom"]
    assert_close(t2n(out["face_geom"]), r, rtol=1e-4, atol=1e-5 * np.abs(r).max(), what="GeomDecoder")
