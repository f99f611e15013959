"""GPU parity of the hand-MVP decoder pieces (SURVEY.md §8 row R8: csrc/conv_wnub.cu, csrc/mvp_prims.cu,
goliath_b200/hand_mvp.py) against vectors produced by RUNNING the reference's own code on CPU in fp64
(tests/golden/hand_mvp_ref.npz <- tests/golden/make_hand_mvp_golden.py)."""
import json
import os

import numpy as np
import pytest
import torch

from util import assert_close, t2n

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hand_mvp_ref.npz")


def _f(g, cuda):
    return lambda k: torch.from_numpy(g[k]).float().to(cuda)


def _tol(ref, r):
    return dict(rtol=r, atol=r * 0.1 * float(np.abs(ref).max()))


def test_conv2d_wnub_chain_vs_reference_layers(cuda):
    from goliath_b200 import nn as gnn

    g = np.load(GOLD)
    f = _f(g, cuda)
    a, b = gnn.Conv2dWNUB(5, 11, 12, 20, 3, 1, 1), gnn.Conv2dWNUB(11, 7, 12, 20, 3, 1, 1)
    a.fused_slope = 0.2
    net = torch.nn.Sequential(a, gnn.FusedLeakyReLU(), b).to(cuda)
    net.load_state_dict({"0.weight_v": f("cv_p0"), "0.weight_g": f("cv_p1"), "0.bias": f("cv_p2"),
                         "2.weight_v": f("cv_p3"), "2.weight_g": f("cv_p4"), "2.bias": f("cv_p5")})
    x = f("cv_x").requires_grad_()
    y = net(x)
    assert_close(t2n(y), g["cv_y"], what="conv chain output", **_tol(g["cv_y"], 1e-4))
    (y * f("cv_w")).sum().backward()
    assert_close(t2n(x.grad), g["cv_gx"], what="grad input", **_tol(g["cv_gx"], 2e-4))
    for i, p in enumerate([a.weight_v, a.weight_g, a.bias, b.weight_v, b.weight_g, b.bias]):
        r = g["cv_gp%d" % i]
        assert_close(t2n(p.grad), r, what="grad param %d" % i, **_tol(r, 5e-4))


@pytest.mark.parametrize("tag,cin,cout,k", [("b3", 6, 10, 3), ("b1", 7, 5, 1)])
def test_conv_block_vs_reference(cuda, tag, cin, cout, k):
    from goliath_b200 import nn as gnn

    g = np.load(GOLD)
    f = _f(g, cuda)
    blk = gnn.ConvBlock(cin, cout, 9, kernel_size=k, padding=(k - 1) // 2).to(cuda)
    names = json.loads(str(g[tag + "_names"]))
    assert sorted(names) == sorted(n for n, _ in blk.named_parameters()), "parameter names must match the reference's"
    blk.load_state_dict({n: f("%s_p_%s" % (tag, n)) for n in names})
    params = list(blk.named_parameters())

    def run():
        x = f(tag + "_x").requires_grad_()
        y = blk(x)
        grads = torch.autograd.grad((y * f(tag + "_w")).sum(), [x] + [p for _, p in params])
        return y.detach(), dict(zip(["x"] + [n for n, _ in params], grads))

    y, gr = run()
    y2, gr2 = run()
    assert_close(t2n(y), g[tag + "_y"], what="ConvBlock output", **_tol(g[tag + "_y"], 1e-4))
    assert_close(t2n(gr["x"]), g[tag + "_gx"], what="ConvBlock grad input", **_tol(g[tag + "_gx"], 2e-4))
    for n, _ in params:
        r = g["%s_g_%s" % (tag, n)]
        assert_close(t2n(gr[n]), r, what="ConvBlock grad " + n, **_tol(r, 5e-4))
    assert torch.equal(y, y2)
    for n in gr:
        assert torch.equal(gr[n], gr2[n]), n      # fixed-order sums: the same bits on every run


def test_pose_encoder_vs_reference(cuda):
    from goliath_b200.hand_mvp import PoseEncoder

    g = np.load(GOLD)
    f = _f(g, cuda)
    pe = PoseEncoder(8, 12, 6).to(cuda)
    pe.load_state_dict({n: f("pe_p_" + n) for n, _ in pe.named_parameters()})
    pose = f("pe_pose").requires_grad_()
    y = pe(pose)
    assert_close(t2n(y), g["pe_y"], what="PoseEncoder output", **_tol(g["pe_y"], 1e-4))
    (y * f("pe_w")).sum().backward()
    assert_close(t2n(pose.grad), g["pe_gpose"], what="PoseEncoder grad pose", **_tol(g["pe_gpose"], 3e-4))


def test_prim_transforms_vs_reference(cuda):
    from goliath_b200.hand_mvp import prim_transforms

    g = np.load(GOLD)
    f = _f(g, cuda)
    dec = f("pt_dec").requires_grad_()
    pos, rot, scale = prim_transforms(dec, f("pt_posbase"), f("pt_rotbase"), 512.0)
    assert_close(t2n(pos), g["pt_primpos"], what="primpos", rtol=1e-5, atol=1e-6)
    assert_close(t2n(rot), g["pt_primrot"], what="primrot", rtol=1e-5, atol=1e-6)
    assert_close(t2n(scale), g["pt_primscale"], what="primscale", rtol=1e-5, atol=1e-4)
    ((pos * f("pt_w1")).sum() + (rot * f("pt_w2")).sum() + (scale * f("pt_w3")).sum()).backward()
    assert_close(t2n(dec.grad), g["pt_gdec"], what="grad dec", **_tol(g["pt_gdec"], 1e-4))
    # partial upstream gradients (only the rotation used) and the training warm start
    dec2 = f("pt_dec").requires_grad_()
    _, rot2, _ = prim_transforms(dec2, f("pt_posbase"), f("pt_rotbase"), 512.0)
    (rot2 * f("pt_w2")).sum().backward()
    assert torch.isfinite(dec2.grad).all() and float(dec2.grad[:, :3].abs().max()) == 0.0
    dec3 = f("pt_dec").requires_grad_()
    pos3, rot3, scale3 = prim_transforms(dec3, f("pt_posbase"), f("pt_rotbase"), 512.0, zero_delta=True)
    assert_close(t2n(pos3), g["pt_posbase"], what="warm-start primpos", rtol=1e-6, atol=1e-6)
    assert float((scale3.detach() - 512.0).abs().max()) == 0.0
    (pos3.sum() + rot3.sum() + scale3.sum()).backward()
    assert float(dec3.grad.abs().max()) == 0.0


def test_slabs_to_primrgba_vs_reference(cuda):
    from goliath_b200.hand_mvp import slabs_to_primrgba

    g = np.load(GOLD)
    f = _f(g, cuda)
    rgb, alpha = f("sl_rgb").requires_grad_(), f("sl_alpha").requires_grad_()
    ref = torch.from_numpy(g["sl_primrgba"]).float()
    out = slabs_to_primrgba(rgb, alpha, (4, 4, 2))
    assert out.shape == ref.shape and torch.equal(out.cpu(), ref), "plain re-layout must be exact"
    # valid-primitive gather (render_raymarcher.py:44-46) and raw-output activations (hand_mvp.py:434,472) in one pass
    valid = torch.tensor([1, 0, 1, 1, 0, 0, 1, 1, 1, 0, 1, 1, 1, 1, 0, 1], dtype=torch.bool)
    w = torch.randn(2, int(valid.sum()), 2, 4, 4, 4, generator=torch.Generator().manual_seed(3)).to(cuda)
    out2 = slabs_to_primrgba(rgb, alpha, (4, 4, 2), valid_prims=valid.to(cuda), raw=True)
    rgb_r, alpha_r = rgb.detach().clone().requires_grad_(), alpha.detach().clone().requires_grad_()
    act = torch.cat([torch.relu(25.0 * rgb_r + 100.0), torch.relu(alpha_r)], 2)
    exp = act.view(2, 2, 4, 4, 4, 4, 4).permute(0, 3, 5, 1, 4, 6, 2).reshape(2, 16, 2, 4, 4, 4)[:, valid.to(cuda)].contiguous()
    assert torch.equal(out2, exp)
    (out2 * w).sum().backward()
    (exp * w).sum().backward()
    assert torch.equal(rgb.grad, rgb_r.grad) and torch.equal(alpha.grad, alpha_r.grad)


def test_trans_decoder_full_size_vs_torch(cuda):
    """TransDecoder at its real size (64 ch @64x64) against a library restatement with the same parameters;
    the layer arithmetic itself is pinned by the reference-layer fixtures above."""
    from goliath_b200.hand_mvp import TransDecoder

    torch.manual_seed(5)
    td = TransDecoder(64).to(cuda)
    with torch.no_grad():
        for m in td.dec0:
            if hasattr(m, "bias") and m.bias is not None:
                m.bias.normal_(0, 0.1)
    x = torch.randn(2, 64, 64, 64, device=cuda)
    dp, dr, ds = td(x)
    with torch.no_grad():
        h = x.double().cpu()
        convs = [m for m in td.dec0 if hasattr(m, "weight_v")]
        for i, m in enumerate(convs):
            wgt = (m.weight_g * m.weight_v / m.weight_v.norm()).double().cpu()
            h = torch.nn.functional.conv2d(h, wgt, None, 1, 1) + m.bias.double().cpu()[None]
            if i + 1 < len(convs):
                h = torch.nn.functional.leaky_relu(h, 0.2)
        h = h.view(2, 9, -1).permute(0, 2, 1)
    assert_close(t2n(dp), (h[..., 0:3] * 1e-4).numpy(), what="dpos", **_tol((h[..., 0:3] * 1e-4).numpy(), 1e-4))
    assert_close(t2n(dr), (h[..., 3:6] * 0.01).numpy(), what="drvec", **_tol((h[..., 3:6] * 0.01).numpy(), 1e-4))
    assert_close(t2n(ds), torch.exp(0.01 * h[..., 6:9]).numpy(), what="dscale", rtol=1e-5, atol=1e-6)


def test_hand_mvp_decode_to_raymarch_end_to_end(cuda):
    """joint -> TransDecoder -> prim_transforms; joint -> alpha / rgb DeconvContentDecoder -> slabs_to_primrgba ->
    mvpraymarch, forward + backward through every piece (sizes of the real model, B = 1)."""
    from goliath_b200 import mvpraymarch, utils
    from goliath_b200.hand_mvp import DeconvContentDecoder, TransDecoder, prim_transforms, slabs_to_primrgba

    torch.manual_seed(11)
    B, K = 1, 4096
    td = TransDecoder(64).to(cuda)
    alphadec, rgbdec = DeconvContentDecoder(8, 64, 1).to(cuda), DeconvContentDecoder(8, 66, 3).to(cuda)
    joint = torch.randn(B, 64, 64, 64, device=cuda, requires_grad=True)
    cond = torch.randn(B, 2, 64, 64, device=cuda)
    # base frame: primitives on a 64x64 grid wrapped on a cylinder, identity-ish rotations
    u, v = torch.meshgrid(torch.linspace(0, 2 * np.pi, 65)[:-1], torch.linspace(-0.5, 0.5, 64), indexing="ij")
    posbase = torch.stack([0.4 * torch.cos(u), v, 0.4 * torch.sin(u)], -1).reshape(1, K, 3).to(cuda)
    rotbase = torch.eye(3).expand(1, K, 3, 3).contiguous().to(cuda)
    primpos, primrot, primscale = prim_transforms(td.raw(joint), posbase, rotbase, prim_scale=48.0)
    alpha_raw = alphadec(joint).view(B, 8, 1, 1024, 1024)
    rgb_raw = rgbdec(torch.cat([joint, cond], 1)).view(B, 8, 3, 1024, 1024)
    valid = torch.ones(K, dtype=torch.bool, device=cuda)
    valid[::7] = False
    tpl = slabs_to_primrgba(rgb_raw, alpha_raw + 0.05, (16, 16, 8), valid_prims=valid, raw=True)
    assert tpl.shape == (B, int(valid.sum()), 8, 16, 16, 4)
    H, W = 48, 40
    campos = torch.tensor([[0.0, 0.0, -2.5]], device=cuda)
    camrot = torch.eye(3, device=cuda)[None]
    focal = torch.tensor([[120.0, 120.0]], device=cuda)
    princpt = torch.tensor([[W / 2.0, H / 2.0]], device=cuda)
    raypos, raydir, tminmax = utils.compute_raydirs(campos, camrot, focal, princpt, (W, H), 1.0)
    out = mvpraymarch.mvpraymarch(raypos, raydir, 1.0 / 256, tminmax,
                                  (primpos[:, valid].contiguous(), primrot[:, valid].contiguous(),
                                   primscale[:, valid].contiguous()), tpl, None)
    assert out.shape == (B, H, W, 4) and torch.isfinite(out).all()
    assert float(out[..., 3].max()) > 0.0, "rays must hit the primitives"
    out.sum().backward()
    assert torch.isfinite(joint.grad).all() and float(joint.grad.abs().max()) > 0.0
    for mod in (td, alphadec, rgbdec):
        for n, p in mod.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), n
