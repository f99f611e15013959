"""GPU checks of the relightable hand teacher (DESIGN.md row R8″: csrc/mvp_raymarch.cu `gb_mvp_shadow_march`,
csrc/olat_teacher.cu, goliath_b200/hand_teacher.py): parity with the reference's `OLATRGBDecoder` run on CPU in fp64
(tests/golden/hand_olat_ref.npz), and, at the config's size, each kernel against the formulation it replaces."""
import json
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from util import assert_close, rel_err, t2n

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hand_olat_ref.npz")


def _rm(radius):
    return types.SimpleNamespace(dt=1.0 / radius, volume_radius=radius)


def _mismatch(a, b, what, fp32_err):
    """None when |a - b| <= rtol (|b| + max|b|) on 99% of the elements and the norm-wise relative error is <= `norm`,
    else a message.  rtol = max(1e-4, 4 e) and norm = max(1e-3, 4 e), where e is the norm-wise error of the
    reference's own code run in fp32 against its fp64 run (stored with the golden): the U-Net gradients are long
    sums with cancellation that fp32 evaluates to several 1e-4 however it is ordered.  The fraction and the 1e-3 floor
    allow for the few voxels that the splat's RED order moves where its weight is near zero (as
    test_shadow_splat_vs_oracle does)."""
    rtol, norm = max(1e-4, 4 * fp32_err), max(1e-3, 4 * fp32_err)
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ok = (np.abs(a - b) <= rtol * (np.abs(b) + np.abs(b).max())).mean()
    err = rel_err(a, b)
    if ok < 0.99 or err > norm:
        return "%s: %.5f of the elements within %.1e, norm-wise relative error %.2e (bound %.1e)" % (
            what, ok, rtol, err, norm)
    return None


def _golden_decoder(g, cuda):
    from goliath_b200.hand_teacher import OLATRGBDecoder

    dec = OLATRGBDecoder(64, (8, 8, 4), 8, 8, _rm(100.0), 100.0, n_init_channels=4, n_enc_dims=[8] * 5,
                         shadow_img_size=48).to(cuda)
    dec.load_state_dict({k: torch.from_numpy(g["sd_" + k]) for k in dec.state_dict()})
    return dec


def _golden_inputs(g, cuda):
    f = lambda k: torch.from_numpy(g["in_" + k]).float().to(cuda)
    return [f("campos"), None, None, f("primpos"), f("primrot"), f("primscale"), f("primalpha"), f("valid_prims"),
            f("joint_feat").requires_grad_(), f("light_pos"), f("light_intensity")]


@pytest.mark.parametrize("tag,iteration", [("warm", 0), ("sig", 5000)])
def test_decoder_vs_reference(cuda, tag, iteration):
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_hand_olat_golden import lattice, upstream_grads

    g = np.load(GOLD)
    dec = _golden_decoder(g, cuda).train()
    args = _golden_inputs(g, cuda)
    xs = []
    dec.enc_layers[0].register_forward_pre_hook(lambda m, a: xs.append(a[0].detach().clone()))
    out = dec(*args, iteration)
    assert set(out) == {"primrgb", "primshadow", "texolat"}
    for c in range(2):
        x, ref = t2n(lattice(xs[c])), g["x%d" % c]
        assert_close(x[:, :24], ref[:, :24], rtol=1e-4, what="chunk %d light / view features" % c)
        assert_close(x[:, 24:], ref[:, 24:], rtol=1e-3, atol=1e-3, frac=0.999, what="chunk %d 1 - shadow" % c)
    assert_close(t2n(lattice(out["primshadow"])), g["primshadow"], rtol=1e-3, atol=1e-3, frac=0.999,
                 what="primshadow")
    e32 = json.loads(str(g["fp32_err"]))
    res = {tag + "_primrgb": out["primrgb"], tag + "_texolat": out["texolat"]}
    w_rgb, w_tex = (w.float().to(cuda) for w in upstream_grads(out["primrgb"].shape, out["texolat"].shape))
    ((out["primrgb"] * w_rgb).sum() + (out["texolat"] * w_tex).sum()).backward()
    res[tag + "_g_joint_feat"] = args[8].grad
    res.update({tag + "_g_" + n: p.grad for n, p in dec.named_parameters()})
    bad = [_mismatch(t2n(lattice(v)), g[k], k, e32.get(k, 0.0)) for k, v in res.items()]
    bad = [m for m in bad if m]
    assert not bad, "\n".join(bad)


def _hand_scene(cuda, B=1, L=5, seed=0):
    """config-size scene: 64 x 64 primitives of 8 x 16 x 16 voxels in a hand-sized box, volradius 2000."""
    gen = torch.Generator().manual_seed(seed)
    K, U = 4096, 1024
    q, _ = torch.linalg.qr(torch.randn(B, K, 3, 3, generator=gen))
    s = {"campos": torch.randn(B, 3, generator=gen) * 1500.0,
         "primpos": torch.randn(B, K, 3, generator=gen) * torch.tensor([250.0, 120.0, 250.0]),
         "primrot": q, "primscale": 60.0 + 40.0 * torch.rand(B, K, 3, generator=gen),
         "primalpha": torch.randn(B, 8, 1, U, U, generator=gen).abs() * 3.0,
         "valid_prims": (torch.rand(K, generator=gen) > 0.1).float(),
         "light_pos": F.normalize(torch.randn(B, L, 3, generator=gen), dim=-1) * 6000.0,
         "light_intensity": torch.rand(B, L, 3, generator=gen) + 0.1}
    return {k: v.contiguous().to(cuda) for k, v in s.items()}


def _full_decoder(cuda):
    from goliath_b200.hand_teacher import OLATRGBDecoder

    return OLATRGBDecoder(1024, (16, 16, 8), 64, 64, _rm(2000.0), 2000.0).to(cuda)


def test_shadow_march_vs_expanded_template(cuda):
    """the shared-template march against mvpraymarch(with_shadow=True) on the reference's expanded 4-channel template,
    same rays; the march itself must stay below the memory of one expanded B*L template"""
    from goliath_b200.hand_teacher import light_cameras
    from goliath_b200.mvpraymarch import mvpraymarch
    from goliath_b200.utils import compute_raydirs

    s = _hand_scene(cuda)
    dec = _full_decoder(cuda)
    B, L = s["light_pos"].shape[:2]
    K = 4096
    with torch.no_grad():
        prims = dec._prims(s["primpos"], s["primrot"], s["primscale"], s["primalpha"], s["valid_prims"])
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        shadow = dec.shadow_march(prims, s["light_pos"])
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        template_bytes = B * L * K * 8 * 16 * 16 * 4 * 4
        assert peak < template_bytes, (peak, template_bytes)
        ours = shadow[..., 0:1] / (shadow[..., 1:] + 1e-5)

        alpha = s["primalpha"].reshape(B, 8, 1, 64, 16, 64, 16).permute(0, 3, 5, 1, 4, 6, 2).reshape(B, K, 8, 16, 16, 1)
        alpha = s["valid_prims"][None, :, None, None, None, None] * alpha
        tpl = torch.cat([torch.full((B, K, 8, 16, 16, 3), 255.0, device=cuda), alpha], -1)
        tpl = tpl[:, None].expand(-1, L, -1, -1, -1, -1, -1).reshape(B * L, K, 8, 16, 16, 4).contiguous()
        ex = lambda t: t[:, None].expand(B, L, *t.shape[1:]).reshape(B * L, *t.shape[1:]).contiguous()
        lpos, lrot, focal, princpt = light_cameras(s["primpos"], s["valid_prims"], s["light_pos"], 1024, 1024)
        pix = dec.pixel_coords[None].expand(B * L, -1, -1, -1).contiguous()
        raypos, raydir, tminmax = compute_raydirs(lpos, lrot, focal, princpt, pix, 2000.0)
        _, ref = mvpraymarch(raypos, raydir, 1.0 / 2000.0, tminmax,
                             (ex(s["primpos"] / 2000.0), ex(s["primrot"]), ex(s["primscale"])), tpl, None,
                             with_shadow=True)
    assert (shadow[..., 1] > 0).float().mean() > 0.01
    assert_close(t2n(ours), t2n(ref), rtol=1e-3, atol=1e-3, frac=0.999, what="shadow")


def _features_torch(primpos, primrot, primscale, valid, light_pos, campos, shadow, volradius, X, Y, Z, npx, npy):
    """the feature block of the teacher (hand_teacher_mvp.py:359-439) restated with torch ops"""
    B, K = primpos.shape[:2]
    L = light_pos.shape[1]
    dev = primpos.device
    lz, ly, lx = (torch.linspace(-1.0, 1.0, n, device=dev) for n in (Z, Y, X))
    grid = torch.stack(torch.meshgrid(lz, ly, lx, indexing="ij"))           # [3, Z, Y, X]
    local = grid.permute(0, 3, 2, 1).reshape(3, -1)                         # flat xi*(Y*Z) + yi*Z + zi
    world = volradius * (primpos[..., None] + primrot @ (local / primscale[..., None]))  # [B, K, 3, Z*Y*X]
    world = world.reshape(B, npy, npx, 3, Z, Y, X)                          # ... re-read as (z', y', x')
    rot = primrot.reshape(B, npy, npx, 3, 3)
    mask = valid.reshape(npy, npx)[:, :, None, None, None, None]

    def frame(d):  # [B, h, w, 3, Z, Y, X] -> masked R^T d, laid out [B, Z*3, U, U]
        d = torch.einsum("bhwef,bhwezyx->bhwfzyx", rot, F.normalize(d, dim=3)) * mask
        return d.permute(0, 4, 3, 1, 5, 2, 6).reshape(B, Z * 3, npy * Y, npx * X)

    light = torch.cat([frame(light_pos[:, l, None, None, :, None, None, None] - world) for l in range(L)], 1)
    light = light.reshape(B * L, Z * 3, npy * Y, npx * X)
    view = frame(campos[:, None, None, :, None, None, None] - world)
    view = view[:, None].expand(-1, L, -1, -1, -1).reshape(B * L, Z * 3, npy * Y, npx * X)
    sf = (shadow[..., 0] / (shadow[..., 1] + 1e-5)).reshape(B * L, npy, npx, Z, Y, X)
    sf = sf.permute(0, 3, 1, 4, 2, 5).reshape(B * L, Z, npy * Y, npx * X)
    primshadow = sf.reshape(B, L, Z, 1, npy * Y, npx * X).expand(-1, -1, -1, 3, -1, -1).sum(1) / L
    return torch.cat([light, view, 1.0 - sf], 1), primshadow, sf


def test_features_vs_torch(cuda):
    s = _hand_scene(cuda, seed=1)
    dec = _full_decoder(cuda)
    B, L = s["light_pos"].shape[:2]
    gen = torch.Generator().manual_seed(3)
    shadow = torch.rand(B * L, 4096, 8, 16, 16, 2, generator=gen).to(cuda)
    shadow[..., 1] += 0.05
    with torch.no_grad():
        prims = dec._prims(s["primpos"], s["primrot"], s["primscale"], s["primalpha"], s["valid_prims"])
        feat, primshadow, sf = dec.features(prims, s["campos"], s["light_pos"], shadow, want_shadow_feat=True)
        ref, ref_ps, ref_sf = _features_torch(s["primpos"], s["primrot"], s["primscale"], s["valid_prims"],
                                              s["light_pos"], s["campos"], shadow, 2000.0, 16, 16, 8, 64, 64)
        assert_close(t2n(feat), t2n(ref), rtol=1e-4, what="U-Net input")
        assert_close(t2n(sf), t2n(ref_sf), rtol=1e-6, what="shadow feature")
        assert_close(t2n(primshadow), t2n(ref_ps), rtol=1e-6, what="primshadow")
        again = primshadow.clone()
        dec.features(prims, s["campos"], s["light_pos"], shadow, primshadow=again)
        assert_close(t2n(again), t2n(ref_ps + ref_ps), rtol=1e-6, what="primshadow, second chunk")


@pytest.mark.parametrize("warm", [False, True])
def test_compose_vs_autograd(cuda, warm):
    from goliath_b200.hand_teacher import olat_compose

    B, L, Z, U = 1, 5, 8, 1024
    gen = torch.Generator().manual_seed(5)
    tex = (torch.randn(B * L, 4 * Z, U, U, generator=gen) * 3.0).to(cuda)
    inten = (torch.rand(B, L, 3, generator=gen) + 0.1).to(cuda)
    sf = torch.rand(B * L, Z, U, U, generator=gen).to(cuda) if warm else None
    prev = torch.randn(B, Z, 3, U, U, generator=gen).to(cuda)
    g_rgb = torch.randn(B, Z, 3, U, U, generator=gen).to(cuda)
    g_tol = torch.randn(B, L, Z, 3, U, U, generator=gen).to(cuda)

    t_ref = tex.clone().requires_grad_()
    t = t_ref.view(B, L, Z, 4, U, U)
    s = sf.view(B, L, Z, 1, U, U) if warm else torch.sigmoid(t[:, :, :, :1])
    texolat_ref = 25.0 * t[:, :, :, 1:] + 100.0
    rgb_ref = prev + (s * F.relu(texolat_ref) * inten[:, :, None, :, None, None]).sum(1)
    ((rgb_ref * g_rgb).sum() + (texolat_ref * g_tol).sum()).backward()

    t_ours = tex.clone().requires_grad_()
    rgb, texolat = olat_compose(t_ours, inten, Z, sf, prev.clone(), want_texolat=True)
    assert_close(t2n(rgb), t2n(rgb_ref), rtol=1e-5, what="rgb")
    assert_close(t2n(texolat), t2n(texolat_ref), rtol=1e-6, what="texolat")
    ((rgb * g_rgb).sum() + (texolat * g_tol).sum()).backward()
    assert_close(t2n(t_ours.grad), t2n(t_ref.grad), rtol=1e-5, what="grad tex")
    if warm:
        assert float(t_ours.grad.view(B, L, Z, 4, U, U)[:, :, :, 0].abs().max()) == 0.0


def test_forward_in_cuda_graph(cuda):
    g = np.load(GOLD)
    dec = _golden_decoder(g, cuda).eval()
    args = _golden_inputs(g, cuda)
    args[8] = args[8].detach()
    with torch.no_grad():
        eager = dec(*args)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            dec(*args)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = dec(*args)
        graph.replay()
        torch.cuda.synchronize()
    assert_close(t2n(out["primrgb"]), t2n(eager["primrgb"]), rtol=1e-3, atol=1e-3, frac=0.999, what="graph rgb")
    assert_close(t2n(out["primshadow"]), t2n(eager["primshadow"]), rtol=1e-3, atol=1e-3, frac=0.999,
                 what="graph primshadow")
