"""GPU checks of the body encoders (csrc/downconv_wnub.cu, gb_lbs_unskin_fwd, goliath_b200/{nn,lbs,mesh_vae}.py): every
ConvDownBlock shape of mesh_vae.Encoder / FaceEncoder against the fp64 restatement, the fused input conditioning against
F.interpolate * mask, unpose against fp64 and the reference's fixture, both encoders and `encode` against
tests/golden/body_encoder_ref.npz, and `encode` driving the body decoder.

The module's name sorts it after every other GPU module on purpose: tests/test_body_texture_gpu.py::test_unet_vs_oracle
calibrates its bound on torch's own fp32 error, which depends on what the process allocated before it (it fails after
tests/test_body_decoder_gpu.py alone when the two composite tests between them are deselected), so nothing new runs
ahead of it."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import body_encoder_restate as br
import lbs_recipe as R

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "body_encoder_ref.npz")
BLOCKS = [b + (1,) for b in br.ENCODER_BLOCKS] + [(16, 32, 64, 2), (5, 7, 32, 1)]
KEYS = ("embs", "embs_mu", "embs_logvar")


def _nrel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _maxrel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


class _NoTF32:
    def __enter__(self):
        self.old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("cin,cout,size,groups", BLOCKS)
def test_downconv_block_vs_oracle(cuda, cin, cout, size, groups, B):
    from goliath_b200.nn import ConvDownBlock

    ref = br.seeded_fill(br.ConvDownBlock(cin, cout, size, groups), seed=size + cin + groups).to(cuda)
    blk = ConvDownBlock(cin, cout, size, groups=groups).to(cuda)
    blk.load_state_dict(ref.state_dict(), strict=True)
    g = torch.Generator(device=cuda).manual_seed(size)
    x = torch.randn(B, cin, size, size, device=cuda, generator=g)
    w = torch.randn(B, cout, size // 2, size // 2, device=cuda, generator=g)

    def run(module, dtype):
        module = module.to(dtype)
        xi = x.to(dtype).requires_grad_()
        out = module(xi)
        names = [n for n, _ in module.named_parameters()]
        grads = torch.autograd.grad((out * w.to(dtype)).sum(), [xi] + [p for _, p in module.named_parameters()])
        return out.detach(), dict(zip(["x"] + names, grads))

    with _NoTF32():
        o64, g64 = run(ref, torch.float64)
        o32, g32 = run(ref, torch.float32)
    out, gr = run(blk, torch.float32)
    out2, gr2 = run(blk, torch.float32)
    assert _maxrel(out, o64) <= 1e-4
    assert set(gr) == set(g64)
    for n in g64:
        bound = max(1e-4, 4 * _nrel(g32[n], g64[n]))
        assert _nrel(gr[n], g64[n]) <= bound, (n, _nrel(gr[n], g64[n]), bound)
        assert torch.equal(gr[n], gr2[n]), n      # fixed-order sums: the same bits on every run
    assert torch.equal(out, out2)


@pytest.mark.parametrize("case", ["body", "face", "ratio_0.75"])
def test_fused_conditioning(cuda, case):
    """the first block's input resize + mask against F.interpolate * mask feeding the same block: the body ratio
    (1024 -> 512), the face window read in place, and 384 x 640 -> 512 (one axis up, one down)"""
    from goliath_b200.nn import ConvDownBlock

    g = torch.Generator(device=cuda).manual_seed(4)
    blk = ConvDownBlock(3, 8, 512).to(cuda)
    blk.load_state_dict(br.seeded_fill(br.ConvDownBlock(3, 8, 512), seed=1).state_dict())
    mask = (torch.rand(1, 1, 512, 512, device=cuda, generator=g) < 0.8)
    full = torch.randn(2, 3, 1024, 1024, device=cuda, generator=g)
    src = {"body": full, "face": full[:, :, 512:, :512], "ratio_0.75": full[:, :, :384, 100:740]}[case]
    assert case == "body" or not src.is_contiguous()
    want_in = F.interpolate(src * 0.7, size=(512, 512), mode="bilinear") * mask
    w = torch.randn(2, 8, 256, 256, device=cuda, generator=g)
    params = list(blk.parameters())
    got = blk(src, resize_mask=mask, scale=0.7)
    want = blk(want_in)
    assert _maxrel(got, want) <= 2e-6
    gg = torch.autograd.grad((got * w).sum(), params)
    gw = torch.autograd.grad((want * w).sum(), params)
    for (n, _), a, b in zip(blk.named_parameters(), gg, gw):
        assert _nrel(a, b) <= 2e-6, n
    with pytest.raises(RuntimeError, match="no backward"):
        blk(src.clone().requires_grad_(), resize_mask=mask)


def _lbs(cuda, kind="tree24", seed=100, degenerate=None):
    from goliath_b200.lbs import LBSModule

    model, cfg, template, scales = R.skinned_model(kind, seed)
    m = LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0]).to(cuda)
    if degenerate is not None:
        m.lbs_fn.skin_weights[degenerate] = 0.0     # every influence zero: the blended matrix is the zero matrix
    return m


@pytest.mark.parametrize("B", [1, 3])
def test_unpose_vs_reference_fixture(cuda, B):
    """The error bound follows the conditioning: the synthetic skeleton blends up to eight unrelated joint transforms
    per vertex, so some blended matrices are close to singular (the fixture keeps each vertex's condition number);
    the skeleton test accepts the fp32 joint matrices within 1e-4 of their largest entry, and the inverse amplifies
    their error by that number, so the bound is that allowance times the condition number."""
    g = np.load(GOLD)
    m = _lbs(cuda)
    reg = torch.from_numpy(g["unpose_B%d_in" % B]).to(cuda)
    mo = R.motion(B, 400 + B).to(cuda)
    out = m.unpose(reg, mo)
    ref, cond = torch.from_numpy(g["unpose_B%d_out" % B]).to(cuda), torch.from_numpy(g["unpose_B%d_cond" % B]).to(cuda)
    err = (out - ref).norm(dim=-1)
    bound = 1e-4 * cond * (ref.norm(dim=-1) + 1.0)
    assert bool((err <= bound).all()), float((err / bound).max())
    # and against the fp64 inverse of the same fp32 joint matrices: only the final rounding is left
    f = m.lbs_fn
    mats = f.skeleton(mo, m.lbs_scale.reshape(1, -1).expand(B, -1)).double()
    want = br.unskinning(mats, f.skin_indices, f.skin_weights.double(), reg.double() / m.global_scaling.double()) \
        - m.lbs_template_verts.double()
    assert float(((out - want).norm(dim=-1) / (want.norm(dim=-1) + 1.0)).max()) <= 1e-6
    # pose(unpose(v)) returns v
    back = m.pose(out, mo)
    assert float(((back - reg).norm(dim=-1) / (1e-4 * cond * (reg.norm(dim=-1) + 1.0))).max()) <= 1.0
    plain = f.unpose(mo, m.lbs_scale.reshape(1, -1).expand(B, -1), reg) - m.lbs_template_verts
    scaled = f.unskin(mats.float(), reg, m.lbs_template_verts, torch.ones(3, device=cuda))
    assert torch.allclose(plain, scaled, rtol=1e-6, atol=1e-6)
    with pytest.raises(RuntimeError, match="no backward"):
        m.unpose(reg.clone().requires_grad_(), mo)


def test_unpose_degenerate_vertex_is_nan(cuda):
    g = np.load(GOLD)
    reg = torch.from_numpy(g["unpose_B3_in"]).to(cuda)
    mo = R.motion(3, 403).to(cuda)
    good = _lbs(cuda).unpose(reg, mo)
    out = _lbs(cuda, degenerate=7).unpose(reg, mo)
    assert bool(torch.isnan(out[:, 7]).all())
    keep = torch.ones(reg.shape[1], dtype=torch.bool, device=cuda)
    keep[7] = False
    assert torch.equal(out[:, keep], good[:, keep]) and bool(torch.isfinite(good).all())


def _encoders(cuda):
    from goliath_b200.mesh_vae import Encoder, FaceEncoder

    mask = br.synthetic_mask()
    refs = (br.seeded_fill(br.Encoder(n_embs=1024, mask=mask)), br.seeded_fill(br.FaceEncoder(mask=mask, n_embs=256)))
    enc, face = Encoder(n_embs=1024, mask=mask).to(cuda), FaceEncoder(mask=mask, n_embs=256).to(cuda)
    enc.load_state_dict(refs[0].state_dict(), strict=True)
    face.load_state_dict(refs[1].state_dict(), strict=True)
    return enc, face, refs


def test_encoders_vs_reference_fixture(cuda):
    g = np.load(GOLD)
    enc, face, refs = _encoders(cuda)
    enc.eval(), face.eval()
    for B in (1, 2):
        uv = br.seeded_uv(B).to(cuda)
        for name, prefix, mod in (("encoder", "", enc), ("encoder_face", "face_", face)):
            out = mod(uv)
            assert set(out) == {prefix + k for k in KEYS}
            for k in KEYS:
                assert _maxrel(out[prefix + k].cpu(), torch.from_numpy(g["%s_B%d_%s" % (name, B, k)])) <= 1e-4, (name, k)
            assert torch.equal(out[prefix + "embs"], out[prefix + "embs_mu"])
            assert out[prefix + "embs"].data_ptr() != out[prefix + "embs_mu"].data_ptr()
    # gradients of the fixture's linear functional at B = 2
    for name, prefix, mod in (("encoder", "", enc), ("encoder_face", "face_", face)):
        out = mod(uv)
        gen = torch.Generator().manual_seed(5)
        loss = sum((out[prefix + k] * torch.randn(out[prefix + k].shape, generator=gen).to(cuda)).sum() for k in KEYS[1:])
        params = dict(mod.named_parameters())
        sub = "encoder." if prefix else ""
        grads = torch.autograd.grad(loss, [params[sub + n] for n in br.GRAD_PARAMS])
        for n, gr in zip(br.GRAD_PARAMS, grads):
            assert _nrel(gr.cpu(), torch.from_numpy(g["%s_grad_%s" % (name, n)])) <= 2e-4, (name, n)


def test_encoder_training_noise_and_bitwise_backward(cuda):
    enc, _, _ = _encoders(cuda)
    enc.noise_std = 0.5
    uv = br.seeded_uv(2).to(cuda)
    enc.train()
    torch.manual_seed(11)
    out = enc(uv)
    torch.manual_seed(11)
    noise = torch.randn_like(out["embs_mu"])
    want = out["embs_mu"] + torch.exp(out["embs_logvar"]) * noise * 0.5
    assert torch.equal(out["embs"], want) and not torch.equal(out["embs"], out["embs_mu"])
    grads = []
    for _ in range(2):
        torch.manual_seed(11)
        o = enc(uv)
        grads.append(torch.autograd.grad(o["embs"].square().sum() + o["embs_logvar"].sum(), list(enc.parameters())))
    for (n, _), a, b in zip(enc.named_parameters(), *grads):
        assert torch.equal(a, b) and bool(torch.isfinite(a).all()), n
    with pytest.raises(RuntimeError, match="no backward"):
        enc(uv.clone().requires_grad_())


def _body(cuda):
    """LBS module on the tube mesh and the tube's UV layout at 1024^2"""
    from goliath_b200.geom import GeometryModule
    from goliath_b200.lbs import LBSModule

    model, cfg, template, scales = R.tube_model(7)
    lbs = LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0]).to(cuda)
    tube = R.TubeGeometry()
    index, _, bary = tube.render_index_images(1024)
    v2uv = torch.arange(lbs.lbs_fn.num_verts, dtype=torch.int32)[:, None].expand(-1, 4).contiguous()
    geo = GeometryModule(tube.vi.to(torch.int32), index, bary, vt=tube.vt, v2uv=v2uv).to(cuda)
    return lbs, geo


def _registered(lbs, B, seed, cuda):
    mo = R.motion(B, seed).to(cuda)
    g = torch.Generator().manual_seed(seed)
    return lbs.pose(0.1 * torch.randn(B, lbs.lbs_fn.num_verts, 3, generator=g).to(cuda), mo), mo


def test_encode_end_to_end_and_graph_replay(cuda):
    from goliath_b200 import mesh_vae
    from goliath_b200.graph import Graphed

    enc, face, refs = _encoders(cuda)
    enc.eval(), face.eval()
    lbs, geo = _body(cuda)
    reg, mo = _registered(lbs, 2, 31, cuda)
    with torch.no_grad():
        out = mesh_vae.encode(lbs, geo, enc, face, reg, mo)
        uv = geo.to_uv(lbs.unpose(reg, mo))
        want = {**refs[0].to(cuda).double().eval()(uv.double()), **refs[1].to(cuda).double().eval()(uv.double())}
    assert set(out) == set(want) and len(out) == 6
    for k in want:
        assert _maxrel(out[k], want[k]) <= 1e-4, k
    # no host synchronisation, and a captured graph replayed on new inputs equals the eager result
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.no_grad():
            mesh_vae.encode(lbs, geo, enc, face, reg, mo)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    reg_in, mo_in = reg.clone(), mo.clone()
    with torch.no_grad():
        gr = Graphed(lambda: mesh_vae.encode(lbs, geo, enc, face, reg_in, mo_in))
        reg2, mo2 = _registered(lbs, 2, 32, cuda)
        reg_in.copy_(reg2), mo_in.copy_(mo2)
        replay = gr()
        eager = mesh_vae.encode(lbs, geo, enc, face, reg2, mo2)
    for k in eager:
        assert torch.equal(replay[k], eager[k]) and not torch.equal(eager[k], out[k]), k


def test_encode_drives_the_decoder(cuda):
    """encode -> ConvDecoder -> LBSModule.pose, trained through: the decoder is driven by an encoded code"""
    import seams_restate as sr
    from goliath_b200 import mesh_vae
    from oracle import mesh_vae_oracle as mo_

    enc, face, _ = _encoders(cuda)
    enc.train(), face.train()
    lbs, geo = _body(cuda)
    cfg = dict(uv_size=1024, init_uv_size=64, n_pose_dims=6, n_pose_enc_channels=16, n_embs=1024,
               n_embs_enc_channels=32, n_face_embs=256, n_init_channels=64, n_min_channels=4)
    dec = mesh_vae.ConvDecoder(geo, seam_sampler=sr.stand_in_sampler(), assets=mo_.synthetic_masks(n_pose_dims=6),
                               **cfg).to(cuda)
    mo_.seeded_fill(dec, seed=3)
    reg, mo = _registered(lbs, 1, 41, cuda)
    torch.manual_seed(0)
    codes = mesh_vae.encode(lbs, geo, enc, face, reg, mo)
    preds = dec(mo, codes["embs"], codes["face_embs"])
    geom = lbs.pose(preds["geom_delta_rec"], mo)
    loss = (geom - reg).square().mean() + preds["tex_mean_rec"].square().mean()
    params = list(enc.parameters()) + list(face.parameters())
    grads = torch.autograd.grad(loss, params)
    for (n, _), gr in zip(list(enc.named_parameters()) + list(face.named_parameters()), grads):
        assert bool(torch.isfinite(gr).all()) and float(gr.abs().max()) > 0, n
