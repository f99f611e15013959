"""GPU checks of the body decoder (DESIGN.md row R9: csrc/upconv_wnub.cu, goliath_b200/{nn,seams,geom,mesh_vae}.py):
every UpConvBlockDeep shape of mesh_vae.ConvDecoder against the fp64 oracle block, the seam sampler and from_uv
against the reference's fixture (tests/golden/seams_ref.npz) and the torch restatement at 1024^2, and the whole decoder
against the reference's fixture (tests/golden/mesh_vae_ref.npz) and the fp64 oracle's autograd."""
import os

import numpy as np
import pytest
import torch

import seams_restate as sr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CFG = dict(uv_size=1024, init_uv_size=64, n_pose_dims=98, n_pose_enc_channels=16, n_embs=1024, n_embs_enc_channels=32,
           n_face_embs=256, n_init_channels=64, n_min_channels=4)
OUTPUTS = ("geom_delta_rec", "geom_uv_delta_rec", "tex_mean_rec", "embs_conv", "pose_conv")
BLOCKS = [(128, 128, 8, 1), (128, 128, 16, 1), (128, 64, 32, 1), (64, 32, 64, 1), (32, 64, 8, 1), (64, 64, 16, 1),
          (64, 32, 32, 1), (128, 64, 128, 2), (64, 32, 256, 2), (32, 16, 512, 2), (16, 8, 1024, 2)]


def _nrel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _maxrel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("cin,cout,size,groups", BLOCKS)
def test_upconv_block_vs_oracle(cuda, cin, cout, size, groups, B):
    from goliath_b200.nn import UpConvBlockDeep
    from oracle import mesh_vae_oracle as mo

    ref = mo.seeded_fill(mo.UpConvBlockDeep(cin, cout, size, groups), seed=size + cin + groups).to(cuda)
    blk = UpConvBlockDeep(cin, cout, size, groups=groups).to(cuda)
    blk.load_state_dict(ref.state_dict(), strict=True)
    g = torch.Generator(device=cuda).manual_seed(size)
    x = torch.randn(B, cin, size // 2, size // 2, device=cuda, generator=g)
    w = torch.randn(B, cout, size, size, device=cuda, generator=g)

    def run(module, dtype):
        module = module.to(dtype)
        xi = x.to(dtype).requires_grad_()
        out = module(xi)
        names = [n for n, _ in module.named_parameters()]
        grads = torch.autograd.grad((out * w.to(dtype)).sum(), [xi] + [p for _, p in module.named_parameters()])
        return out.detach(), dict(zip(["x"] + names, grads))

    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        o64, g64 = run(ref, torch.float64)
        o32, g32 = run(ref, torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    out, gr = run(blk, torch.float32)
    out2, gr2 = run(blk, torch.float32)
    assert _maxrel(out, o64) <= 1e-4
    assert set(gr) == set(g64)
    for n in g64:
        bound = max(1e-4, 4 * _nrel(g32[n], g64[n]))
        assert _nrel(gr[n], g64[n]) <= bound, (n, _nrel(gr[n], g64[n]), bound)
        assert torch.equal(gr[n], gr2[n]), n      # fixed-order sums: the same bits on every run
    assert torch.equal(out, out2)


def _gpu_seams(g, cuda):
    from goliath_b200.seams import SeamSampler

    return SeamSampler({k: g[k] for k in ("dst_ij", "src_ij", "uvs", "weights")}).to(cuda)


def test_seams_and_from_uv_vs_fixture(cuda):
    from goliath_b200 import geom

    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(HERE, "golden", "seams_ref.npz")).items()}
    s = _gpu_seams(g, cuda)
    tex = g["tex"].float().to(cuda).requires_grad_()
    outs = {"impaint": s.impaint(tex), "resample": s.resample(tex), "forward": s(tex),
            "chain": s.resample(s.resample(s.impaint(tex)))}
    for k, t in outs.items():
        assert _maxrel(t.cpu(), g[k]) <= 1e-5, k
        (gt,) = torch.autograd.grad((t * g["w_" + k].float().to(cuda)).sum(), [tex])
        assert _maxrel(gt.cpu(), g["g_" + k]) <= 1e-5, k
    uvmap = g["uvmap"].float().to(cuda).requires_grad_()
    mod = geom.GeometryModule(torch.zeros(1, 3, dtype=torch.int32), torch.zeros(1, 1, 3), torch.zeros(1, 1, 3),
                              vt=g["vt"], v2uv=g["v2uv"]).to(cuda)
    for sv in (geom.sample_uv(uvmap, g["vt"].to(cuda), g["v2uv"].to(cuda)), mod.from_uv(uvmap)):
        assert _maxrel(sv.detach().cpu(), g["sample_uv"]) <= 1e-5
        (gu,) = torch.autograd.grad((sv * g["w_sample_uv"].float().to(cuda)).sum(), [uvmap])
        assert _maxrel(gu.cpu(), g["g_uvmap"]) <= 1e-5


def test_seams_and_from_uv_at_1024(cuda):
    from goliath_b200 import geom
    from goliath_b200.seams import SeamSampler

    data = sr.synthetic_seams(1024)
    s = SeamSampler(data).to(cuda)
    ts = sr.TorchSeamSampler(*(data[k].to(cuda) for k in ("dst_ij", "src_ij", "uvs", "weights")))
    gen = torch.Generator(device=cuda).manual_seed(0)
    x = torch.randn(2, 8, 1024, 1024, device=cuda, generator=gen)
    w = torch.randn(2, 8, 1024, 1024, device=cuda, generator=gen)
    xd = x.double().requires_grad_()
    ref = ts.resample(ts.resample(ts.impaint(xd)))
    (gref,) = torch.autograd.grad((ref * w.double()).sum(), [xd])
    xg = x.clone().requires_grad_()
    grads = []
    for _ in range(2):
        out = s.resample(s.resample(s.impaint(xg)))
        grads.append(torch.autograd.grad((out * w).sum(), [xg])[0])
    assert _maxrel(out, ref) <= 1e-5 and _maxrel(grads[0], gref) <= 1e-5
    assert torch.equal(grads[0], grads[1])
    # impaint + resample in one gather
    assert _maxrel(s(x), ts.resample(ts.impaint(x.double()))) <= 1e-5
    # from_uv at the decoder's size, padded v2uv rows
    rng = np.random.default_rng(1)
    vt = torch.as_tensor(rng.random((9000, 2)) * 1.02 - 0.01, dtype=torch.float32)
    v2uv = torch.as_tensor(rng.integers(0, 9000, (7306, 4)), dtype=torch.int32)
    v2uv[::3, 2:] = v2uv[::3, :1]
    uv = torch.randn(2, 3, 1024, 1024, device=cuda, generator=gen)
    mod = geom.GeometryModule(torch.zeros(1, 3, dtype=torch.int32), torch.zeros(1, 1, 3), torch.zeros(1, 1, 3),
                              vt=vt, v2uv=v2uv).to(cuda)
    wv = torch.randn(2, 7306, 3, device=cuda, generator=gen)
    uvd = uv.double().requires_grad_()
    rv = sr.sample_uv(uvd, vt.to(cuda).double(), v2uv.to(cuda))
    (grv,) = torch.autograd.grad((rv * wv.double()).sum(), [uvd])
    uvg = uv.clone().requires_grad_()
    gg = []
    for _ in range(2):
        v = mod.from_uv(uvg)
        gg.append(torch.autograd.grad((v * wv).sum(), [uvg])[0])
    assert _maxrel(v, rv) <= 1e-5 and _maxrel(gg[0], grv) <= 1e-5 and torch.equal(gg[0], gg[1])


def _pair(cuda, B, seams=None, seed=20240613):
    from goliath_b200.mesh_vae import ConvDecoder
    from oracle import mesh_vae_oracle as mo

    ref_seam = sr.stand_in_sampler() if seams is None else sr.TorchSeamSampler(*(seams[k].to(cuda) for k in (
        "dst_ij", "src_ij", "uvs", "weights")))
    from_uv = sr.uv_vertex_gather()
    ref = mo.seeded_fill(mo.ConvDecoder(mo.synthetic_masks(), None, None), seed=seed).to(cuda)
    ref.from_uv = from_uv.from_uv
    if seams is None:
        dec_seam = sr.stand_in_sampler()
    else:
        from goliath_b200.seams import SeamSampler

        dec_seam = SeamSampler(seams).to(cuda)
    dec = ConvDecoder(from_uv, seam_sampler=dec_seam, assets=mo.synthetic_masks(), **CFG).to(cuda)
    dec.load_state_dict(ref.state_dict(), strict=False)
    pose, embs, face = (t.to(cuda) for t in mo.seeded_inputs(batch=B))
    return ref, ref_seam, dec, (pose, embs, face)


def _oracle_forward(ref, seam, inputs):
    """oracle.mesh_vae_oracle.ConvDecoder.forward with impaint, resample, resample as the decoder calls them"""
    calls = iter((seam.impaint, seam.resample, seam.resample))
    ref.resample = lambda x: next(calls)(x)
    return ref(*inputs)


def test_decoder_forward_vs_reference_fixture(cuda):
    ref, seam, dec, inputs = _pair(cuda, 1)
    g = np.load(os.path.join(HERE, "golden", "mesh_vae_ref.npz"))
    with torch.no_grad():
        out = dec(*inputs)
        want = _oracle_forward(ref, seam, inputs)
    for k in OUTPUTS:
        t = out[k].double().reshape(-1).cpu()
        r = g["out_" + k]
        assert list(out[k].shape) == g["shape_" + k].tolist(), k
        got = np.concatenate([[t.mean().item(), t.std().item(), t.abs().max().item()],
                              t[torch.linspace(0, t.numel() - 1, 256).long()].numpy()])
        exp = np.concatenate([r[:3], r[4:]])
        assert np.all(np.abs(got - exp) <= 1e-4 * r[2] + 1e-5 * np.abs(exp)), (k, np.abs(got - exp).max(), r[2])
        assert _maxrel(out[k], want[k]) <= 1e-4, k


def test_decoder_with_gpu_seam_sampler(cuda):
    seams = sr.synthetic_seams(1024)
    ref, seam, dec, inputs = _pair(cuda, 2, seams=seams)
    with torch.no_grad():
        out = dec(*inputs)
        want = _oracle_forward(ref, seam, inputs)
    for k in OUTPUTS:
        assert _maxrel(out[k], want[k]) <= 1e-4, k


def test_decoder_backward_vs_fp64_oracle(cuda):
    ref, seam, dec, inputs = _pair(cuda, 4)
    gen = torch.Generator(device=cuda).manual_seed(9)
    with torch.no_grad():
        shapes = {k: v.shape for k, v in dec(*inputs).items()}
    ws = {k: torch.randn(s, device=cuda, generator=gen) for k, s in shapes.items()}

    def grads(module, dtype, oracle):
        module = module.to(dtype)
        inp = [t.to(dtype) for t in inputs]
        out = _oracle_forward(module, seam, inp) if oracle else module(*inp)
        loss = sum((out[k] * ws[k].to(dtype)).sum() for k in OUTPUTS)
        names = [n for n, _ in module.named_parameters()]
        return out, dict(zip(names, torch.autograd.grad(loss, [p for _, p in module.named_parameters()])))

    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        o64, g64 = grads(ref, torch.float64, True)
        _, g32 = grads(ref, torch.float32, True)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    out, gd = grads(dec, torch.float32, False)
    for k in OUTPUTS:
        assert _maxrel(out[k], o64[k]) <= 1e-4, k
    assert set(gd) == set(g64)
    bad = []
    for n in g64:
        bound = max(1e-4, 4 * _nrel(g32[n], g64[n]))
        if _nrel(gd[n], g64[n]) > bound:
            bad.append((n, _nrel(gd[n], g64[n]), bound))
    assert not bad, bad


def test_decoder_sync_free_and_graph_replay(cuda):
    from goliath_b200.geom import GeometryModule
    from goliath_b200.graph import Graphed

    seams = sr.synthetic_seams(1024)
    _, _, dec, inputs = _pair(cuda, 2, seams=seams)
    rng = np.random.default_rng(2)
    vt = torch.as_tensor(rng.random((9000, 2)), dtype=torch.float32)
    v2uv = torch.as_tensor(rng.integers(0, 9000, (7306, 4)), dtype=torch.int32)
    dec.geo_fn = GeometryModule(torch.zeros(1, 3, dtype=torch.int32), torch.zeros(1, 1, 3), torch.zeros(1, 1, 3),
                                vt=vt, v2uv=v2uv).to(cuda)
    pose, embs, face = (t.clone().requires_grad_(False) for t in inputs)
    out = dec(pose, embs, face)                   # builds the gather tables
    sum(v.sum() for v in out.values()).backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = dec(pose, embs, face)
        sum(v.sum() for v in out.values()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    with torch.no_grad():
        eager = {k: v.clone() for k, v in dec(pose, embs, face).items()}
        gr = Graphed(lambda: dec(pose, embs, face))
        replay = gr()
        for k in OUTPUTS:
            assert torch.equal(replay[k], eager[k]), k
