"""CPU checks of the body encoders: the plain-torch restatement (tests/body_encoder_restate.py) against the fixture
frozen from the reference's own run (tests/golden/body_encoder_ref.npz), the state-dict layout of the library's
modules against the reference's frozen key list, the fp64 unskinning round trip, and argument validation."""
import json
import os

import numpy as np
import pytest
import torch

import body_encoder_restate as br
import lbs_recipe as R

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "body_encoder_ref.npz")
KEYS = ("embs", "embs_mu", "embs_logvar")


def _frozen(g, name):
    return json.loads(bytes(g[name + "_keys_json"]).decode())


def _layout(module):
    return {k: [list(v.shape), str(v.dtype)] for k, v in module.state_dict().items()}


def test_restatement_vs_reference_fixture():
    g = np.load(GOLD)
    mask = br.synthetic_mask()
    uv = br.seeded_uv(2)
    for name, prefix, mod in (("encoder", "", br.Encoder(n_embs=1024, mask=mask)),
                              ("encoder_face", "face_", br.FaceEncoder(mask=mask, n_embs=256))):
        br.seeded_fill(mod).eval()
        out = mod(uv)
        for k in KEYS:
            want = torch.from_numpy(g["%s_B2_%s" % (name, k)])
            assert float((out[prefix + k].detach() - want).abs().max() / want.abs().max()) <= 2e-5, (name, k)
        gen = torch.Generator().manual_seed(5)
        loss = sum((out[prefix + k] * torch.randn(out[prefix + k].shape, generator=gen)).sum() for k in KEYS[1:])
        params = dict(mod.named_parameters())
        sub = "encoder." if prefix else ""
        grads = torch.autograd.grad(loss, [params[sub + n] for n in br.GRAD_PARAMS])
        for n, gr in zip(br.GRAD_PARAMS, grads):
            want = torch.from_numpy(g["%s_grad_%s" % (name, n)])
            assert float((gr - want).norm() / want.norm()) <= 1e-4, (name, n)


def test_state_dict_layout_is_the_references():
    """a reference checkpoint's `encoder.*` / `encoder_face.*` entries load with strict=True: same keys, shapes and
    dtypes, the bool mask buffer included"""
    from goliath_b200.mesh_vae import Encoder, FaceEncoder
    from goliath_b200.nn import ConvDownBlock

    g = np.load(GOLD)
    mask = br.synthetic_mask()
    enc, face = Encoder(n_embs=1024, mask=mask), FaceEncoder(mask=mask, n_embs=256)
    assert _layout(enc) == _frozen(g, "encoder")
    assert _layout(face) == _frozen(g, "encoder_face")
    assert torch.equal(enc.mask, br.Encoder(n_embs=4, mask=mask).mask) and enc.mask.dtype == torch.bool
    ref = br.seeded_fill(br.FaceEncoder(mask=mask, n_embs=256))
    face.load_state_dict(ref.state_dict(), strict=True)
    blk = {k: list(v.shape) for k, v in ConvDownBlock(8, 16, 256).state_dict().items()}
    want = {k[len("joint_conv_blocks.0."):]: v[0] for k, v in _frozen(g, "encoder").items()
            if k.startswith("joint_conv_blocks.0.")}
    assert blk == want and len(blk) == 9
    grouped = ConvDownBlock(16, 32, 64, groups=2)
    assert _layout(grouped) == _layout(br.ConvDownBlock(16, 32, 64, groups=2))
    assert grouped.conv2.weight_v.shape == (32, 8, 3, 3) and grouped.conv2.bias.shape == (32, 32, 32)


def test_glorot_init_matches_the_reference_bounds():
    from goliath_b200.mesh_vae import Encoder

    enc = Encoder(n_embs=32, mask=br.synthetic_mask())
    c2 = enc.joint_conv_blocks[1].conv2              # 16 -> 32, 3x3: bound = gain * sqrt(2 / ((16 + 32) * 9)) * sqrt(3)
    bound = np.sqrt(2 / 1.04) * np.sqrt(2.0 / (48 * 9)) * np.sqrt(3.0)
    assert 0.9 * bound < float(c2.weight_v.abs().max()) <= bound * (1 + 1e-6)
    assert float(c2.bias.abs().max()) == 0.0
    assert float((c2.weight - c2.weight_v).abs().max()) <= 1e-6 * bound     # g = ||v||: the weight is the sample


def test_unskinning_round_trip_fp64():
    model, cfg, _, _ = R.skinned_model("tree24", 100)
    from goliath_b200.lbs import LinearBlendSkinning

    f = LinearBlendSkinning(model, cfg)
    g = torch.Generator().manual_seed(1)
    rot = torch.linalg.qr(torch.randn(2, 24, 3, 3, generator=g, dtype=torch.float64))[0]
    mats = torch.cat([rot * (0.5 + torch.rand(2, 24, 1, 1, generator=g, dtype=torch.float64)),
                      torch.randn(2, 24, 3, 1, generator=g, dtype=torch.float64)], -1)
    v = torch.randn(2, f.num_verts, 3, generator=g, dtype=torch.float64)
    w = f.skin_weights.double()
    posed = br.skinning(mats, f.skin_indices, w, v)
    cond = torch.linalg.cond(br.blended(mats, f.skin_indices, w)[..., :3])
    assert float(((br.unskinning(mats, f.skin_indices, w, posed) - v).norm(dim=-1) / cond).max()) <= 1e-13
    assert float(((br.skinning(mats, f.skin_indices, w, br.unskinning(mats, f.skin_indices, w, v)) - v).norm(dim=-1)
                  / cond).max()) <= 1e-13


def test_argument_validation():
    from goliath_b200.lbs import LBSModule
    from goliath_b200.mesh_vae import Encoder, FaceEncoder
    from goliath_b200.nn import ConvDownBlock

    mask = br.synthetic_mask()
    with pytest.raises(ValueError, match="mask must be"):
        Encoder(n_embs=8, mask=mask[None])
    with pytest.raises(ValueError, match="mask must be"):
        FaceEncoder(mask=mask[:512], n_embs=8)
    with pytest.raises(ValueError):
        ConvDownBlock(8, 16, 63)
    with pytest.raises(ValueError):
        ConvDownBlock(6, 16, 64, groups=4)
    with pytest.raises(NotImplementedError):
        ConvDownBlock(8, 16, 64, wnorm_dim=1)
    enc = Encoder(n_embs=8, mask=mask)
    with pytest.raises(RuntimeError, match="CUDA only"):
        enc(torch.zeros(1, 3, 1024, 1024))
    blk = ConvDownBlock(8, 16, 64)
    with pytest.raises(RuntimeError, match="CUDA"):
        blk(torch.zeros(1, 8, 64, 64))
    with pytest.raises(RuntimeError, match="needs a"):
        blk(torch.zeros(1, 8, 32, 32))
    with pytest.raises(RuntimeError, match="resize_mask"):
        blk(torch.zeros(1, 8, 64, 64), resize_mask=torch.ones(1, 1, 32, 32, dtype=torch.bool))
    with pytest.raises(NotImplementedError, match="inside the block"):
        blk.conv2(torch.zeros(1, 8, 64, 64))
    model, cfg, template, scales = R.skinned_model("tree24", 100)
    m = LBSModule(model, cfg, template, scales, global_scaling=[10.0, 10.0, 10.0])
    with pytest.raises(RuntimeError, match="CUDA"):
        m.unpose(torch.zeros(1, m.lbs_fn.num_verts, 3), torch.zeros(1, 12))
