"""CPU checks of the body decoder (DESIGN.md row R9, goliath_b200/mesh_vae.py): the checkpoint layout of the
reference's `mesh_vae.ConvDecoder`, strict loading of a state dict of the oracle restatement, the torch restatement
of the seam sampler and sample_uv (tests/seams_restate.py) against the reference's own run (tests/golden/seams_ref.npz),
and the refusal of CPU tensors."""
import json
import os
import types

import numpy as np
import pytest
import torch

import seams_restate as sr

HERE = os.path.dirname(os.path.abspath(__file__))
MESH_GOLD = os.path.join(HERE, "golden", "mesh_vae_ref.npz")
SEAMS_GOLD = os.path.join(HERE, "golden", "seams_ref.npz")
CFG = dict(uv_size=1024, init_uv_size=64, n_pose_dims=98, n_pose_enc_channels=16, n_embs=1024, n_embs_enc_channels=32,
           n_face_embs=256, n_init_channels=64, n_min_channels=4)  # mesh_vae_example.yml


def _decoder(**kw):
    from goliath_b200.mesh_vae import ConvDecoder
    from oracle import mesh_vae_oracle as mo

    cfg = dict(CFG, **kw)
    return ConvDecoder(types.SimpleNamespace(from_uv=lambda t: t), seam_sampler=sr.stand_in_sampler(),
                       assets=mo.synthetic_masks(), **cfg)


def test_checkpoint_layout_matches_the_reference():
    g = np.load(MESH_GOLD)
    dec = _decoder()
    keys = json.loads(bytes(g["keys_json"]).decode())
    assert {k: list(v.shape) for k, v in dec.state_dict().items()} == keys
    assert sum(p.numel() for p in dec.parameters()) == int(g["n_params"]) == 58_739_420
    assert dec.pose_cond_mask.dtype == torch.int32 and dec.n_channels == [64, 32, 16, 8, 4]
    assert [b.groups for b in dec.conv_blocks] == [2, 2, 2, 2]
    assert tuple(dec.conv_blocks[-1].conv1.weight_v.shape) == (16, 8, 3, 3)
    # the reference's glorot: effective weight == weight_v, bias zero
    c = dec.conv_blocks[0].conv2
    assert torch.allclose(c.weight.detach(), c.weight_v, rtol=1e-5, atol=1e-7) and float(c.bias.abs().max()) == 0.0


def test_oracle_state_dict_loads_strictly():
    from oracle import mesh_vae_oracle as mo

    dec = _decoder(uv_size=256)
    ref = mo.seeded_fill(mo.ConvDecoder(mo.synthetic_masks(), None, None, uv_size=256))
    dec.load_state_dict(ref.state_dict(), strict=True)
    for k, v in ref.state_dict().items():
        assert torch.equal(dec.state_dict()[k], v), k


def test_seam_restatement_matches_the_reference_fixture():
    g = {k: torch.from_numpy(v) for k, v in np.load(SEAMS_GOLD).items()}
    s = sr.TorchSeamSampler(g["dst_ij"], g["src_ij"], g["uvs"], g["weights"])
    tex = g["tex"].clone().requires_grad_()
    outs = {"impaint": s.impaint(tex), "resample": s.resample(tex), "forward": s.resample(s.impaint(tex)),
            "chain": s.resample(s.resample(s.impaint(tex)))}
    for k, t in outs.items():
        torch.testing.assert_close(t, g[k], rtol=1e-12, atol=1e-12, msg=k)
        (gt,) = torch.autograd.grad((t * g["w_" + k]).sum(), [tex])
        torch.testing.assert_close(gt, g["g_" + k], rtol=1e-12, atol=1e-12, msg="grad " + k)
    uvmap = g["uvmap"].clone().requires_grad_()
    sv = sr.sample_uv(uvmap, g["vt"], g["v2uv"])
    torch.testing.assert_close(sv, g["sample_uv"], rtol=1e-12, atol=1e-12)
    (gu,) = torch.autograd.grad((sv * g["w_sample_uv"]).sum(), [uvmap])
    torch.testing.assert_close(gu, g["g_uvmap"], rtol=1e-12, atol=1e-12)
    # the fixture's data covers what it is there for
    dst = {tuple(r) for r in g["dst_ij"].tolist()}
    src = [tuple(r) for r in g["src_ij"].tolist()]
    assert len(dst) == len(src) and dst & set(src) and max(src.count(r) for r in src) > 1
    assert float(g["uvs"].min()) < 0 and float(g["uvs"].max()) > 1
    assert {0.0, 1.0} <= set(g["weights"].reshape(-1).tolist())
    assert float(g["vt"].min()) < 0 and float(g["vt"].max()) > 1


def test_cpu_tensors_raise():
    from goliath_b200.nn import UpConvBlockDeep
    from goliath_b200.seams import SeamSampler

    dec = _decoder(uv_size=128)
    with pytest.raises(RuntimeError):
        dec(torch.zeros(1, 104), torch.zeros(1, 1024), torch.zeros(1, 256))
    with pytest.raises(RuntimeError):
        UpConvBlockDeep(8, 4, 16, groups=2)(torch.zeros(1, 8, 8, 8))
    s = SeamSampler(sr.synthetic_seams(32, n_pairs=20))
    with pytest.raises(RuntimeError):
        s.resample(torch.zeros(1, 2, 32, 32))
    with pytest.raises(NotImplementedError):
        UpConvBlockDeep(8, 4, 16, wnorm_dim=1)
