"""CPU checks of the drivable body avatar `goliath_b200.mesh_vae_drivable.AutoEncoder` against
tests/golden/body_drive_ref.npz (the reference's own model, made by tests/golden/make_body_drive_golden.py): the
fixture's shape, the state-dict keys and shapes (a state dict with the reference's keys loads strictly), the buffers the
constructor prepares, the face decoder's checkpoint path, and the errors for unsupported arguments."""
import json
import os

import numpy as np
import pytest
import torch

import body_drive_restate as bd

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "body_drive_ref.npz")


def _json(z, k):
    return json.loads(bytes(z[k]).decode())


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def model():
    from goliath_b200.mesh_vae_drivable import AutoEncoder

    return AutoEncoder(**bd.config(), assets=bd.assets())


def test_fixture_well_formed(gold):
    assert os.path.getsize(GOLD) < 1_000_000
    for mode in ("eval", "train"):
        keys = _json(gold, mode + "_out_keys_json")
        for k in ("geom", "tex_rec", "rgb", "shadow_map", "face_tex_cond", "face_dec_preds.face_tex",
                  "face_dec_preds.face_geom", "learn_blur_weights"):
            assert k in keys, (mode, k)
        assert ("pose_shadow_map" in keys) == (mode == "train")
        assert ("ao_map" in keys) == (mode == "train")
        for k in keys:
            s = gold["%s_out_%s" % (mode, k)]
            assert s.shape == (260,) and np.isfinite(s).all(), k
            assert s[3] == np.prod(gold["%s_shape_out_%s" % (mode, k)]), k
            assert 0.0 <= float(gold["%s_err32_out_%s" % (mode, k)]) < 1e-2, k
        names = _json(gold, mode + "_grad_names_json")
        for m in ("encoder.", "encoder_face.", "decoder.", "decoder_view.", "pose_to_shadow.", "upscale_net.", "cal.",
                  "learn_blur.", "pixel_cal."):
            assert any(n.startswith(m) for n in names), (mode, m)
        assert any(n.startswith("shadow_net.") for n in names) == (mode == "train")
        for n in names:
            assert np.isfinite(gold["%s_grad_%s" % (mode, n)]).all(), n
    assert gold["in_lbs_motion"].shape == (2, 12) and gold["in_face_embs"].shape == (2, 256)


def test_state_dict_keys_match_reference(gold, model):
    want = _json(gold, "keys_json")
    got = {k: list(v.shape) for k, v in model.state_dict().items()}
    assert set(got) == set(want), sorted(set(got) ^ set(want))[:20]
    assert got == want
    for k in ("encoder.geo_fn.index_image", "decoder_face.texmod.14.weight_v", "decoder_face.bias",
              "decoder_face.frontal_view", "encoder_face.tex_cond_mask", "pose_to_shadow.conv_block.8.bias",
              "renderer.image_size"):
        assert k in got, k
    sd = {k: torch.zeros(v) for k, v in want.items()}
    sd["renderer.image_size"] = torch.tensor([bd.H, bd.W])
    model.load_state_dict(sd, strict=True)


def test_constructor_buffers_match_reference(gold):
    from goliath_b200.mesh_vae_drivable import AutoEncoder

    m = AutoEncoder(**bd.config(), assets=bd.assets())
    for k in ("tex_mean", "meye_mask"):
        f = getattr(m, k).double().reshape(-1)
        idx = torch.linspace(0, f.numel() - 1, 256, dtype=torch.float64).long()
        got = np.concatenate([[f.mean().item(), f.std().item(), f.abs().max().item(), float(f.numel())], f[idx].numpy()])
        np.testing.assert_allclose(got, gold["buf_" + k], rtol=2e-6, atol=1e-6 * abs(gold["buf_" + k][2]))
    np.testing.assert_array_equal(m.face_cond_mask.numpy(), gold["buf_face_cond_mask"])
    tcm = m.encoder_face.tex_cond_mask
    assert tcm.dtype == torch.float32
    np.testing.assert_allclose(tcm.numpy(), gold["buf_tex_cond_mask"], rtol=0, atol=1e-6)
    assert 0.0 < float(((tcm > 0) & (tcm < 1)).double().mean())      # a soft mask, not cast to bool
    np.testing.assert_array_equal(m.decoder_face.frontal_view.numpy(), gold["buf_frontal_view"])
    assert m.tex_std == 64.0 and m.pose_to_shadow_enabled and m.encoder.mean_scale == 1.0
    assert m.decoder.tex_scale == 1.0 and m.decoder.verts_scale == 1.0


def test_decoder_face_checkpoint_loads_without_mutating_config(tmp_path):
    from goliath_b200.face import FaceDecoderFrontal
    from goliath_b200.mesh_vae_drivable import AutoEncoder

    a = bd.assets()
    src = FaceDecoderFrontal(a, n_vert_out=3 * bd.N_FACE_VERTS)
    with torch.no_grad():
        src.bias.fill_(0.25)
    sd = {k: v for k, v in src.state_dict().items() if k != "frontal_view"}   # strict=False tolerates the gap
    path = str(tmp_path / "face.pt")
    torch.save(sd, path)
    cfg = bd.config()
    cfg["decoder_face"]["ckpt"] = path
    before = dict(cfg["decoder_face"])
    m = AutoEncoder(**cfg, assets=a)
    assert cfg["decoder_face"] == before
    assert torch.equal(m.decoder_face.bias, src.bias)
    assert torch.equal(m.decoder_face.texmod[0].weight_v, src.texmod[0].weight_v)


def test_unsupported_arguments_raise(model):
    from goliath_b200.face import FaceDecoderFrontal
    from goliath_b200.mesh_vae_drivable import AutoEncoder

    a = bd.assets()
    cfg = bd.config()
    cfg["cal"] = None
    with pytest.raises(ValueError, match="pixel_cal needs cal"):
        AutoEncoder(**cfg, assets=a)
    for drop in ({"renderer": None}, {"renderer": None, "pixel_cal": None}):
        cfg = bd.config()
        cfg.update(drop)
        with pytest.raises(ValueError, match="no renderer"):
            AutoEncoder(**cfg, assets=a)
    with pytest.raises(ValueError, match="encode=False"):
        model(torch.zeros(1, 12), torch.zeros(1, 3), encode=False)
    with pytest.raises(ValueError, match="tex_roi"):
        FaceDecoderFrontal(a, tex_roi=((0, 0), (512, 512)))

