"""CPU checks of the body avatar's frame `goliath_b200.mesh_vae.AutoEncoder` against tests/golden/body_frame_ref.npz
(the reference's own AutoEncoder, made by tests/golden/make_body_frame_golden.py): the fixture's shape, the state-dict
keys and shapes (a state dict with the reference's keys loads strictly), the buffers the constructor prepares on the
CPU, and the errors for missing UV images and unsupported arguments."""
import json
import os

import numpy as np
import pytest
import torch

import body_frame_restate as bf

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "body_frame_ref.npz")
OUT_KEYS = ["geom", "tex_rec", "geom_delta_rec", "geom_uv_delta_rec", "tex_mean_rec", "embs_conv", "pose_conv",
            "shadow_map", "ao_map", "shadow_map_lowres", "tex_view_rec", "cond_view", "embs", "embs_mu", "embs_logvar",
            "face_embs", "face_embs_mu", "face_embs_logvar", "rgb", "alpha", "depth_disc_mask", "depth",
            "learn_blur_weights"]


def _json(z, k):
    return json.loads(bytes(z[k]).decode())


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def model():
    from goliath_b200.mesh_vae import AutoEncoder

    return AutoEncoder(**bf.config(), assets=bf.assets())


def test_fixture_well_formed(gold):
    assert os.path.getsize(GOLD) < 1_000_000
    assert _json(gold, "out_keys_json") == OUT_KEYS
    names = _json(gold, "grad_names_json")
    for m in ("encoder.", "encoder_face.", "decoder.", "decoder_view.", "shadow_net.", "upscale_net.", "cal.",
              "learn_blur.", "pixel_cal."):
        assert any(n.startswith(m) for n in names), m
    for k in OUT_KEYS:
        if k == "depth_disc_mask":
            continue
        s = gold["out_" + k]
        assert s.shape == (260,) and np.isfinite(s).all() and s[3] == np.prod(gold["shape_out_" + k]), k
        assert 0.0 <= float(gold["err32_out_" + k]) < 1e-2, k
    for n in names:
        assert np.isfinite(gold["grad_" + n]).all() and gold["grad_" + n][2] > 0.0, n
    mask = gold["depth_disc_mask"]
    assert mask.dtype == bool and mask.shape == (2, 1, bf.H, bf.W) and 0 < mask.sum() < mask.size // 2
    assert gold["in_pose"].shape == (2, 12) and gold["in_registration_vertices"].shape[0] == 2


def test_state_dict_keys_match_reference(gold, model):
    want = _json(gold, "keys_json")
    got = {k: list(v.shape) for k, v in model.state_dict().items()}
    assert set(got) == set(want), sorted(set(got) ^ set(want))[:20]
    assert got == want
    for k in ("decoder.geo_fn.index_image", "decoder_view.geo_fn.valid_mask", "decoder.seam_sampler.uvs",
              "upscale_net.out_block.weight_v", "tex_mean", "cal.holder.params", "pixel_cal.bias", "renderer.image_size"):
        assert k in got, k
    assert not any(k.startswith("composer.") for k in got)
    # a state dict with exactly the reference's keys and shapes loads strictly
    sd = {k: torch.zeros(v) for k, v in want.items()}
    sd["renderer.image_size"] = torch.tensor([bf.H, bf.W])
    model.load_state_dict(sd, strict=True)


def test_constructor_buffers_match_reference(gold):
    from goliath_b200.mesh_vae import AutoEncoder

    m = AutoEncoder(**bf.config(), assets=bf.assets())
    for k in ("tex_mean", "meye_mask"):
        t = getattr(m, k)
        assert t.shape == (1, 3 if k == "tex_mean" else 1, 2048, 2048) and t.dtype == torch.float32
        f = t.double().reshape(-1)
        idx = torch.linspace(0, f.numel() - 1, 256, dtype=torch.float64).long()
        got = np.concatenate([[f.mean().item(), f.std().item(), f.abs().max().item(), float(f.numel())], f[idx].numpy()])
        np.testing.assert_allclose(got, gold["buf_" + k], rtol=2e-6, atol=1e-6 * abs(gold["buf_" + k][2]))
    np.testing.assert_array_equal(m.face_cond_mask.numpy(), gold["buf_face_cond_mask"])
    assert m.tex_std == 64.0
    assert m.cal.holder.key_list == sorted(bf.CAMERAS) and m.learn_blur.cameras == bf.CAMERAS
    assert m.cal.identity_idx == sorted(bf.CAMERAS).index(bf.IDENTITY)
    assert m.cal.grey_idxs == [sorted(bf.CAMERAS).index("410244")]
    assert m.pixel_cal.bias.shape == (len(bf.CAMERAS), 1, bf.W // bf.DS, bf.H // bf.DS)


@pytest.mark.parametrize("missing", ["index_image", "face_index_image", "valid_mask"])
def test_missing_uv_images_raise(missing):
    from goliath_b200.mesh_vae import AutoEncoder

    a = bf.assets()
    del a[missing]
    with pytest.raises(ValueError, match=missing):
        AutoEncoder(**bf.config(), assets=a)


def test_unsupported_arguments_raise(model):
    from goliath_b200.mesh_vae import AutoEncoder

    a = bf.assets()
    with pytest.raises(NotImplementedError, match="pose_to_shadow"):
        AutoEncoder(**bf.config(), assets=a, pose_to_shadow={"n_pose_dims": 104, "uv_size": 2048})
    cfg = bf.config()
    cfg["cal"] = None
    with pytest.raises(ValueError, match="pixel_cal needs cal"):
        AutoEncoder(**cfg, assets=a)
    with pytest.raises(ValueError, match="encode=False"):
        model(torch.zeros(1, 12), torch.zeros(1, 3), encode=False)


def test_geometry_module_keys_unchanged_without_the_new_buffers():
    from goliath_b200.geom import GeometryModule

    g = GeometryModule(torch.zeros(4, 3, dtype=torch.int64), torch.zeros(8, 8, 3), torch.zeros(8, 8, 3))
    assert list(g.state_dict()) == ["vi", "index_image", "bary_image"]
