"""CPU checks of the relightable hand teacher's frame (`goliath_b200.hand_teacher.AutoEncoder`): the layout of
tests/golden/hand_teacher_frame_ref.npz, our model's state-dict keys and shapes against the reference's, the
constructor's training state, the [B,L,1] intensity broadcast, and the errors for CPU tensors and `with_shadow`."""
import json
import os

import numpy as np
import pytest
import torch

import hand_frame_restate as hf
import hand_teacher_frame_restate as ht

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hand_teacher_frame_ref.npz")
MARCH_KEYS = ("raypos", "raydir", "tminmax", "primpos", "primrot", "primscale", "template")


@pytest.fixture(scope="module")
def model():
    from goliath_b200.hand_teacher import AutoEncoder

    return AutoEncoder(**hf.config(), assets=hf.assets())


def _keys(z, name):
    return json.loads(bytes(z[name]).decode())


def test_fixture_layout():
    z = np.load(GOLD)
    base = ["primrgb", "valid_prims", "primalpha", "primpos", "primscale", "primrot", "geom_lbs", "primshadow"]
    for mode in ht.MODES:
        train = mode in ht.GRAD_MODES
        want = base + (["texolat"] if train else []) + ["primrgba", "rgb", "alpha", "ae"]
        if mode != "env":
            want.append("learn_blur_weights")
        assert _keys(z, "%s_out_keys_json" % mode) == want, mode
        for k in want:
            if k not in ("valid_prims", "ae"):
                assert "%s_out_%s" % (mode, k) in z and "%s_err32_out_%s" % (mode, k) in z, (mode, k)
        for k in MARCH_KEYS:
            assert "%s_march_%s" % (mode, k) in z, (mode, k)
        for k in ("rgb", "alpha", "primrgba"):
            assert "%s_shadow_%s" % (mode, k) in z, (mode, k)
        names = _keys(z, "grad_names_json")
        post = ["rayrgba", "cal.holder.params", "learn_blur.weights_raw"]
        assert all(("%s_pre_%s" % (mode, n) in z) == train for n in names), mode
        assert all(("%s_post_%s" % (mode, n) in z) == train for n in post), mode
    H, W = hf.H, hf.W
    assert tuple(z["eval_shape_out_rgb"]) == (2, 3, H, W)
    assert tuple(z["env_shape_out_rgb"]) == (2, 3, ht.ENV_H, ht.ENV_W)
    assert tuple(z["train_shape_out_texolat"]) == (2, 1, 8, 3, 1024, 1024)  # the last of two chunks of lights
    assert tuple(z["eval_shape_out_primrgba"]) == (2, 4096, 8, 16, 16, 4)
    assert tuple(z["in_light_intensity"].shape) == (2, ht.L, 3)
    assert tuple(z["env_in_light_intensity"].shape) == (2, 1, 1)
    assert sorted(n.split(".")[0] for n in _keys(z, "grad_names_json")) == sorted(
        ["poseencoder"] * 2 + ["poseencoder2"] * 2 + ["geomdecoder"] * 4 + ["relightdecoder"] * 2)


def test_state_dict_matches_reference(model):
    want = _keys(np.load(GOLD), "keys_json")
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == want
    from goliath_b200.hand_mvp import AutoEncoder as HandAE

    hand = set(HandAE(**hf.config(), assets=hf.assets()).state_dict())
    extra = set(want) - hand
    assert hand <= set(want)
    assert extra and all(k.startswith(("poseencoder2.", "relightdecoder.enc_layers.", "relightdecoder.dec_layers."))
                         for k in extra)


def test_constructor_leaves_geometry_in_eval(model):
    assert model.training and not model.geomdecoder.training
    assert model.relightdecoder.training and model.poseencoder2.training and model.rgbdecoder.training
    assert model.relightdecoder.raymarcher is model.raymarcher and model.relightdecoder.chunksize == 5
    assert model.relightdecoder.pixel_coords.shape == (1024, 1024, 2)


def test_unit_intensity_broadcast():
    from goliath_b200.hand_teacher import _colour_intensity

    one = torch.rand(2, 4, 1)
    out = _colour_intensity(one)
    assert out.shape == (2, 4, 3) and torch.equal(out, one.expand(-1, -1, 3))
    rgb = torch.rand(2, 4, 3)
    assert _colour_intensity(rgb) is rgb


def test_cpu_tensors_are_refused(model):
    z = np.load(GOLD)
    inp = {k: torch.from_numpy(z["in_" + k]) for k in ("pose", "campos", "K", "Rt", "light_pos", "light_intensity")}
    with pytest.raises(RuntimeError, match="CUDA only"):
        model(**inp, camera_id=list(hf.BATCH_CAMERAS))


def test_render_with_shadow_raises(model):
    with pytest.raises(NotImplementedError, match="with_shadow"):
        model.render(torch.eye(3)[None], torch.eye(3, 4)[None], {}, with_shadow=True)
