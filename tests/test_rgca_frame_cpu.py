"""CPU checks of the head avatar's frame (`goliath_b200.rgca.AutoEncoder`): its state-dict keys and shapes against the
reference's (tests/golden/head_frame_ref.npz), the construction errors, and SingleLightCycleDecorator's light
positions against the reference's formula (ca_code/utils/light_decorator.py:184-221)."""
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import head_frame_restate as hr  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "head_frame_ref.npz")


def _model(**kw):
    from goliath_b200.rgca import AutoEncoder

    torch.manual_seed(0)
    return AutoEncoder(**{**hr.config(), **kw}, assets=hr.assets())


def test_state_dict_keys_match_reference():
    z = np.load(GOLDEN)
    want = json.loads(z["keys_json"].tobytes().decode())
    sd = _model().state_dict()
    assert {k: list(v.shape) for k, v in sd.items()} == want
    assert not any("v2uv" in k for k in sd)
    # a reference-shaped checkpoint loads with strict=True
    ref_sd = {k: torch.zeros(s) for k, s in want.items()}
    m = _model()
    m.load_state_dict(ref_sd, strict=True)
    assert m.geo_fn is m.decoder.geo_fn


@pytest.mark.parametrize("name", ["index_image", "bary_image", "face_index_image", "valid_mask"])
def test_missing_uv_image_is_named(name):
    from goliath_b200.rgca import AutoEncoder

    with pytest.raises(ValueError, match="missing: %s" % name):
        AutoEncoder(**hr.config(), assets=hr.assets(drop=(name,)))


def test_uv_image_size_follows_slab():
    from goliath_b200.rgca import AutoEncoder

    with pytest.raises(ValueError, match="must be 256 x 256"):
        AutoEncoder(**hr.config(slab=256), assets=hr.assets(slab=128))


def test_n_diff_sh_other_than_8_raises():
    with pytest.raises(ValueError, match="n_diff_sh"):
        _model(n_diff_sh=6)


def test_flags_and_reference_attributes():
    m = _model(cal=None, learn_blur=False)
    assert not m.cal_enabled and not m.learn_blur_enabled
    assert not hasattr(m, "cal") and not hasattr(m, "learn_blur")
    m = _model()
    assert m.cal_enabled and m.learn_blur_enabled
    assert (m.height, m.width, m.n_diff_sh, m.bg_weight) == (hr.H, hr.W, 8, 1.0)


def _reference_light(index, cycle, axis, trans):
    """light_decorator.py:185-208, restated"""
    index = index % cycle
    angle = (abs(index) / cycle) * 2 * np.pi
    if axis == 0:
        p = np.asarray([0.0, 1100.0 * np.sin(angle), 1100.0 * np.cos(angle)]).astype(np.float32)
    elif axis == 1:
        p = np.asarray([-1.0 * 1100.0 * np.sin(angle), 300.0, 1100.0 * np.cos(angle)]).astype(np.float32)
    else:
        p = np.asarray([1100.0 * np.cos(angle), 1100.0 * np.sin(angle), 0.0]).astype(np.float32)
    p = 1100.0 * p / np.linalg.norm(p)
    if trans is not None:
        p += trans
    return p


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("key", ["head_pose", "pose", None])
def test_single_light_cycle_positions(axis, key):
    from goliath_b200.light_decorator import SingleLightCycleDecorator

    seen = {}
    dec = SingleLightCycleDecorator(lambda **d: seen.update(d) or d, cycle=96, light_rotate_axis=axis)
    B = 4
    data = {"campos": torch.zeros(B, 3), "index": [0, 17, 95, 250]}
    trans = np.asarray([[10.0, -20.0, 30.0], [0.5, 0.25, -4.0], [0.0, 0.0, 0.0], [-7.0, 3.0, 1.0]], np.float32)
    if key == "head_pose":
        hp = torch.zeros(B, 3, 4)
        hp[:, :, 3] = torch.from_numpy(trans)
        data["head_pose"] = hp
    elif key == "pose":
        data["pose"] = torch.cat([torch.from_numpy(trans), torch.randn(B, 5)], 1)
    dec(**data)
    want = np.stack([_reference_light(data["index"][i], 96, axis, None if key is None else trans[i])
                     for i in range(B)])
    assert seen["light_pos"].shape == (B, 1, 3) and seen["light_pos"].dtype == torch.float32
    np.testing.assert_array_equal(seen["light_pos"][:, 0].numpy(), want)
    assert seen["light_intensity"].shape == (B, 1, 1) and bool((seen["light_intensity"] == 1).all())
    assert seen["n_lights"].dtype == torch.int32 and seen["n_lights"].tolist() == [1] * B
    assert seen["is_fullylit_frame"].shape == (1,)
