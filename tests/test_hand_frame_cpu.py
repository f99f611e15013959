"""CPU checks of the hand avatar's frame (`goliath_b200.hand_mvp.AutoEncoder`): construction from the synthetic assets,
the reference's state-dict keys and shapes (tests/golden/hand_frame_ref.npz, the reference's own AutoEncoder), a
strict load of a reference-shaped dict, the error for a missing UV image, and the valid-primitive buffer with its
slot table and count."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import hand_frame_restate as hf

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hand_frame_ref.npz")


@pytest.fixture(scope="module")
def model():
    from goliath_b200.hand_mvp import AutoEncoder

    return AutoEncoder(**hf.config(), assets=hf.assets())


def test_state_dict_matches_reference(model):
    want = json.loads(bytes(np.load(GOLD)["keys_json"]).decode())
    got = {k: list(v.shape) for k, v in model.state_dict().items()}
    assert got == want
    # the shared modules repeat under the decoders, as in the reference
    assert model.geomdecoder.geo_fn is model.geo_fn and model.rgbdecoder.geo_fn is model.geo_fn
    assert model.geomdecoder.lbs_fn is model.lbs_fn
    assert model.raymarcher.dt == 1.0 / 2000.0 and model.raymarcher.volume_radius == 2000.0
    assert model.renderer.image_size.tolist() == [hf.H, hf.W]


def test_reference_shaped_dict_loads_strictly(model):
    want = json.loads(bytes(np.load(GOLD)["keys_json"]).decode())
    own = model.state_dict()
    g = torch.Generator().manual_seed(3)
    sd = {k: (torch.randn(shape, generator=g) if own[k].is_floating_point() else own[k].clone())
          for k, shape in want.items()}
    res = model.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    k = "geomdecoder.transdecoder.dec0.0.weight_v"
    assert torch.equal(model.state_dict()[k], sd[k])


@pytest.mark.parametrize("name", ["face_index_image_impaint", "bary_image_impaint", "valid_mask"])
def test_missing_uv_image_is_named(name):
    from goliath_b200.hand_mvp import AutoEncoder

    a = hf.assets()
    del a[name]
    with pytest.raises(ValueError, match=name):
        AutoEncoder(**hf.config(), assets=a)


def test_valid_prims_slot_table_and_count():
    """isolated valid texels at the four corners of cells: area interpolation to 64 x 64 marks exactly those cells"""
    from goliath_b200.hand_mvp import AutoEncoder

    a = hf.assets()
    mask = np.zeros((1024, 1024, 1), bool)
    cells = {(0, 0): (0, 0), (3, 5): (15, 15), (10, 20): (0, 15), (40, 2): (15, 0), (63, 63): (15, 15)}
    for (cy, cx), (oy, ox) in cells.items():
        mask[16 * cy + oy, 16 * cx + ox] = True
    a["valid_mask"] = torch.as_tensor(mask)
    m = AutoEncoder(**hf.config(), assets=a)
    rule = (F.interpolate(torch.as_tensor(mask).float()[None].permute(0, 3, 1, 2), (64, 64), mode="area") != 0)
    rule = rule.reshape(-1)
    want = torch.zeros(64 * 64, dtype=torch.bool)
    want[[64 * cy + cx for cy, cx in cells]] = True
    assert torch.equal(rule, want) and torch.equal(m.valid_prims, want)
    slot = torch.full((64 * 64,), -1, dtype=torch.int32)
    slot[sorted(64 * cy + cx for cy, cx in cells)] = torch.arange(len(cells), dtype=torch.int32)
    assert m.valid_slot.dtype == torch.int32 and torch.equal(m.valid_slot, slot)
    assert m.n_valid == len(cells)
    assert "valid_prims" not in m.state_dict() and "valid_slot" not in m.state_dict()


def test_fixture_model_valid_prims(model):
    """the synthetic tube covers part of the UV square: some primitives are invalid, most are valid"""
    z = np.load(GOLD)
    assert torch.equal(model.valid_prims, torch.as_tensor(z["valid_prims"]))
    assert 0 < model.n_valid < 4096 and model.n_valid == int(model.valid_prims.sum())
