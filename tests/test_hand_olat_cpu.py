"""CPU-side checks of the relightable hand teacher's host code (DESIGN.md row R8″) against vectors produced by running
the reference's `OLATRGBDecoder` (tests/golden/hand_olat_ref.npz <- tests/golden/make_hand_olat_golden.py): checkpoint
layout, the light cameras, and the fail-loudly rule."""
import json
import os
import types

import numpy as np
import pytest
import torch

from util import assert_close

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hand_olat_ref.npz")


def _rm(radius):
    return types.SimpleNamespace(dt=1.0 / radius, volume_radius=radius)


def test_state_dict_matches_reference():
    from goliath_b200.hand_teacher import OLATRGBDecoder

    g = np.load(GOLD)
    big = OLATRGBDecoder(1024, (16, 16, 8), 64, 64, _rm(2000.0), 2000.0)
    assert sorted([k, list(v.shape)] for k, v in big.state_dict().items()) == sorted(json.loads(str(g["layout_default"])))
    del big
    small = OLATRGBDecoder(64, (8, 8, 4), 8, 8, _rm(100.0), 100.0, n_init_channels=4, n_enc_dims=[8] * 5,
                           shadow_img_size=48)
    sd = small.state_dict()
    assert sorted(sd) == json.loads(str(g["state_dict"]))
    for k, v in sd.items():
        assert tuple(v.shape) == g["sd_" + k].shape, k
    small.load_state_dict({k: torch.from_numpy(g["sd_" + k]) for k in sd})


def test_light_cameras_match_reference():
    from goliath_b200.hand_teacher import light_cameras

    g = np.load(GOLD)
    d = lambda k: torch.from_numpy(g[k]).double()
    light_pos = d("in_light_pos")
    before = light_pos.clone()
    for c, sl in enumerate((slice(0, 5), slice(5, 7))):
        lpos, lrot, focal, princpt = light_cameras(d("in_primpos"), d("in_valid_prims"), light_pos[:, sl], 48, 48)
        assert_close(lpos.numpy(), g["cam%d_pos" % c], rtol=1e-6, what="light position")
        assert_close(lrot.numpy(), g["cam%d_rot" % c], rtol=1e-5, what="light rotation")
        assert_close(focal.numpy(), g["cam%d_focal" % c], rtol=1e-5, what="focal fit over the valid primitives")
        assert_close(princpt.numpy(), g["cam%d_princpt" % c], rtol=1e-6, what="principal point")
    assert torch.equal(light_pos, before)


def test_build_cam_rot_mat_matches_reference_without_writing_its_input():
    from goliath_b200.hand_teacher import build_cam_rot_mat

    g = np.load(GOLD)
    campos = torch.from_numpy(g["rot_campos"]).double()
    before = campos.clone()
    assert (campos[:, 0].abs() + campos[:, 2].abs() < 1e-8).sum() == 2  # two cameras on the y axis
    center = torch.from_numpy(g["rot_center"]).double()
    assert_close(build_cam_rot_mat(campos, center).numpy(), g["rot_mat"], rtol=1e-5, what="rotation, centred")
    assert_close(build_cam_rot_mat(campos).numpy(), g["rot_mat_origin"], rtol=1e-5, what="rotation, origin")
    assert torch.equal(campos, before)


def test_cpu_tensors_are_refused():
    from goliath_b200.hand_teacher import OLATRGBDecoder, olat_compose

    dec = OLATRGBDecoder(16, (4, 4, 2), 4, 4, _rm(100.0), 100.0, n_init_channels=2, n_enc_dims=[4] * 5,
                         shadow_img_size=8)
    B, L, K = 1, 2, 16
    with pytest.raises(RuntimeError, match="CUDA"):
        dec(torch.zeros(B, 3), None, None, torch.zeros(B, K, 3), torch.eye(3).expand(B, K, 3, 3),
            torch.ones(B, K, 3), torch.zeros(B, 2, 1, 16, 16), torch.ones(K), torch.zeros(B, 2, 1, 1),
            torch.ones(B, L, 3), torch.ones(B, L, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        olat_compose(torch.zeros(B * L, 8, 16, 16), torch.ones(B, L, 3), 2)
