"""CPU: the UV rasteriser's restatement (tests/uv_raster_restate.py) against the reference's own functions run with it
(tests/golden/uv_images_ref.npz), the orientation of the map, and the argument errors of goliath_b200.geom's UV-layout
functions."""
import os

import numpy as np
import pytest
import torch

import uv_raster_restate as rr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "uv_images_ref.npz")


@pytest.fixture(scope="module")
def ref():
    return np.load(GOLDEN)


@pytest.mark.parametrize("U", (48, 64))
@pytest.mark.parametrize("flip", (False, True))
def test_restatement_matches_reference_transforms(ref, U, flip):
    """the NDC vertices the kernel computes (1 - vt, the flip, 2 vt - 1) rasterise to the reference's face image, and
    the restated barycentrics equal the reference's bit for bit"""
    k = "%d/%s/" % (U, "flip" if flip else "noflip")
    vt, vti = torch.as_tensor(ref["%d/vt" % U]), torch.as_tensor(ref["%d/vti" % U])
    face = rr.raster(rr.ndc_vertices(vt, flip), vti, U)
    np.testing.assert_array_equal(face.numpy(), ref[k + "face"])
    bary = rr.barys(vt, vti, face, flip)
    assert np.array_equal(bary.numpy().view(np.int32), ref[k + "bary"].view(np.int32))


def test_fixture_covers_its_cases(ref):
    """the layouts reach what they are meant to: overlaps resolved to the lower id, a skipped zero-area face, texels
    left un-impainted at both thresholds in the far case, and equidistant ties"""
    vt, vti = torch.as_tensor(ref["64/vt"]), torch.as_tensor(ref["64/vti"])
    face = torch.as_tensor(ref["64/noflip/face"].astype(np.int64))
    ids = set(np.unique(ref["64/noflip/face"]).tolist())
    zero_area = vti.shape[0] - 6  # layout(): the collinear face
    assert zero_area not in ids and 0 in ids
    # face 0 lies under the chart: some texel inside both keeps 0
    ok, _, i0, i1, j0, j1 = rr.face_boxes(rr.ndc_vertices(vt, False), vti, 64)
    assert bool(ok[0]) and not bool(ok[zero_area])
    assert (face == 0).sum() > 0 and (face > 0).sum() > 0
    for t in ("100", "7.5"):
        assert (ref["far/impaint%s" % t] == -1).any()
    d2 = ref["64/noflip/d2"]
    i, j = np.nonzero(d2 > 0)
    # a tie: an invalid texel with two valid texels at its distance
    valid = ref["64/noflip/face"] >= 0
    vi_, vj_ = np.nonzero(valid)
    ties = 0
    for a, b in zip(i, j):
        ties += int(((vi_ - a) ** 2 + (vj_ - b) ** 2 == d2[a, b]).sum() > 1)
    assert ties > 0


@pytest.mark.parametrize("flip", (False, True))
def test_orientation_anchor(flip):
    """a triangle at u ~ v ~ 0 lands in row 0, column 0 without the flip and in the last row with it"""
    U = 16
    vt = torch.tensor([[0.0, 0.0], [2.5 / U, 0.0], [0.0, 2.5 / U]])
    face = rr.raster(rr.ndc_vertices(vt, flip), torch.tensor([[0, 1, 2]]), U)
    row = U - 1 if flip else 0
    assert face[row, 0] == 0 and face[U - 1 - row, 0] == -1 and (face >= 0).sum() == 3


def test_edge_and_vertex_centres_are_covered():
    """inclusive test: a texel centre on a vertex and on an edge is covered, for either winding"""
    U = 16
    c = lambda k: (k + 0.5) / U
    vt = torch.tensor([[c(2), c(2)], [c(8), c(2)], [c(2), c(8)]])
    for tri in ([0, 1, 2], [0, 2, 1]):
        face = rr.raster(rr.ndc_vertices(vt, False), torch.tensor([tri]), U)
        assert face[2, 2] == 0 and face[2, 8] == 0 and face[8, 2] == 0 and face[5, 5] == 0 and face[5, 6] == -1


def test_argument_errors():
    from goliath_b200 import geom

    vt, vti = torch.rand(3, 2), torch.tensor([[0, 1, 2]])
    with pytest.raises(ValueError, match="square"):
        geom.make_uv_face_index(vt, vti, (32, 16))
    with pytest.raises(ValueError, match="square"):
        geom.make_uv_barys(vt, vti, (16, 32))
    with pytest.raises(ValueError, match="unknown model"):
        geom.uv_assets({"vi": vti, "vt": vt, "vti": vti}, "urhand")
    with pytest.raises(ValueError, match="no valid texel"):
        geom.index_image_impaint(torch.full((8, 8, 3), -1, dtype=torch.int64))
    with pytest.raises(ValueError, match="no valid texel"):
        geom.index_image_impaint(torch.full((8, 8), -1, dtype=torch.int64))
    with pytest.raises(ValueError, match=r"\[H,W\]"):
        geom.index_image_impaint(torch.zeros(2, 8, 8, 3, dtype=torch.int64))


def test_threshold_and_tie_tables():
    """sqrt(d2) < threshold in double, capped at the image diagonal; offsets grouped by squared length, then (di, dj)"""
    from goliath_b200 import geom

    assert geom._max_d2(7.5, 64, 64) == 56 and geom._max_d2(100.0, 64, 64) == 2 * 63 ** 2
    assert geom._max_d2(100.0, 512, 512) == 9999 and geom._max_d2(10.0, 512, 512) == 99
    assert geom._max_d2(0.0, 8, 8) == -1 and geom._max_d2(float("inf"), 8, 8) == 98
    off, start = geom._offset_table(25, 64, 64, "cpu")
    off, start = off.numpy(), start.numpy()
    d2 = (off ** 2).sum(1)
    assert np.all(np.diff(d2) >= 0) and len(start) == 27 and start[-1] == len(off)
    for d in range(26):
        grp = off[start[d]:start[d + 1]]
        assert np.all((grp ** 2).sum(1) == d)
        assert [tuple(x) for x in grp] == sorted(tuple(x) for x in grp)
    assert [tuple(x) for x in off[start[25]:start[26]]][:3] == [(-5, 0), (-4, -3), (-4, 3)]
