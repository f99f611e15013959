"""GPU: the UV layout images of goliath_b200.geom (csrc/uv_layout.cu) against the reference's own functions
(tests/golden/uv_images_ref.npz, pytorch3d's rasteriser replaced by this project's restated conventions), against the
restatement and scipy's exact distance transform on a synthetic layout of real-avatar size at 1024^2 and 2048^2, and
the five frames built from a topology and `uv_assets`."""
import json
import os

import numpy as np
import pytest
import torch

import uv_raster_restate as rr
from goliath_b200 import _lib, geom, synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "uv_images_ref.npz")
CASES = [(U, flip) for U in (48, 64) for flip in (False, True)]


@pytest.fixture(scope="module")
def ref():
    return np.load(GOLDEN)


def _np(t):
    return t.detach().cpu().numpy()


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _topo(ref, U):
    return (torch.as_tensor(ref["%d/vt" % U]), torch.as_tensor(ref["%d/vti" % U]), torch.as_tensor(ref["%d/vi" % U]),
            torch.as_tensor(ref["%d/v2uv" % U]))


def _check_impaint(before, after, want, d2_want, src, d2):
    """same destination set as the KDTree's, every source at exactly the KDTree's distance, and the values equal
    wherever the nearest valid texel is unique"""
    valid = (before != -1).any(-1) if before.ndim == 3 else before != -1
    changed = lambda im: ~valid & ((im != -1).any(-1) if im.ndim == 3 else im != -1)
    np.testing.assert_array_equal(changed(after), changed(want))
    np.testing.assert_array_equal(d2, d2_want)
    H, W = valid.shape
    di, dj = np.nonzero(changed(after))
    s = src[di, dj]
    assert (s >= 0).all()
    si, sj = s // W, s % W
    assert valid[si, sj].all()
    np.testing.assert_array_equal((si - di) ** 2 + (sj - dj) ** 2, d2_want[di, dj])
    vi_, vj_ = np.nonzero(valid)
    unique = np.array([((vi_ - a) ** 2 + (vj_ - b) ** 2 == d2_want[a, b]).sum() == 1 for a, b in zip(di, dj)])
    assert unique.any() and (~unique).any()
    np.testing.assert_array_equal(after[di[unique], dj[unique]], want[di[unique], dj[unique]])
    np.testing.assert_array_equal(after[~changed(after)], before[~changed(after)])
    fixed = ~changed(after)
    fixed[di[unique], dj[unique]] = True
    return fixed


# ------------------------------------------------------------------------------------ against the reference
@pytest.mark.gpu
@pytest.mark.parametrize("U,flip", CASES)
def test_images_vs_reference(cuda, ref, U, flip):
    k = "%d/%s/" % (U, "flip" if flip else "noflip")
    vt, vti, vi, _ = _topo(ref, U)
    face = geom.make_uv_face_index(vt, vti, U, flip_uv=flip)
    assert face.dtype == torch.int64 and face.is_cuda
    np.testing.assert_array_equal(_np(face), ref[k + "face"])
    vidx = geom.make_uv_vert_index(vt, vi, vti, U, flip_uv=flip)
    assert vidx.dtype == torch.int64 and vidx.device == vi.device
    np.testing.assert_array_equal(_np(vidx), ref[k + "vert_index"])
    face_b, bary = geom.make_uv_barys(vt, vti, (U, U), flip_uv=flip)
    assert bary.dtype == torch.float32 and bary.device == vt.device
    np.testing.assert_array_equal(_np(face_b), ref[k + "face"])
    assert _bits_equal(_np(bary), ref[k + "bary"])


@pytest.mark.gpu
@pytest.mark.parametrize("U,flip", CASES)
@pytest.mark.parametrize("threshold", (100.0, 7.5))
def test_impaint_vs_kdtree(cuda, ref, U, flip, threshold):
    k = "%d/%s/" % (U, "flip" if flip else "noflip")
    kt = k + "impaint%g/" % threshold
    vidx = ref[k + "vert_index"].astype(np.int64)
    bary = ref[k + "bary"]
    src, d2 = geom._impaint_sources(torch.as_tensor(vidx), threshold, return_d2=True)
    src, d2 = _np(src), _np(d2)
    imp, bimp = geom.index_image_impaint(torch.as_tensor(vidx), torch.as_tensor(bary), threshold)
    assert imp.device.type == "cpu" and imp.dtype == torch.int64
    fixed = _check_impaint(vidx, _np(imp), ref[kt + "index"], ref[k + "d2"], src, d2)
    assert _bits_equal(_np(bimp)[fixed], ref[kt + "bary"][fixed])
    face = ref[k + "face"].astype(np.int64)
    fimp = _np(geom.index_image_impaint(torch.as_tensor(face), distance_threshold=threshold))
    _check_impaint(face, fimp, ref[kt + "face"], ref[k + "d2"], src, d2)


@pytest.mark.gpu
@pytest.mark.parametrize("threshold", (100.0, 7.5))
def test_impaint_far_chart(cuda, ref, threshold):
    """texels farther than the threshold stay invalid, at 100 as at 7.5"""
    face = ref["far/face"].astype(np.int64)
    src, d2 = geom._impaint_sources(torch.as_tensor(face), threshold, return_d2=True)
    out = _np(geom.index_image_impaint(torch.as_tensor(face), distance_threshold=threshold))
    assert (out == -1).any()
    _check_impaint(face, out, ref["far/impaint%g" % threshold], ref["far/d2"], _np(src), _np(d2))


@pytest.mark.gpu
@pytest.mark.parametrize("U,flip", CASES)
def test_geometry_module_vs_reference(cuda, ref, U, flip):
    """from_topology's buffers (impaint=True), render_index_images (the face image un-impainted) and init_primitives
    equal the reference's; where the reference's KDTree picked among equidistant texels, the source lies at its
    distance (checked above), so the comparison is restricted to texels whose value it fixes"""
    from goliath_b200.hand_mvp import init_primitives

    k = "%d/%s/" % (U, "flip" if flip else "noflip")
    vt, vti, vi, v2uv = _topo(ref, U)
    m = geom.GeometryModule.from_topology(vi, vt, vti, v2uv, U, flip_uv=flip, impaint=True)
    sd = m.state_dict()
    assert set(sd) == {"vi", "vt", "vti", "v2uv", "index_image", "bary_image", "face_index_image", "valid_mask"}
    np.testing.assert_array_equal(_np(sd["valid_mask"]), ref[k + "module/valid_mask"])
    # texels whose nearest valid texel is unique: every impainted value is fixed there
    d2 = ref[k + "d2"]
    valid = ref[k + "face"] >= 0
    vi_, vj_ = np.nonzero(valid)
    fixed = valid.copy()
    for a, b in zip(*np.nonzero(~valid)):
        fixed[a, b] = ((vi_ - a) ** 2 + (vj_ - b) ** 2 == d2[a, b]).sum() == 1
    for name in ("index_image", "face_index_image"):
        np.testing.assert_array_equal(_np(sd[name])[fixed], ref[k + "module/" + name][fixed])
    assert _bits_equal(_np(sd["bary_image"])[fixed], ref[k + "module/bary_image"][fixed])
    # the reference's module keys load strictly
    want = {n: torch.as_tensor(ref[k + "module/" + n].astype(np.int64) if ref[k + "module/" + n].dtype == np.int16
                               else ref[k + "module/" + n]) for n in ("index_image", "bary_image", "face_index_image",
                                                                      "valid_mask")}
    want.update(vi=vi, vt=vt, vti=vti, v2uv=v2uv)
    m.load_state_dict(want, strict=True)

    m = geom.GeometryModule.from_topology(vi, vt, vti, v2uv, U, flip_uv=flip)
    ri, rf, rb = m.render_index_images(U, flip_uv=flip, impaint=True)
    np.testing.assert_array_equal(_np(rf), ref[k + "render/face"])
    np.testing.assert_array_equal(_np(ri)[fixed], ref[k + "render/index"][fixed])
    assert _bits_equal(_np(rb)[fixed], ref[k + "render/bary"][fixed])
    if not flip:
        pv, pt, pb = init_primitives(U, 64, m)
        st = U // 8  # init_primitives' stride for 64 primitives
        cells = fixed[st // 2::st, st // 2::st]
        assert cells.any()
        np.testing.assert_array_equal(_np(pv), ref[k + "prims/vidx"])
        np.testing.assert_array_equal(_np(pt), ref[k + "prims/vtidx"])
        assert _bits_equal(_np(pb)[cells], ref[k + "prims/bary"][cells])


@pytest.mark.gpu
def test_float64_vt_is_rounded_to_fp32(cuda, ref):
    """a float64 vt is rounded to fp32 before the raster and the barycentrics; the map comes back in float64"""
    vt, vti, vi, _ = _topo(ref, 64)
    vt64 = vt.double() + 1e-12  # below fp32 resolution at these coordinates: rounds back to vt
    f32, b32 = geom.make_uv_barys(vt, vti, 64)
    f64, b64 = geom.make_uv_barys(vt64, vti, 64)
    assert b64.dtype == torch.float64
    assert torch.equal(f64, f32) and torch.equal(b64, b32.double())


# ------------------------------------------------------------------------------------- at avatar size
@pytest.fixture(scope="module")
def layout():
    return synthetic.uv_layout()


@pytest.mark.gpu
@pytest.mark.parametrize("U", (1024, 2048))
def test_avatar_size(cuda, layout, U):
    import scipy.ndimage as ndi

    vt, vti, vi = layout["vt"], layout["vti"], layout["vi"]
    face, index, bary, valid = geom._index_images(vt, vti, vi, U, False, face=True, vert=True, bary=True, valid=True)
    want = rr.raster(rr.ndc_vertices(vt, False), vti, U)
    np.testing.assert_array_equal(_np(face), _np(want))
    # the large face goes through the CTA-per-face path
    ok, _, i0, i1, j0, j1 = rr.face_boxes(rr.ndc_vertices(vt, False), vti, U)
    assert int(((i1 - i0 + 1) * (j1 - j0 + 1))[ok].max()) > 256 and bool((want == vti.shape[0] - 1).any())
    assert 0.3 < float((want < 0).float().mean()) < 0.7
    assert _bits_equal(_np(bary), _np(rr.barys(vt, vti, want, False)))
    assert torch.equal(valid.cpu(), want >= 0)
    np.testing.assert_array_equal(_np(index), np.where(_np(want)[..., None] >= 0, _np(vi)[_np(want).clip(0)], -1))

    src, d2 = geom._impaint_sources(index, 100.0, return_d2=True)
    src, d2 = _np(src), _np(d2)
    edt = ndi.distance_transform_edt(_np(want) < 0)
    np.testing.assert_array_equal(d2, np.rint(edt ** 2).astype(np.int64))
    far = np.sqrt(d2.astype(np.float64)) >= 100.0
    assert far.any()
    assert ((src >= 0) == (~far & (d2 > 0))).all()
    # the tie rule by brute force: the smallest row-major index among the valid texels at distance sqrt(d2)
    validn = _np(want) >= 0
    rng = np.random.default_rng(3)
    cand = np.flatnonzero((d2 > 0) & ~far)
    for p in rng.choice(cand, 400, replace=False):
        a, b = divmod(int(p), U)
        r = int(np.ceil(np.sqrt(d2[a, b])))
        ii, jj = np.mgrid[max(a - r, 0):min(a + r, U - 1) + 1, max(b - r, 0):min(b + r, U - 1) + 1]
        hit = validn[ii, jj] & ((ii - a) ** 2 + (jj - b) ** 2 == d2[a, b])
        assert hit.any()
        assert src[a, b] == (ii[hit] * U + jj[hit]).min()

    # two calls give the same bits
    m1 = geom.GeometryModule.from_topology(vi, vt, vti, layout["v2uv"], U, impaint=True)
    m2 = geom.GeometryModule.from_topology(vi, vt, vti, layout["v2uv"], U, impaint=True)
    for n, t in m1.state_dict().items():
        assert torch.equal(t, m2.state_dict()[n]), n
    imp = _np(m1.index_image)
    dst = ~validn & ~far
    np.testing.assert_array_equal(imp[dst], _np(index)[src[dst] // U, src[dst] % U])


# ------------------------------------------------------------------------------------------- the frames
def _frame_case(name):
    """(AutoEncoder class, config, assets without their UV images, uv size) of a frame's existing test fixture"""
    if name in ("hand_mvp", "hand_teacher_mvp"):
        import hand_frame_restate as hf

        a, size, cfg = hf.assets(), 1024, hf.config()
        if name == "hand_mvp":
            from goliath_b200.hand_mvp import AutoEncoder
        else:
            from goliath_b200.hand_teacher import AutoEncoder
    elif name == "rgca":
        import head_frame_restate as hr
        from goliath_b200.rgca import AutoEncoder

        a, size, cfg = hr.assets(), hr.SLAB, hr.config()
    elif name == "mesh_vae":
        import body_frame_restate as bf
        from goliath_b200.mesh_vae import AutoEncoder

        a, size, cfg = bf.assets(), 1024, bf.config()
    else:
        import body_drive_restate as bd
        from goliath_b200.mesh_vae_drivable import AutoEncoder

        a, size, cfg = bd.assets(), 1024, bd.config()
    for k in ("index_image", "bary_image", "face_index_image", "valid_mask", "face_index_image_impaint",
              "bary_image_impaint"):
        a.pop(k, None)
    return AutoEncoder, cfg, a, size


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["rgca", "mesh_vae", "mesh_vae_drivable", "hand_mvp", "hand_teacher_mvp"])
def test_frame_builds_from_topology(cuda, name):
    """topology + uv_assets(...) builds the frame; its geo_fn buffers equal from_topology's with the model's flags and
    a reference-keyed geo_fn.* state dict loads strictly"""
    AutoEncoder, cfg, a, size = _frame_case(name)
    with pytest.raises(ValueError):
        AutoEncoder(**cfg, assets=a)
    a.update(geom.uv_assets(a["topology"], name, uv_size=size))
    m = AutoEncoder(**cfg, assets=a)
    flip, impaint, with_v2uv, _ = geom.UV_ASSET_FLAGS[name]
    t = a["topology"]
    want = geom.GeometryModule.from_topology(t["vi"], t["vt"], t["vti"], t["v2uv"] if with_v2uv else None, size,
                                             flip_uv=flip, impaint=impaint)
    got = m.geo_fn.state_dict()
    assert set(got) == set(want.state_dict())
    for n, w in want.state_dict().items():
        assert torch.equal(got[n].cpu(), w.cpu()), n
    m.geo_fn.load_state_dict({n: w.to(torch.int64) if not w.is_floating_point() and w.dtype != torch.bool else w
                              for n, w in want.state_dict().items()}, strict=True)
    if name == "hand_mvp":
        import hand_frame_restate as hf

        z = np.load(os.path.join(os.path.dirname(GOLDEN), "hand_frame_ref.npz"))
        m = hf.seeded_fill(m).to(cuda).eval()
        inp = {k: torch.from_numpy(z["in_" + k]).to(cuda)
               for k in ("pose", "campos", "ambient_occlusion", "K", "Rt", "background")}
        inp["camera_id"] = list(hf.BATCH_CAMERAS)
        with torch.no_grad():
            preds = m(**inp, iteration=5000)
        assert bool(torch.isfinite(preds["rgb"]).all()) and bool(torch.isfinite(preds["alpha"]).all())


# ---------------------------------------------------------------------------------------- launch counts
@pytest.mark.gpu
@pytest.mark.parametrize("F", [0, 1, 300])
def test_launch_count(cuda, tmp_path, F):
    """gb_launch_count's delta equals the kernels torch.profiler records for the new entry points"""
    K = _lib.kernels()
    U = 64
    vt = torch.rand(max(F, 1) * 3, 2, device=cuda)
    vti = torch.arange(max(F, 1) * 3, device=cuda, dtype=torch.int32).reshape(-1, 3)[:F].contiguous()
    vi = vti.clone()
    grid = torch.rand(U, device=cuda)
    ws = torch.zeros(K.gb_uv_raster_workspace_bytes(F, U), dtype=torch.uint8, device=cuda)
    face = torch.zeros(U, U, dtype=torch.int64, device=cuda)
    vidx = torch.zeros(U, U, 3, dtype=torch.int64, device=cuda)
    bary = torch.zeros(U, U, 3, device=cuda)
    valid = torch.zeros(U, U, dtype=torch.bool, device=cuda)
    off, start = geom._offset_table(50, U, U, cuda)
    iws = torch.zeros(K.gb_uv_impaint_workspace_bytes(U, U), dtype=torch.uint8, device=cuda)
    d2 = torch.zeros(U, U, dtype=torch.int32, device=cuda)
    src = torch.zeros(U, U, dtype=torch.int32, device=cuda)
    out = torch.zeros_like(vidx)

    def call():
        K.gb_uv_index_images(F, U, 0, vt, vti, vi, grid, ws, face, vidx, bary, valid)
        K.gb_uv_impaint_sources(U, U, 3, vidx, 50, off, start, iws, d2, src)
        K.gb_uv_impaint_gather(U * U, src, vidx, out, 6, None, None, 0, None, None, 0)

    K_ = _lib.kernels()
    for _ in range(3):  # the profiler can drop an activity record now and then; a miscount repeats every time
        torch.cuda.synchronize()
        before = K_.gb_launch_count()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        delta = K_.gb_launch_count() - before
        trace = tmp_path / "trace.json"
        prof.export_chrome_trace(str(trace))
        kernels = [e["name"] for e in json.loads(trace.read_text())["traceEvents"] if e.get("cat") == "kernel"]
        if delta == len(kernels):
            break
    assert delta == len(kernels) == (4 if F else 2) + 3 + 1, (delta, kernels)
