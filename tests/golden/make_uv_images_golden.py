"""Generate tests/golden/uv_images_ref.npz by RUNNING the reference's own UV-layout functions on CPU
(ca_code/utils/geom.py: make_uv_face_index, make_uv_vert_index, bary_coords, make_uv_barys, index_image_impaint,
GeometryModule.__init__ / render_index_images, imported) and `init_primitives` (sliced out of
ca_code/models/hand_mvp.py by AST), with two substitutions:

  * the `th.device("cuda")` default of make_uv_face_index is redirected to the CPU;
  * pytorch3d's Meshes / rasterize_meshes are replaced by tests/uv_raster_restate.raster, this project's rasteriser
    conventions restated in fp32 (pytorch3d is third-party: DESIGN.md R12, parity unpinned).

Everything else is the reference's: `1 - vt`, the flip, `2 vt - 1`, the sample grid, the barycentric formula and the
impaint, whose KDTree is sklearn's own; its distances are stored beside its choices.

Layouts (tests/golden/make_uv_images_golden.layout) at U = 48 and 64, flip_uv both ways: a chart of quads whose
corners sit on texel centres (texel centres exactly on edges and vertices), split with both windings; a large face
overlapping the chart with a lower id and random faces overlapping it with higher ids; a zero-area face; a face with
vt outside [0, 1]; a small far chart; a triangle at u ~ v ~ 0.  An impaint-only case at U = 160 keeps the valid
texels in one corner, so thresholds 100 and 7.5 both leave texels un-impainted.

Needs /root/reference and sklearn; the .npz is committed.   Usage: python tests/golden/make_uv_images_golden.py
"""
import ast
import os
import sys
import types
import warnings

import numpy as np
import torch as th

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "uv_images_ref.npz")
SRC_HAND = "/root/reference/ca_code/models/hand_mvp.py"
SIZES = (48, 64)
THRESHOLDS = (100.0, 7.5)
FAR_U = 160


def layout(U, seed=0):
    """(vt [N,2] fp32, vti [F,3] int64, vi [F,3] int64, v2uv [V,2] int64) of the test layout at size U"""
    rng = np.random.default_rng(seed + U)
    c = lambda k: (k + 0.5) / U  # a texel centre
    vt, faces = [], []

    def add(*uv):
        vt.extend(uv)
        return list(range(len(vt) - len(uv), len(vt)))

    # a large face under the chart, with the lowest id: it wins wherever it overlaps
    faces.append(add((c(6), c(6)), (c(20), c(8)), (c(9), c(22))))
    # the chart: 4 x 4 quads of 3 x 3 texels, corners on texel centres, split with alternating windings
    g = np.array(add(*[(c(4 + 3 * a), c(5 + 3 * b)) for a in range(5) for b in range(5)])).reshape(5, 5)
    for a in range(4):
        for b in range(4):
            v00, v10, v01, v11 = g[a, b], g[a + 1, b], g[a, b + 1], g[a + 1, b + 1]
            if (a + b) % 2:
                faces += [[v00, v10, v11], [v00, v11, v01]]
            else:
                faces += [[v00, v11, v10], [v00, v01, v11]]
    # random faces overlapping the chart (higher ids)
    for _ in range(6):
        p = rng.uniform(c(3), c(18), size=(3, 2))
        faces.append(add(*map(tuple, p)))
    # a zero-area face (collinear corners on texel centres)
    faces.append(add((c(30), c(30)), (c(33), c(33)), (c(36), c(36))))
    # a face reaching outside [0, 1]
    faces.append(add((-0.2, 0.9), (0.2, 1.3), (0.15, 0.75)))
    # a second chart to the right, with both windings
    h = add((c(U - 14), c(10)), (c(U - 4), c(12)), (c(U - 9), c(20)), (c(U - 3), c(24)))
    faces += [[h[0], h[1], h[2]], [h[1], h[3], h[2]]]
    # a small far chart
    faces.append(add((c(U - 6), c(U - 5)), (c(U - 3), c(U - 5)), (c(U - 5), c(U - 2))))
    # the orientation anchor at u ~ v ~ 0
    faces.append(add((0.0, 0.0), (2.5 / U, 0.0), (0.0, 2.5 / U)))
    vt = np.asarray(vt, np.float32)
    vti = np.asarray(faces, np.int64)
    V = len(vt) // 2 + 3
    vi = (vti * 7 + 3) % V
    v2uv = np.stack([np.arange(V), np.arange(V)[::-1]], axis=1).astype(np.int64) % len(vt)
    return vt, vti, vi, v2uv


def far_layout(U=FAR_U):
    """one small chart in the top-left corner of a U x U map"""
    vt = np.asarray([[1.5 / U, 1.5 / U], [9.5 / U, 2.5 / U], [3.5 / U, 8.5 / U]], np.float32)
    vti = np.asarray([[0, 1, 2]], np.int64)
    return vt, vti, vti.copy(), np.asarray([[0, 1], [1, 2], [2, 0]], np.int64)


def _reference():
    sys.path.insert(0, "/root/reference")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, HERE)
    from make_lbs_golden import _stub

    _stub()
    import ca_code.utils.geom as geom
    import uv_raster_restate as rr

    class Meshes:
        def __init__(self, verts, faces):
            self.verts, self.faces = verts, faces

    def rasterize_meshes(meshes, image_size, faces_per_pixel=1, z_clip_value=None, bin_size=None, **kw):
        assert faces_per_pixel == 1 and bin_size == 0 and image_size[0] == image_size[1]
        assert bool((meshes.verts[0][:, 2] == 1).all())
        face = rr.raster(meshes.verts[0], meshes.faces[0], image_size[0])
        return face[None, ..., None], None, None, None

    shim = types.ModuleType("th_cpu")
    shim.__dict__.update({k: getattr(th, k) for k in dir(th) if not k.startswith("__")})
    shim.device = lambda *a, **k: th.device("cpu")
    geom.th, geom.Meshes, geom.rasterize_meshes = shim, Meshes, rasterize_meshes
    ns = {"th": th}
    src = open(SRC_HAND).read()
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name == "init_primitives":
            exec(ast.get_source_segment(src, node), ns)
    return geom, ns["init_primitives"]


def _kdtree(index_image):
    """sklearn's KDTree query of index_image_impaint, for the distances: d2 [H,W] int32 (0 at valid texels)"""
    from sklearn.neighbors import KDTree

    valid = (index_image != -1).any(dim=-1) if index_image.dim() == 3 else index_image != -1
    vij, iij = th.stack(th.where(valid), -1), th.stack(th.where(~valid), -1)
    d, _ = KDTree(vij.numpy()).query(iij.numpy())
    d2 = np.zeros(valid.shape, np.int32)
    d2[iij[:, 0].numpy(), iij[:, 1].numpy()] = np.rint(d[:, 0] ** 2).astype(np.int32)
    assert np.array_equal(np.sqrt(d2[~valid.numpy()].astype(np.float64)), d[:, 0])
    return d2


def main():
    if not os.path.isdir("/root/reference/ca_code"):
        sys.exit("needs /root/reference (build container only)")
    warnings.filterwarnings("ignore")
    geom, init_primitives = _reference()
    out = {}
    i16 = lambda t: t.numpy().astype(np.int16)
    for U in SIZES:
        vt, vti, vi, v2uv = layout(U)
        out["%d/vt" % U], out["%d/vti" % U], out["%d/vi" % U], out["%d/v2uv" % U] = vt, vti, vi, v2uv
        vt_t, vti_t, vi_t = th.as_tensor(vt), th.as_tensor(vti), th.as_tensor(vi)
        for flip in (False, True):
            k = "%d/%s/" % (U, "flip" if flip else "noflip")
            face = geom.make_uv_face_index(vt_t, vti_t, U, flip_uv=flip)
            vidx = geom.make_uv_vert_index(vt_t, vi_t, vti_t, U, flip_uv=flip)
            face_b, bary = geom.make_uv_barys(vt_t, vti_t, U, flip_uv=flip)
            assert th.equal(face, face_b)
            out[k + "face"], out[k + "vert_index"], out[k + "bary"] = i16(face), i16(vidx), bary.numpy()
            out[k + "d2"] = _kdtree(vidx)
            for t in THRESHOLDS:
                imp, bimp = geom.index_image_impaint(vidx, bary, t)
                fimp = geom.index_image_impaint(face, distance_threshold=t)
                out[k + "impaint%g/index" % t], out[k + "impaint%g/bary" % t] = i16(imp), bimp.numpy()
                out[k + "impaint%g/face" % t] = i16(fimp)
            m = geom.GeometryModule(vi_t, vt_t, vti_t, th.as_tensor(v2uv), U, flip_uv=flip, impaint=True)
            for name, buf in m.state_dict().items():
                if name not in ("vi", "vt", "vti", "v2uv"):
                    out[k + "module/" + name] = buf.numpy().astype(np.int16) if buf.dtype == th.int64 else buf.numpy()
            ri, rf, rb = m.render_index_images(U, flip_uv=flip, impaint=True)
            out[k + "render/index"], out[k + "render/face"], out[k + "render/bary"] = i16(ri), i16(rf), rb.numpy()
            if not flip:
                pv, pt, pb = init_primitives(U, 64, m)
                out[k + "prims/vidx"], out[k + "prims/vtidx"], out[k + "prims/bary"] = i16(pv), i16(pt), pb.numpy()
    vt, vti, vi, _ = far_layout()
    out["far/vt"], out["far/vti"] = vt, vti
    face = geom.make_uv_face_index(th.as_tensor(vt), th.as_tensor(vti), FAR_U, flip_uv=False)
    out["far/face"], out["far/d2"] = i16(face), _kdtree(face)
    for t in THRESHOLDS:
        out["far/impaint%g" % t] = i16(geom.index_image_impaint(face, distance_threshold=t))
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d bytes)" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
