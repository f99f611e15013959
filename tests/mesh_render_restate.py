"""Torch restatement of the body render's conventions (DESIGN.md R9'', csrc/mesh_raster.cu) for the tests and for
tests/golden/make_mesh_render_golden.py, and the small meshes the tests run on.

  * `raster_bruteforce`: every face against every pixel, in fp64 (or fp32 with the kernel's expression order);
  * `render_at`: depth, perspective-correct barycentrics, vt_img and the grid_sample render at a fixed index image,
    differentiable in v_pix and tex (the interior gradient);
  * `drtk_stub()`: a `drtk` module built from these, with an identity `edge_grad_estimator`."""
import types

import numpy as np
import torch
import torch.nn.functional as F

PIX_OFF = 0.5


def _edge(ax, ay, bx, by, px, py):
    return (bx - ax) * (py - ay) - (by - ay) * (px - ax)


def screen_bary(v, vi, px, py):
    """v [V,3] one item; returns lambda [F,3,...], area [F], z [F,3] for sample points px, py (broadcast)"""
    t = v[vi.long()]                                           # [F,3,3]
    x, y, z = t[..., 0], t[..., 1], t[..., 2]
    sh = (-1,) + (1,) * px.dim()
    xs = [x[:, k].reshape(sh) for k in range(3)]
    ys = [y[:, k].reshape(sh) for k in range(3)]
    area = _edge(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2])
    a = area.reshape(sh)
    l0 = _edge(xs[1], ys[1], xs[2], ys[2], px, py) / a
    l1 = _edge(xs[2], ys[2], xs[0], ys[0], px, py) / a
    l2 = _edge(xs[0], ys[0], xs[1], ys[1], px, py) / a
    return torch.stack([l0, l1, l2], 1), area, z


def raster_bruteforce(v_pix, vi, H, W, dtype=torch.float64):
    """index [B,H,W] int32 and the winning depth [B,H,W]; every face against every pixel"""
    B = v_pix.shape[0]
    yy, xx = torch.meshgrid(torch.arange(H, dtype=dtype), torch.arange(W, dtype=dtype), indexing="ij")
    px, py = xx + PIX_OFF, yy + PIX_OFF
    idx = torch.full((B, H, W), -1, dtype=torch.int32)
    dep = torch.full((B, H, W), float("inf"), dtype=dtype)
    for b in range(B):
        v = v_pix[b].to(dtype)
        lam, area, z = screen_bary(v, vi, px, py)
        ok = (z > 0).all(1) & torch.isfinite(v[vi.long()]).all(2).all(1) & (area != 0) & torch.isfinite(area)
        inside = (lam >= 0).all(1) & ok[:, None, None]
        q = lam / z[:, :, None, None]
        d = 1 / (q[:, 0] + q[:, 1] + q[:, 2])
        d = torch.where(inside, d, torch.full_like(d, float("inf")))
        best, arg = d.min(0)                                   # first (smallest id) of the smallest depth
        idx[b] = torch.where(torch.isfinite(best), arg.to(torch.int32), torch.full_like(arg, -1, dtype=torch.int32))
        dep[b] = best
    return idx, dep


def render_at(v_pix, vi, vti, vt, tex, index_img):
    """differentiable depth [B,H,W], bary [B,3,H,W], vt_img [B,2,H,W], mask [B,1,H,W], render [B,C,H,W]"""
    B, H, W = index_img.shape
    dt = v_pix.dtype
    yy, xx = torch.meshgrid(torch.arange(H, dtype=dt, device=v_pix.device),
                            torch.arange(W, dtype=dt, device=v_pix.device), indexing="ij")
    px, py = (xx + PIX_OFF).reshape(-1), (yy + PIX_OFF).reshape(-1)
    fidx = index_img.reshape(B, -1).long()
    cov = fidx >= 0
    f = fidx.clamp(min=0)
    outs = []
    for b in range(B):
        t = v_pix[b][vi.long()[f[b]]]                          # [P,3 corners,3]
        x, y, z = t[..., 0], t[..., 1], t[..., 2]
        area = _edge(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2])
        area = torch.where(cov[b], area, torch.ones_like(area))
        lam = torch.stack([_edge(x[:, 1], y[:, 1], x[:, 2], y[:, 2], px, py),
                           _edge(x[:, 2], y[:, 2], x[:, 0], y[:, 0], px, py),
                           _edge(x[:, 0], y[:, 0], x[:, 1], y[:, 1], px, py)], 1) / area[:, None]
        lam = torch.where(cov[b][:, None], lam, torch.full_like(lam, 1.0 / 3.0))
        zz = torch.where(cov[b][:, None], z, torch.ones_like(z))
        q = lam / zz
        zi = q.sum(1, keepdim=True)
        bary = q / zi
        uv = (vt * 2.0 - 1.0)[vti.long()[f[b]]]                # [P,3,2]
        vtp = (bary[..., None] * uv).sum(1)
        m = cov[b].to(dt)
        outs.append(((1 / zi[:, 0]) * m, bary * m[:, None], vtp * m[:, None], m))
    depth = torch.stack([o[0] for o in outs]).reshape(B, H, W)
    bary = torch.stack([o[1] for o in outs]).permute(0, 2, 1).reshape(B, 3, H, W)
    vt_img = torch.stack([o[2] for o in outs]).permute(0, 2, 1).reshape(B, 2, H, W)
    mask = torch.stack([o[3] for o in outs]).reshape(B, 1, H, W)
    render = F.grid_sample(tex, vt_img.permute(0, 2, 3, 1), mode="bilinear", align_corners=False) * mask
    return dict(depth_img=depth, bary_img=bary, vt_img=vt_img, mask=mask, render=render)


def drtk_stub():
    """`drtk` as render_drtk.py imports it: transform / rasterize / render / interpolate restating the conventions
    (rasterize decides coverage in fp32 with the kernel's expression order), edge_grad_estimator the identity"""
    m = types.ModuleType("drtk")

    def transform(v, K=None, Rt=None):
        v_cam = torch.einsum("bij,bvj->bvi", Rt[:, :3, :3], v) + Rt[:, None, :3, 3]
        p = torch.einsum("bij,bvj->bvi", K, v_cam)
        return torch.cat([p[..., :2] / v_cam[..., 2:3], v_cam[..., 2:3]], -1)

    def rasterize(v_pix, vi, height, width):
        return raster_bruteforce(v_pix.detach().float(), vi, height, width, torch.float32)[0]

    def render(v_pix, vi, index_img):
        r = render_at(v_pix, vi, vi, torch.zeros(int(vi.max()) + 1, 2, dtype=v_pix.dtype), torch.zeros(
            v_pix.shape[0], 1, 1, 1, dtype=v_pix.dtype), index_img)
        return r["depth_img"], r["bary_img"]

    def interpolate(vert_attributes, vi, index_img, bary_img):
        B, H, W = index_img.shape
        f = index_img.long().clamp(min=0)
        a = torch.stack([vert_attributes[b][vi.long()[f[b]]] for b in range(B)])   # [B,H,W,3,D]
        out = (bary_img.permute(0, 2, 3, 1)[..., None] * a).sum(3)
        return (out * (index_img >= 0)[..., None]).permute(0, 3, 1, 2)

    m.transform, m.rasterize, m.render, m.interpolate = transform, rasterize, render, interpolate
    m.edge_grad_estimator = lambda v_pix, vi, bary_img, img, index_img: img
    return m


# ------------------------------------------------------------------------------------------ meshes


def _mesh(verts, faces, H, W, uv=None, B=1, seed=0):
    v = torch.as_tensor(np.asarray(verts, np.float32))
    if v.dim() == 2:
        v = v[None].expand(B, -1, -1).clone()
    vi = torch.as_tensor(np.asarray(faces), dtype=torch.int32)
    rng = np.random.default_rng(seed)
    vt = torch.as_tensor(rng.uniform(0.05, 0.95, size=(v.shape[1], 2)).astype(np.float32) if uv is None else
                         np.asarray(uv, np.float32))
    return dict(v_pix=v, vi=vi, vti=vi.clone(), vt=vt, H=H, W=W)


def cases():
    """name -> small mesh in pixel space (v_pix [B,V,3], vi, vti, vt, H, W), one per raster edge case"""
    H, W = 24, 32
    c = {}
    # a grid of quads whose vertices lie on pixel sample points: every edge runs through sample points
    g = np.stack(np.meshgrid(np.arange(3, 30, 4) + 0.5, np.arange(2, 23, 4) + 0.5), -1).reshape(-1, 2)
    nx = 7
    z = 2.0 + 0.01 * np.arange(len(g))
    faces = []
    for r in range(5):
        for k in range(nx - 1):
            i = r * nx + k
            faces += [(i, i + 1, i + nx), (i + 1, i + nx + 1, i + nx)] if (r + k) % 2 else [(i, i + nx + 1, i + nx),
                                                                                            (i, i + 1, i + nx + 1)]
    c["on_edges"] = _mesh(np.concatenate([g, z[:, None]], 1), faces, H, W)
    # coplanar duplicates: the same triangle three times (two by index, one by position)
    v = [[4, 3, 5], [28, 5, 5], [10, 21, 5], [4, 3, 5], [28, 5, 5], [10, 21, 5], [2, 2, 9], [30, 2, 9], [16, 23, 9]]
    c["duplicates"] = _mesh(v, [(6, 7, 8), (0, 1, 2), (3, 4, 5), (0, 1, 2)], H, W)
    # z <= 0 (one vertex at 0, one behind), and a face in front of them that is drawn
    v = [[2, 2, 1], [30, 3, 0], [12, 22, 1], [3, 20, 2], [29, 21, -1], [15, 1, 2], [5, 5, 3], [25, 6, 3], [14, 19, 3]]
    c["behind"] = _mesh(v, [(0, 1, 2), (3, 4, 5), (6, 7, 8)], H, W)
    # zero area: collinear and repeated vertices, over a regular face
    v = [[2, 2, 1], [10, 10, 1], [20, 20, 1], [5, 18, 2], [5, 18, 2], [25, 3, 2], [1, 1, 4], [31, 2, 4], [16, 23, 4]]
    c["zero_area"] = _mesh(v, [(0, 1, 2), (3, 4, 5), (6, 7, 8), (0, 0, 1)], H, W)
    # partly and fully off screen
    v = [[-10, -5, 2], [12, 4, 2], [3, 15, 2], [25, 18, 3], [45, 20, 3], [30, 40, 3], [40, 30, 1], [60, 35, 1],
         [50, 50, 1], [-20, 5, 2], [-5, 6, 2], [-12, 20, 2]]
    c["off_screen"] = _mesh(v, [(0, 1, 2), (3, 4, 5), (6, 7, 8), (9, 10, 11)], H, W)
    # a face larger than the image (the CTA-per-face path), under a small one
    v = [[-100, -80, 6], [200, -50, 4], [10, 300, 5], [8, 6, 2], [20, 9, 2], [12, 17, 2]]
    c["huge"] = _mesh(v, [(0, 1, 2), (3, 4, 5)], H, W)
    # UVs outside [0, 1] (zero padding at the texture border)
    v = [[1, 1, 2], [31, 2, 2.5], [2, 23, 3], [30, 22, 2], [31, 2, 2.5], [2, 23, 3]]
    c["uv_out"] = _mesh(v, [(0, 1, 2), (3, 4, 5)], H, W, uv=[[-0.3, -0.2], [1.4, 0.1], [0.2, 1.3], [1.1, 1.2],
                                                           [1.4, 0.1], [0.2, 1.3]])
    return c


def random_mesh(B=2, H=40, W=56, n=60, seed=1):
    """overlapping random triangles of 3-15 px at depths 1-5, two items with different vertex positions, no vertex on
    a sample point (a random sub-pixel offset)"""
    rng = np.random.default_rng(seed)
    ctr = rng.uniform([0, 0], [W, H], size=(n, 2))
    verts = []
    for b in range(B):
        ang = np.arange(3) * 2.1 + rng.uniform(0, 2 * np.pi, size=(n, 1))
        off = rng.uniform(3, 15, size=(n, 3, 1)) * np.stack([np.cos(ang), np.sin(ang)], -1)
        xy = ctr[:, None] + off + rng.uniform(-0.5, 0.5, size=(1, 1, 2)) + 0.137 * b
        z = rng.uniform(1, 5, size=(n, 3))
        verts.append(np.concatenate([xy, z[..., None]], -1).reshape(-1, 3))
    faces = np.arange(3 * n).reshape(n, 3)
    return _mesh(np.stack(verts), faces, H, W, seed=seed)
