"""A torch restatement (CPU, fp32, one rounding per operation) of this project's UV-layout conventions
(csrc/uv_layout.cu, DESIGN.md R12).  pytorch3d's rasterize_meshes, which the reference's make_uv_face_index calls, is a
third-party package; tests/golden/make_uv_images_golden.py puts `raster` in its place, and the GPU tests compare the
kernels with these functions bit for bit.

  * texel (i, j) samples the NDC point (x_j, y_i), x_k = y_k = 1 - (2 k + 1) / U;
  * a face with |e(v0, v1, v2)| <= 1e-8 is skipped, e(a, b, p) = (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x);
  * a texel is inside when the three edge functions are all >= 0 (positive area) or all <= 0 (negative area);
  * a texel covered by several faces takes the lowest face id (all faces lie at z = 1).

Each face is tested over its texel box (one texel of margin around its NDC bounding box, clipped to the image), the
same box the kernel walks, so the restatement stays affordable at 2048^2."""
import torch

ZERO_AREA = torch.tensor(1e-8, dtype=torch.float32)
_INT_MAX = 2 ** 31 - 1


def ndc_vertices(vt, flip_uv):
    """the kernel's NDC vertices of vt [N,2]: x = 2 (1 - u) - 1, y = 2 (1 - v) - 1 (flip: 2 (1 - (1 - v)) - 1)"""
    vt = torch.as_tensor(vt, dtype=torch.float32)
    a = 1.0 - vt[:, 0]
    b = 1.0 - vt[:, 1]
    if flip_uv:
        b = 1.0 - b
    return torch.stack([2.0 * a - 1.0, 2.0 * b - 1.0], dim=1)


def pix_ndc(U):
    """x_k = 1 - (2 k + 1) / U in fp32"""
    return 1.0 - (2 * torch.arange(U) + 1).to(torch.float32) / float(U)


def _edge(ax, ay, bx, by, px, py):
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def face_boxes(ndc, faces, U):
    """(ok [F] bool, area [F], i0, i1, j0, j1 [F] int64) as the kernel's face_box computes them"""
    t = ndc[faces.long()]
    x, y = t[..., 0], t[..., 1]
    area = _edge(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2])
    ok = (area.abs() > ZERO_AREA) & torch.isfinite(area)
    Uf = float(U)
    xmin, xmax = torch.minimum(torch.minimum(x[:, 0], x[:, 1]), x[:, 2]), torch.maximum(torch.maximum(x[:, 0], x[:, 1]), x[:, 2])
    ymin, ymax = torch.minimum(torch.minimum(y[:, 0], y[:, 1]), y[:, 2]), torch.maximum(torch.maximum(y[:, 0], y[:, 1]), y[:, 2])
    j0 = torch.clamp(torch.ceil(((1.0 - xmax) * Uf - 1.0) * 0.5) - 1.0, min=0.0)
    j1 = torch.clamp(torch.floor(((1.0 - xmin) * Uf - 1.0) * 0.5) + 1.0, max=Uf - 1.0)
    i0 = torch.clamp(torch.ceil(((1.0 - ymax) * Uf - 1.0) * 0.5) - 1.0, min=0.0)
    i1 = torch.clamp(torch.floor(((1.0 - ymin) * Uf - 1.0) * 0.5) + 1.0, max=Uf - 1.0)
    ok &= (j0 <= j1) & (i0 <= i1)
    return ok, area, i0.long(), i1.long(), j0.long(), j1.long()


def raster(ndc, faces, U, chunk=1 << 22):
    """face image [U,U] int64 (-1 uncovered) of the NDC triangles ndc[faces] ([N,2] or [N,3] fp32, [F,3])"""
    ndc = torch.as_tensor(ndc, dtype=torch.float32)[:, :2].contiguous()
    faces = torch.as_tensor(faces).long()
    ok, area, i0, i1, j0, j1 = face_boxes(ndc, faces, U)
    P = pix_ndc(U)
    img = torch.full((U * U,), _INT_MAX, dtype=torch.int64)
    fid = torch.nonzero(ok)[:, 0]
    if fid.numel() == 0:
        return torch.full((U, U), -1, dtype=torch.int64)
    bh, bw = (i1 - i0 + 1)[fid], (j1 - j0 + 1)[fid]
    # group the faces by their box rounded up to powers of two, and test each group's padded boxes at once
    ph = 2 ** torch.ceil(torch.log2(bh.double())).long()
    pw = 2 ** torch.ceil(torch.log2(bw.double())).long()
    for h, w in sorted(set(zip(ph.tolist(), pw.tolist()))):
        grp = fid[(ph == h) & (pw == w)]
        step = max(1, chunk // (h * w))
        for s in range(0, grp.numel(), step):
            f = grp[s:s + step]
            di, dj = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
            i = i0[f, None] + di.reshape(1, -1)
            j = j0[f, None] + dj.reshape(1, -1)
            keep = (i <= i1[f, None]) & (j <= j1[f, None])
            tri = ndc[faces[f]]
            x = [tri[:, k, 0:1] for k in range(3)]
            y = [tri[:, k, 1:2] for k in range(3)]
            px, py = P[j.clamp(max=U - 1)], P[i.clamp(max=U - 1)]
            w0 = _edge(x[1], y[1], x[2], y[2], px, py)
            w1 = _edge(x[2], y[2], x[0], y[0], px, py)
            w2 = _edge(x[0], y[0], x[1], y[1], px, py)
            pos = area[f, None] > 0
            inside = torch.where(pos, (w0 >= 0) & (w1 >= 0) & (w2 >= 0), (w0 <= 0) & (w1 <= 0) & (w2 <= 0)) & keep
            t = (i * U + j)[inside]
            img.scatter_reduce_(0, t, f[:, None].expand_as(i)[inside], "amin")
    img[img == _INT_MAX] = -1
    return img.view(U, U)


def uv_grid(U):
    """the reference's sample grid (geom.py:133-136), built with the same torch call"""
    return torch.linspace(0.5, U - 0.5, U) / U


def barys(vt, vti, face, flip_uv):
    """bary_coords (geom.py:86-106, with its +-1e-6 clamp) of the texel centres (g[j], g[i]) in the UV triangle of
    face [U,U] (vt with its v flipped when flip_uv), fp32, zero where face < 0"""
    vt = torch.as_tensor(vt, dtype=torch.float32).clone()
    if flip_uv:
        vt[:, 1] = 1 - vt[:, 1]
    U = face.shape[0]
    g = uv_grid(U)
    tri = vt[torch.as_tensor(vti).long()[face.clamp(min=0)]]  # [U,U,3,2]
    px, py = g[None, :].expand(U, U), g[:, None].expand(U, U)
    x, x1, x2 = px - tri[..., 2, 0], tri[..., 0, 0] - tri[..., 2, 0], tri[..., 1, 0] - tri[..., 2, 0]
    y, y1, y2 = py - tri[..., 2, 1], tri[..., 0, 1] - tri[..., 2, 1], tri[..., 1, 1] - tri[..., 2, 1]
    denom = y2 * x1 - y1 * x2
    n0 = y2 * x - x2 * y
    n1 = x1 * y - y1 * x
    denom = torch.where(denom >= 0, denom.clamp(min=1e-6), denom.clamp(max=-1e-6))
    b0, b1 = n0 / denom, n1 / denom
    out = torch.stack([b0, b1, 1.0 - b0 - b1], dim=-1)
    out[face < 0] = 0
    return out
