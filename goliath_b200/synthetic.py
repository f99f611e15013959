"""Seeded synthetic inputs for the RGCA splat / shade path (recipe: SURVEY.md §8d, BASELINE.md §2).

Generated on the CPU with a fixed torch.Generator so every rank / device / test sees identical bytes.
"""
import math
from typing import Dict

import torch

SEED = 20240613


def ring_camera(k: int, n_ring: int = 16, radius: float = 1000.0, img_h: int = 1024, img_w: int = 667) -> Dict:
    """Camera k on a ring around the origin, looking at it.  Returns viewmat [3,4] (world->camera, row-major)
    and pinhole intrinsics (fx = fy = 3300 * W / 1334)."""
    yaw = 2.0 * math.pi * k / n_ring
    cam = torch.tensor([radius * math.sin(yaw), 0.0, radius * math.cos(yaw)], dtype=torch.float64)
    z = -cam / cam.norm()                       # camera looks at the origin
    up = torch.tensor([0.0, -1.0, 0.0], dtype=torch.float64)   # image y points down
    x = torch.linalg.cross(up, z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    R = torch.stack([x, y, z])                  # rows = camera axes in world space
    t = -R @ cam
    viewmat = torch.cat([R, t[:, None]], 1).to(torch.float32).contiguous()
    f = 3300.0 * (img_w / 1334.0)
    return dict(viewmat=viewmat, fx=f, fy=f, cx=img_w / 2.0, cy=img_h / 2.0, img_h=img_h, img_w=img_w,
                campos=cam.to(torch.float32))


def head_gaussians(G: int = 300_000, seed: int = SEED) -> Dict[str, torch.Tensor]:
    """Ellipsoid-shell Gaussians: radii (90,120,100) mm * (1 + 0.05 N), unit quats (w,x,y,z),
    scales = clamp(softplus(N(0.5,0.7)), 0.1, 20) mm, opacity = sigmoid(N(1,2)), colors ~ U(0,1)."""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(G, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    rad = torch.tensor([90.0, 120.0, 100.0]) * (1.0 + 0.05 * torch.randn(G, 1, generator=g))
    means = (d * rad).contiguous()
    q = torch.randn(G, 4, generator=g)
    quats = (q / q.norm(dim=-1, keepdim=True)).contiguous()
    scales = torch.nn.functional.softplus(0.5 + 0.7 * torch.randn(G, 3, generator=g)).clamp(0.1, 20.0).contiguous()
    opacity = torch.sigmoid(1.0 + 2.0 * torch.randn(G, 1, generator=g)).contiguous()
    colors = torch.rand(G, 3, generator=g).contiguous()
    return dict(means3d=means, quats=quats, scales=scales, opacity=opacity, colors=colors)


def lights(L: int = 32, radius: float = 1100.0, seed: int = SEED + 1) -> Dict[str, torch.Tensor]:
    """L point lights on a Fibonacci lattice, grey intensity ~ U(0.5, 1.5) expanded to 3 channels."""
    g = torch.Generator().manual_seed(seed)
    i = torch.arange(L, dtype=torch.float64) + 0.5
    phi = torch.acos(1.0 - 2.0 * i / L)
    theta = math.pi * (1.0 + 5.0 ** 0.5) * i
    pos = radius * torch.stack([torch.cos(theta) * torch.sin(phi), torch.sin(theta) * torch.sin(phi), torch.cos(phi)], -1)
    inten = (0.5 + torch.rand(L, 1, generator=g)).expand(L, 3)
    return dict(light_pos=pos.to(torch.float32)[None].contiguous(), light_intensity=inten[None].contiguous(),
                n_lights=torch.tensor([L], dtype=torch.int32))


def shade_inputs(G: int, seed: int = SEED + 2) -> Dict[str, torch.Tensor]:
    """SG lobes: un-normalised lobe_dirs ~ N(0,I), sigma = clamp(0.1 exp(N(0,0.5)), 0.01)."""
    g = torch.Generator().manual_seed(seed)
    lobe_dirs = torch.randn(1, G, 3, generator=g).contiguous()
    sigma = (0.1 * torch.exp(0.5 * torch.randn(1, G, generator=g))).clamp(min=0.01).contiguous()
    return dict(lobe_dirs=lobe_dirs, lobe_sigmas=sigma)


def mvp_scene(N: int = 2, side: int = 8, T=(4, 8, 8), img_h: int = 64, img_w: int = 48, seed: int = SEED + 7,
              density: float = 40.0, with_warp: bool = False) -> Dict:
    """Hand-MVP-like synthetic scene (SURVEY.md §8d config 4 recipe, scaled): K = side*side primitives on a UV grid
    wrapped on a cylinder (normalised unit-cube coordinates, volradius = 1), small random rotations, template =
    softplus(1.5 N(0,1)) with the alpha channel shifted, N ring cameras.  Returns CPU tensors + camera parameters."""
    g = torch.Generator().manual_seed(seed)
    K = side * side
    u = (torch.arange(side, dtype=torch.float32) + 0.5) / side
    uu, vv = torch.meshgrid(u, u, indexing="ij")          # uu: around the axis, vv: along it
    ang = 2 * math.pi * uu.reshape(-1)
    rad, height = 0.28, 0.9
    pos = torch.stack([rad * torch.cos(ang), (vv.reshape(-1) - 0.5) * height, rad * torch.sin(ang)], -1)
    pos = pos + 0.01 * torch.randn(K, 3, generator=g)
    normal = torch.stack([torch.cos(ang), torch.zeros(K), torch.sin(ang)], -1)
    tangent = torch.stack([-torch.sin(ang), torch.zeros(K), torch.cos(ang)], -1)
    up = torch.tensor([0.0, 1.0, 0.0]).expand(K, 3)
    R = torch.stack([tangent, up, normal], -1)            # columns = local axes in world space
    # small random rotation
    w = 0.15 * torch.randn(K, 3, generator=g)
    th = w.norm(dim=-1, keepdim=True).clamp(min=1e-8)
    kx = w / th
    Kx = torch.zeros(K, 3, 3)
    Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 0] = -kx[:, 2], kx[:, 1], kx[:, 2]
    Kx[:, 1, 2], Kx[:, 2, 0], Kx[:, 2, 1] = -kx[:, 0], -kx[:, 1], kx[:, 0]
    Rr = torch.eye(3) + torch.sin(th)[..., None] * Kx + (1 - torch.cos(th))[..., None] * (Kx @ Kx)
    R = Rr @ R
    half = torch.tensor([1.3 * math.pi * rad / side, 0.65 * height / side, 0.04])
    primscale = (1.0 / half).expand(K, 3)
    TD, TH, TW = T
    tpl = torch.nn.functional.softplus(1.5 * torch.randn(N, K, TD, TH, TW, 4, generator=g))
    tpl[..., 3] = torch.nn.functional.softplus(1.5 * torch.randn(N, K, TD, TH, TW, generator=g) - 1.0) * density
    out = dict(primpos=pos[None].repeat(N, 1, 1).contiguous(), primrot=R[None].repeat(N, 1, 1, 1).contiguous(),
               primscale=primscale[None].repeat(N, 1, 1).contiguous(), template=tpl.contiguous())
    if with_warp:
        lin = [torch.linspace(-1, 1, s) for s in (TD, TH, TW)]
        zz, yy, xx = torch.meshgrid(*lin, indexing="ij")
        grid = torch.stack([xx, yy, zz], -1)               # channels-last identity warp, (x, y, z)
        out["warp"] = (grid[None, None] + 0.05 * torch.randn(N, K, TD, TH, TW, 3, generator=g)).contiguous()
    # cameras on a ring of radius 2.5 (normalised units) looking at the origin
    viewpos, viewrot = [], []
    for n in range(N):
        c = ring_camera(n * 3 + 1, radius=2.5, img_h=img_h, img_w=img_w)
        viewpos.append(c["campos"])
        viewrot.append(c["viewmat"][:, :3])                # rows = camera axes in world space
    f = 1.6 * min(img_h, img_w)
    out.update(viewpos=torch.stack(viewpos).contiguous(), viewrot=torch.stack(viewrot).contiguous(),
               focal=torch.full((N, 2), f), princpt=torch.tensor([[img_w / 2.0, img_h / 2.0]] * N),
               img_h=img_h, img_w=img_w, volradius=1.0)
    return out


def body_mesh(n_faces: int, img_h: int = 2048, img_w: int = 1334, batch: int = 4, seed: int = SEED) -> Dict:
    """A closed multi-part stand-in for the body template (its face count is not known here): 8 lat-long
    ellipsoids over a 1.8 m tall box, about n_faces faces in all, UVs per vertex; and `batch` cameras 2.3-2.7 m in
    front of it with the configuration's image size (fx = fy = 2000 * H / 2048).  Returns float32 verts [V,3],
    int32 vi / vti [F,3], vt [V,2], K [B,3,3] and Rt [B,3,4]."""
    g = torch.Generator().manual_seed(seed)
    parts = 8
    per = max(n_faces // parts, 8)
    nlon = max(int(math.sqrt(per)), 4)
    nlat = max(per // (2 * nlon) + 1, 3)
    verts, vi, vt = [], [], []
    for k in range(parts):
        lat = torch.linspace(0, math.pi, nlat + 1, dtype=torch.float64)[1:-1]
        lon = torch.arange(nlon, dtype=torch.float64) * (2 * math.pi / nlon)
        ring = torch.stack([torch.sin(lat)[:, None] * torch.cos(lon), torch.cos(lat)[:, None].expand(-1, nlon),
                            torch.sin(lat)[:, None] * torch.sin(lon)], -1).reshape(-1, 3)
        pts = torch.cat([torch.tensor([[0.0, 1.0, 0.0]], dtype=torch.float64), ring,
                         torch.tensor([[0.0, -1.0, 0.0]], dtype=torch.float64)])
        radii = torch.tensor([0.10, 0.22, 0.10], dtype=torch.float64) * (0.7 + 0.6 * torch.rand(3, generator=g))
        centre = torch.tensor([0.5 * (torch.rand(1, generator=g).item() - 0.5), 1.6 * (k + 0.5) / parts - 0.8,
                               0.2 * (torch.rand(1, generator=g).item() - 0.5)], dtype=torch.float64)
        uv = torch.cat([torch.tensor([[0.5, 0.0]], dtype=torch.float64),
                        torch.stack([(lon / (2 * math.pi))[None].expand(nlat - 1, -1),
                                     (lat / math.pi)[:, None].expand(-1, nlon)], -1).reshape(-1, 2),
                        torch.tensor([[0.5, 1.0]], dtype=torch.float64)])
        base = sum(v.shape[0] for v in verts)
        f = []
        for j in range(nlon):
            j1 = (j + 1) % nlon
            f.append((0, 1 + j1, 1 + j))
            for r in range(nlat - 2):
                a, b = 1 + r * nlon + j, 1 + r * nlon + j1
                f += [(a, b, a + nlon), (b, b + nlon, a + nlon)]
            last = 1 + (nlat - 2) * nlon
            f.append((last + j, last + j1, last + nlon))
        verts.append(pts * radii + centre)
        vt.append(uv)
        vi.append(torch.tensor(f, dtype=torch.int64) + base)
    verts, vt, vi = torch.cat(verts).float(), torch.cat(vt).float(), torch.cat(vi).to(torch.int32)
    f = 2000.0 * img_h / 2048.0
    K = torch.tensor([[f, 0.0, img_w / 2.0], [0.0, f, img_h / 2.0], [0.0, 0.0, 1.0]]).expand(batch, 3, 3).clone()
    Rt = torch.zeros(batch, 3, 4)
    for b in range(batch):
        yaw = 0.6 * (torch.rand(1, generator=g).item() - 0.5)
        c, s = math.cos(yaw), math.sin(yaw)
        Rt[b, :, :3] = torch.tensor([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
        Rt[b, :, 3] = torch.tensor([0.0, 0.0, 2.3 + 0.4 * torch.rand(1, generator=g).item()])
    return dict(verts=verts, vi=vi, vti=vi.clone(), vt=vt, K=K, Rt=Rt)


def uv_layout(n_charts: int = 64, quads: int = 16, seed: int = SEED + 11) -> Dict[str, torch.Tensor]:
    """A seeded UV layout of real-avatar size for the UV-image builders (goliath_b200.geom): n_charts jittered grid
    charts of quads x quads quads (2 quads^2 faces each, 32768 faces by default, windings mixed at random) packed in
    u < 0.45, and one large face covering about 9 % of the map; about half the map is uncovered, and its far corner is
    more than 100 texels from any chart at 1024^2.  Returns vt [N,2] fp32, vti [F,3] and vi [F,3] int64 (vi maps the
    UV corners to mesh vertices through a permutation), v2uv [V,1] int64."""
    g = torch.Generator().manual_seed(seed)
    side = int(math.ceil(math.sqrt(n_charts)))
    cell_u, cell_v = 0.43 / side, 0.96 / side
    vts, faces, base = [], [], 0
    for c in range(n_charts):
        u0, v0 = 0.02 + (c % side) * cell_u, 0.02 + (c // side) * cell_v
        a = torch.linspace(0.0, 1.0, quads + 1)
        uu, vv = torch.meshgrid(a * 0.9 * cell_u, a * 0.9 * cell_v, indexing="ij")
        jit = (torch.rand(quads + 1, quads + 1, 2, generator=g) - 0.5) * torch.tensor([cell_u, cell_v]) * (0.3 / quads)
        jit[0, :], jit[-1, :], jit[:, 0], jit[:, -1] = 0, 0, 0, 0
        vts.append(torch.stack([u0 + uu, v0 + vv], -1).add(jit).reshape(-1, 2))
        k = torch.arange((quads + 1) ** 2).reshape(quads + 1, quads + 1)
        q00, q10, q01, q11 = k[:-1, :-1], k[1:, :-1], k[:-1, 1:], k[1:, 1:]
        f = torch.cat([torch.stack([q00, q10, q11], -1).reshape(-1, 3), torch.stack([q00, q11, q01], -1).reshape(-1, 3)])
        flip = torch.rand(f.shape[0], generator=g) < 0.5
        f[flip] = f[flip][:, [0, 2, 1]]
        faces.append(f + base)
        base += (quads + 1) ** 2
    vts.append(torch.tensor([[0.46, 0.02], [0.78, 0.02], [0.46, 0.6]]))
    faces.append(torch.tensor([[base, base + 1, base + 2]]))
    vt = torch.cat(vts).float()
    vti = torch.cat(faces).long()
    V = vt.shape[0]
    perm = torch.randperm(V, generator=g)
    return {"vt": vt, "vti": vti, "vi": perm[vti], "v2uv": torch.arange(V)[:, None]}
