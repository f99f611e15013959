"""Plain-torch restatement of the body avatar's texture branch, device-agnostic and in any dtype, with the reference's
parameter names: `UNetWB` (ca_code/nn/unet.py:14-93), `ShadowUNet` (ca_code/nn/shadow.py:22-188), `UNetViewDecoder`
and `UpscaleNet` (ca_code/models/mesh_vae.py:633-678) and `forward_tex` (mesh_vae.py:204-228), pinned to
tests/golden/body_texture_ref.npz by tests/test_body_texture_cpu.py and used as the fp64 oracle by the GPU tests.
Also the seeded inputs, parameters and view-cosine mesh shared by the fixture script, the tests and the profile."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

import seams_restate as sr

B = 2
UV, SHADOW, UV2K = 1024, 256, 2048  # mesh_vae_example.yml: decoder_view, shadow_net, AutoEncoder's 2k texture
TEX_STD = 64.0


def _wn(v, g):
    return v * (g / torch.linalg.vector_norm(v))


class WN(nn.Module):
    """Conv2dWN(UB) / ConvTranspose2dWNUB: w = g v / ||v||_F; bias None, tied [Cout] or untied [Cout,H,W]"""

    def __init__(self, cin, cout, k, stride=1, padding=0, bias=None, transposed=False):
        super().__init__()
        self.stride, self.padding, self.transposed = stride, padding, transposed
        shape = (cin, cout, k, k) if transposed else (cout, cin, k, k)
        self.weight_v = nn.Parameter(torch.empty(shape))
        self.weight_g = nn.Parameter(torch.empty((1, cout, 1, 1) if transposed else (cout, 1, 1, 1)))
        self.bias = None if bias is None else nn.Parameter(torch.zeros(bias))

    def forward(self, x):
        w = _wn(self.weight_v, self.weight_g)
        if self.transposed:
            y = F.conv_transpose2d(x, w, None, self.stride, self.padding)
        else:
            y = F.conv2d(x, w, None, self.stride, self.padding)
        if self.bias is None:
            return y
        return y + (self.bias[None, :, None, None] if self.bias.dim() == 1 else self.bias[None])


class Act(nn.Sequential):
    """[layer, LeakyReLU(0.2)] with the reference's child indices"""

    def __init__(self, layer, slope=0.2):
        super().__init__(layer, nn.LeakyReLU(slope))


class UNetWB(nn.Module):
    def __init__(self, cin, cout, size, F_=8, out_scale=0.1):
        super().__init__()
        self.out_scale = out_scale
        d = lambda a, b, s: Act(WN(a, b, 4, 2, 1, bias=(b, s, s)))
        u = lambda a, b, s: Act(WN(a, b, 4, 2, 1, bias=(b, s, s), transposed=True))
        self.down1, self.down2 = d(cin, F_, size // 2), d(F_, 2 * F_, size // 4)
        self.down3, self.down4 = d(2 * F_, 4 * F_, size // 8), d(4 * F_, 8 * F_, size // 16)
        self.down5 = d(8 * F_, 16 * F_, size // 32)
        self.up1, self.up2 = u(16 * F_, 8 * F_, size // 16), u(8 * F_, 4 * F_, size // 8)
        self.up3, self.up4 = u(4 * F_, 2 * F_, size // 4), u(2 * F_, F_, size // 2)
        self.up5 = u(F_, F_, size)
        self.out = WN(F_ + cin, cout, 1, bias=(cout, size, size))

    def forward(self, x):
        x1 = x
        x2 = self.down1(x1)
        x3 = self.down2(x2)
        x4 = self.down3(x3)
        x5 = self.down4(x4)
        x6 = self.down5(x5)
        x = self.up1(x6) + x5
        x = self.up2(x) + x4
        x = self.up3(x) + x3
        x = self.up4(x) + x2
        x = self.up5(x)
        return self.out(torch.cat([x, x1], 1)) * self.out_scale


class ShadowUNet(nn.Module):
    def __init__(self, uv_size, ao_mean, shadow_size, beta=1.0, n_dims=64, biases=True):
        super().__init__()
        self.uv_size, self.shadow_size, self.beta = uv_size, shadow_size, beta
        self.register_buffer("ao_mean", F.interpolate(torch.as_tensor(ao_mean)[None], size=(shadow_size,) * 2)[0])
        self.sizes = [shadow_size // 2 ** i for i in range(4)]
        enc = [(1, n_dims)] + [(n_dims, n_dims)] * 3
        dec = [(n_dims, n_dims)] + [(2 * n_dims, n_dims)] * 3
        self.enc_layers = nn.ModuleList([Act(WN(a, b, 3, 1, 1, bias=(b, s, s))) for (a, b), s in zip(enc, self.sizes)])
        self.dec_layers = nn.ModuleList([Act(WN(a, b, 3, 1, 1, bias=(b, s, s)))
                                         for (a, b), s in zip(dec, self.sizes[::-1])])
        s0 = self.sizes[0]
        self.shadow_pred = WN(n_dims, 1, 3, 1, 1, bias=(1, s0, s0) if biases else (1,))

    def forward(self, ao_map):
        if ao_map.shape[-2:] != (self.shadow_size, self.shadow_size):
            ao_map = F.interpolate(ao_map, size=(self.shadow_size, self.shadow_size))
        x = ao_map - self.ao_mean
        acts = []
        for i, layer in enumerate(self.enc_layers):
            x = layer(x)
            acts.append(x)
            if i < 3:
                x = F.interpolate(x, scale_factor=0.5, mode="bilinear", recompute_scale_factor=True, align_corners=True)
        for i, layer in enumerate(self.dec_layers):
            if i > 0:
                prev = acts[-i - 1]
                x = torch.cat([F.interpolate(x, size=prev.shape[2:4], mode="bilinear", align_corners=True), prev], 1)
            x = layer(x)
        low = torch.sigmoid(self.shadow_pred(x) + self.beta)
        full = F.interpolate(low, (self.uv_size,) * 2, mode="bilinear", align_corners=False)
        return {"shadow_map": full, "ao_map": ao_map, "shadow_map_lowres": low}


def vert_normals(v, vi, eps=1e-5):
    pts = v[:, vi]
    n = torch.cross(pts[:, :, 1] - pts[:, :, 0], pts[:, :, 2] - pts[:, :, 0], dim=-1)
    n = n / n.norm(dim=-1, keepdim=True).clamp(min=eps)
    vn = torch.zeros_like(v).index_add_(1, vi.reshape(-1), n[:, :, None].expand(-1, -1, 3, -1).reshape(v.shape[0], -1, 3))
    return vn / vn.norm(dim=-1, keepdim=True).clamp(min=eps)


def view_cos_uv(verts, vi, campos, index_img, bary_img):
    vn = F.normalize(vert_normals(verts, vi), dim=-1)
    v2c = F.normalize(verts - campos[:, None], dim=-1)
    cos = (vn * v2c).sum(-1)
    mask = (index_img != -1).all(-1)
    vals = (cos[:, index_img[mask].long()] * bary_img[mask].to(cos.dtype)).sum(-1)
    out = torch.zeros(verts.shape[0], 1, *index_img.shape[:2], dtype=cos.dtype, device=cos.device)
    out[:, 0, mask] = vals
    return out


class UNetViewDecoder(nn.Module):
    def __init__(self, vi, index_img, bary_img, net_uv_size, n_init_ftrs=8):
        super().__init__()
        self.vi, self.index_img, self.bary_img = vi, index_img, bary_img
        self.unet = UNetWB(4, 3, net_uv_size, n_init_ftrs)

    def forward(self, geom_rec, tex_mean_rec, camera_pos):
        with torch.no_grad():
            vc = view_cos_uv(geom_rec, self.vi, camera_pos, self.index_img, self.bary_img)
        cond = torch.cat([vc.to(tex_mean_rec.dtype), tex_mean_rec], 1)
        return {"tex_view_rec": self.unet(cond), "cond_view": cond}


class UpscaleNet(nn.Module):
    def __init__(self, cin, cout, n_ftrs, size=1024, r=2):
        super().__init__()
        self.conv_block = Act(WN(cin, n_ftrs, 3, 1, 1, bias=(n_ftrs, size, size)))
        self.out_block = WN(n_ftrs, cout * r * r, 1, bias=(cout * r * r, size, size))
        self.r = r

    def forward(self, x):
        return F.pixel_shuffle(self.out_block(self.conv_block(x)), self.r)


class TextureComposer(nn.Module):
    """forward_tex with the reference's operation order; samplers are seams_restate.TorchSeamSampler (out of place)"""

    def __init__(self, seam, seam_2k, tex_mean, tex_std=TEX_STD, n_ftrs=4):
        super().__init__()
        self.upscale_net = UpscaleNet(6, 3, n_ftrs)
        self.seam, self.seam_2k, self.tex_std = seam, seam_2k, tex_std
        self.register_buffer("tex_mean", tex_mean)

    def forward(self, tex_mean_rec, tex_view_rec, shadow_map):
        x = torch.cat([tex_mean_rec, tex_view_rec], 1)
        t = self.seam.resample(self.seam.impaint(tex_mean_rec + tex_view_rec))
        t = F.interpolate(t, size=tuple(self.tex_mean.shape[2:]), mode="bilinear", align_corners=False)
        t = (t + self.upscale_net(x)) * self.tex_std + self.tex_mean
        s = self.seam_2k.resample(self.seam_2k.resample(self.seam_2k.impaint(shadow_map)))
        t = t * s
        return self.seam_2k.resample(self.seam_2k.resample(self.seam_2k.impaint(t)))


def compose(t1, h, v, g, bias, tex_std, tex_mean, s3):
    """the composite kernel's formula: ((U(T1) + PS(out_block(h))) * tex_std + tex_mean) * S3"""
    z = F.conv2d(h, _wn(v, g)) + bias[None]
    u = F.interpolate(t1, scale_factor=2, mode="bilinear", align_corners=False)
    return ((u + F.pixel_shuffle(z, 2)) * tex_std + tex_mean) * s3


# ---------------------------------------------------------------- shared data
def seeded_fill(module, seed):
    """oracle.mesh_vae_oracle.seeded_fill: weight_v ~ N(0, 2/fan), weight_g in [0.5, 1.5), other params 0.05 N(0, 1)"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(module.named_parameters()):
            if name.endswith("weight_v"):
                p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64) * (2.0 / max(1, p[0].numel())) ** 0.5)
            elif name.endswith("weight_g"):
                p.copy_(0.5 + torch.rand(p.shape, generator=g, dtype=torch.float64))
            else:
                p.copy_(0.05 * torch.randn(p.shape, generator=g, dtype=torch.float64))
    return module


def uv_mesh(n=48, size=UV, seed=4):
    """a UV-gridded n x n vertex sheet with a bumpy z: vi [F,3] (int64), verts0 [V,3], index / bary images [S,S,3]
    from the grid's triangulation; texels in the left 40 columns and in random 3 % of the rest are uncovered (-1)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:n, 0:n]
    verts = np.stack([xx / (n - 1), yy / (n - 1), 0.1 * rng.standard_normal((n, n))], -1).reshape(-1, 3)
    q = (yy[:-1, :-1] * n + xx[:-1, :-1]).reshape(-1)
    vi = np.concatenate([np.stack([q, q + 1, q + n], 1), np.stack([q + 1, q + n + 1, q + n], 1)], 0)
    c = (np.arange(size) + 0.5) / size * (n - 1)
    cx, cy = np.meshgrid(c, c)
    ix, iy = np.minimum(cx.astype(int), n - 2), np.minimum(cy.astype(int), n - 2)
    fx, fy = cx - ix, cy - iy
    q = iy * n + ix
    lower = fx + fy < 1
    idx = np.where(lower[..., None], np.stack([q, q + 1, q + n], -1), np.stack([q + 1, q + n + 1, q + n], -1))
    bary = np.where(lower[..., None], np.stack([1 - fx - fy, fx, fy], -1), np.stack([1 - fy, fx + fy - 1, 1 - fx], -1))
    hole = (cx < 40.0 / size * (n - 1)) | (rng.random((size, size)) < 0.03)
    idx[hole] = -1
    bary[hole] = 0.0
    return (torch.as_tensor(vi, dtype=torch.int64), torch.as_tensor(verts, dtype=torch.float64),
            torch.as_tensor(idx, dtype=torch.int32), torch.as_tensor(bary, dtype=torch.float32))


def seeded_inputs(batch=B, seed=31):
    """geom_rec [B,V,3], camera_pos [B,3], tex_mean_rec [B,3,1024,1024], ao_map [B,1,1024,1024] (resized to 256^2 by
    nearest, as the reference does for an AO map of another size), ao_mean [1,512,512], tex_mean [1,3,2048,2048]"""
    g = torch.Generator().manual_seed(seed)
    _, verts0, _, _ = uv_mesh()
    f64 = dict(generator=g, dtype=torch.float64)
    geom = verts0[None] + 0.02 * torch.randn(batch, *verts0.shape, **f64)
    campos = torch.tensor([0.5, 0.5, 3.0], dtype=torch.float64) + torch.randn(batch, 3, **f64)
    tex_mean_rec = 0.3 * torch.randn(batch, 3, UV, UV, **f64)
    ao = torch.rand(batch, 1, UV, UV, **f64)
    ao_mean = 0.5 + 0.1 * torch.randn(1, 512, 512, **f64)
    tex_mean = 100.0 + 20.0 * torch.randn(1, 3, UV2K, UV2K, **f64)
    return {"geom_rec": geom, "camera_pos": campos, "tex_mean_rec": tex_mean_rec, "ao_map": ao, "ao_mean": ao_mean,
            "tex_mean": tex_mean}


def seams():
    return sr.synthetic_seams(UV), sr.synthetic_seams(UV2K, n_pairs=16000, seed=5)
