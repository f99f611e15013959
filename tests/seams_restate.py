"""Plain-torch restatement of the reference's seam sampler (ca_code/utils/seams.py:14-25) and sample_uv
(ca_code/utils/geom.py:281-304), device-agnostic and out of place, pinned to tests/golden/seams_ref.npz by
tests/test_body_decoder_cpu.py; plus device-aware copies of the oracle's decoder stand-ins
(oracle.mesh_vae_oracle.identity_resample / uv_vertex_gather) for maps that live on the GPU."""
import types

import numpy as np
import torch
import torch.nn.functional as F


def impaint_batch(value, dst_ij, src_ij):
    out = value.clone()
    out[:, :, dst_ij[:, 0], dst_ij[:, 1]] = value[:, :, src_ij[:, 0], src_ij[:, 1]]
    return out


def resample_tex(tex, uvs, weights):
    grid = 2.0 * (uvs[None].expand(tex.shape[0], -1, -1, -1) - 0.5)
    return (1.0 - weights) * tex + weights * F.grid_sample(tex, grid.to(tex.dtype), align_corners=False,
                                                           padding_mode="border")


def sample_uv(values_uv, uv_coords, v2uv=None):
    grid = (uv_coords * 2.0 - 1.0)[None, :, None].expand(values_uv.shape[0], -1, -1, -1).to(values_uv.dtype)
    values = F.grid_sample(values_uv, grid, align_corners=True, mode="bilinear").squeeze(-1).permute(0, 2, 1)
    if v2uv is not None:
        values = values[:, v2uv.long()].mean(2)
    return values


class TorchSeamSampler:
    """the reference's SeamSampler behaviour on any device"""

    def __init__(self, dst_ij, src_ij, uvs, weights):
        self.dst_ij, self.src_ij, self.uvs, self.weights = dst_ij.long(), src_ij.long(), uvs, weights

    def impaint(self, x):
        return impaint_batch(x, self.dst_ij, self.src_ij)

    def resample(self, x):
        return resample_tex(x, self.uvs.to(x.dtype), self.weights.to(x.dtype))


def synthetic_seams(size, n_pairs=4000, seed=3):
    """seam data of the reference's layout for a size x size map: unique dst texels, src texels that may repeat and may
    themselves be dst, uvs within half a texel-ish of the identity plus some outside [0, 1], weights in [0, 1]"""
    rng = np.random.default_rng(seed)
    flat = rng.choice(size * size, 2 * n_pairs, replace=False)
    dst = np.stack(np.divmod(flat[:n_pairs], size), 1)
    src_flat = np.concatenate([flat[n_pairs:n_pairs + n_pairs // 2], flat[: n_pairs // 4],
                               rng.choice(flat[n_pairs:], n_pairs - n_pairs // 2 - n_pairs // 4)])
    src = np.stack(np.divmod(src_flat, size), 1)
    yy, xx = np.mgrid[0:size, 0:size]
    uvs = np.stack([(xx + 0.5) / size, (yy + 0.5) / size], -1) + rng.normal(0, 3.0 / size, (size, size, 2))
    uvs[:8] -= 0.02
    w = rng.random((size, size))
    w[rng.random((size, size)) < 0.5] = 0.0
    t = lambda a, d: torch.as_tensor(a, dtype=d)
    return dict(dst_ij=t(dst, torch.int64), src_ij=t(src, torch.int64), uvs=t(uvs, torch.float32),
                weights=t(w, torch.float32))


def identity_resample(x):
    """oracle.mesh_vae_oracle.identity_resample with its grid built on x's device"""
    n, _, h, w = x.shape
    ys = torch.linspace(-1, 1, h, device=x.device).view(1, h, 1).expand(n, h, w) + 1.0 / h
    xs = torch.linspace(-1, 1, w, device=x.device).view(1, 1, w).expand(n, h, w)
    return F.grid_sample(x, torch.stack([xs, ys], -1).to(x.dtype), mode="bilinear", padding_mode="border",
                         align_corners=True)


def uv_vertex_gather(n_verts=7306, seed=5):
    """oracle.mesh_vae_oracle.uv_vertex_gather with its coordinates moved to the map's device"""
    uv = torch.from_numpy(np.random.default_rng(seed).random((1, 1, n_verts, 2)).astype(np.float32)) * 2 - 1

    def from_uv(t):
        return F.grid_sample(t, uv.to(t.device).expand(t.shape[0], -1, -1, -1).to(t.dtype), mode="bilinear",
                             align_corners=False)[:, :, 0].permute(0, 2, 1)

    return types.SimpleNamespace(from_uv=from_uv)


def stand_in_sampler():
    return types.SimpleNamespace(impaint=identity_resample, resample=identity_resample)
