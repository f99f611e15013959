"""Plain-torch restatement (any dtype, CPU or CUDA) of the reference's body encoders, for tests and the profile script:
`blocks.ConvDownBlock` (ca_code/nn/blocks.py:327-379), `mesh_vae.Encoder` / `FaceEncoder` (ca_code/models/
mesh_vae.py:344-436) on the weight-normalised layers of oracle/mesh_vae_oracle.py, and the skinning / unskinning of
ca_code/utils/lbs.py:226-306 on given joint matrices.  Parameter names and shapes are the reference's;
tests/golden/make_body_encoder_golden.py runs the reference's own classes against this module on the same weights and
freezes the result in tests/golden/body_encoder_ref.npz."""
import numpy as np
import torch as th
import torch.nn as nn
import torch.nn.functional as F

from oracle.mesh_vae_oracle import LinearWN, _wn, seeded_fill  # noqa: F401  (seeded_fill is re-exported)

ENCODER_BLOCKS = [(3, 8, 512), (8, 16, 256), (16, 32, 128), (32, 32, 64), (32, 64, 32), (64, 128, 16), (128, 128, 8)]
GRAD_PARAMS = ("verts_conv.conv1.weight_v", "verts_conv.conv_resize.bias", "verts_conv.conv2.weight_g",
               "joint_conv_blocks.2.conv2.weight_g", "joint_conv_blocks.3.conv_resize.weight_v",
               "joint_conv_blocks.5.conv2.bias", "mu.weight_g")


class _Conv(nn.Module):
    """Conv2dWN (tied bias [C]) or Conv2dWNUB (untied bias [C,H,W]) with stride and groups"""

    def __init__(self, cin, cout, k, stride, padding, groups, ub=None):
        super().__init__()
        self.stride, self.padding, self.groups = stride, padding, groups
        self.weight_v = nn.Parameter(th.empty(cout, cin // groups, k, k))
        self.weight_g = nn.Parameter(th.empty(cout, 1, 1, 1))
        self.bias = nn.Parameter(th.zeros(cout) if ub is None else th.zeros(cout, ub, ub))

    def forward(self, x):
        y = F.conv2d(x, _wn(self.weight_v, self.weight_g), None, self.stride, self.padding, 1, self.groups)
        return y + (self.bias[None, :, None, None] if self.bias.dim() == 1 else self.bias[None])


class ConvDownBlock(nn.Module):  # blocks.py:327-379; `size` is the input size
    def __init__(self, cin, cout, size, groups=1, slope=0.2):
        super().__init__()
        self.slope = slope
        self.conv_resize = _Conv(cin, cout, 1, 2, 0, groups)
        self.conv1 = _Conv(cin, cin, 3, 1, 1, groups, ub=size)
        self.conv2 = _Conv(cin, cout, 3, 2, 1, groups, ub=size // 2)

    def forward(self, x):
        skip = self.conv_resize(x)
        x = F.leaky_relu(self.conv1(x), self.slope)
        x = F.leaky_relu(self.conv2(x), self.slope)
        return x + skip


def condition(verts_unposed_uv, mask, verts_scale=1.0, size=512):
    """mesh_vae.py:394-399"""
    return F.interpolate(verts_unposed_uv * verts_scale, size=(size, size), mode="bilinear") * mask


class Encoder(nn.Module):  # mesh_vae.py:344-421
    def __init__(self, n_embs, mask, noise_std=1.0, mean_scale=0.1, logvar_scale=0.1, verts_scale=1.0):
        super().__init__()
        self.noise_std, self.mean_scale, self.logvar_scale, self.verts_scale = noise_std, mean_scale, logvar_scale, verts_scale
        self.verts_conv = ConvDownBlock(*ENCODER_BLOCKS[0])
        mask = th.as_tensor(mask[np.newaxis, np.newaxis], dtype=th.float32)
        self.register_buffer("mask", F.interpolate(mask, size=(512, 512), mode="bilinear").to(th.bool))
        self.joint_conv_blocks = nn.Sequential(*(ConvDownBlock(*b) for b in ENCODER_BLOCKS[1:]))
        self.mu = LinearWN(4 * 4 * 128, n_embs)
        self.logvar = LinearWN(4 * 4 * 128, n_embs)

    def forward(self, verts_unposed_uv):
        x = self.verts_conv(condition(verts_unposed_uv, self.mask, self.verts_scale))
        x = self.joint_conv_blocks(x).reshape(verts_unposed_uv.shape[0], -1)
        mu = self.mean_scale * self.mu(x)
        logvar = self.logvar_scale * self.logvar(x)
        if self.training:
            embs = mu + th.exp(logvar) * th.randn_like(mu) * self.noise_std
        else:
            embs = mu.clone()
        return {"embs": embs, "embs_mu": mu, "embs_logvar": logvar}


class FaceEncoder(nn.Module):  # mesh_vae.py:424-436
    def __init__(self, mask, **kwargs):
        super().__init__()
        self.encoder = Encoder(**kwargs, mask=mask[512:, :512])

    def forward(self, verts_unposed_uv):
        return {"face_" + k: v for k, v in self.encoder(verts_unposed_uv[:, :, 512:, :512]).items()}


# ------------------------------------------------------------------------------------------ skinning on given matrices
def blended(mats, skin_idx, skin_w):
    """[B,J,3,4], [V,8], [V,8] -> the per-vertex blended matrices [B,V,3,4] (lbs.py:290-291)"""
    return (mats[:, skin_idx.long()] * skin_w[None, :, :, None, None].to(mats.dtype)).sum(2)


def skinning(mats, skin_idx, skin_w, verts):  # lbs.py:226-254
    m = blended(mats, skin_idx, skin_w)
    return (m[..., :3] @ verts[..., None])[..., 0] + m[..., 3]


def unskinning(mats, skin_idx, skin_w, verts):  # lbs.py:273-306, as the affine inverse
    m = blended(mats, skin_idx, skin_w)
    return th.linalg.solve(m[..., :3], (verts - m[..., 3])[..., None])[..., 0]


# ------------------------------------------------------------------------------------------ seeded inputs
def synthetic_mask(size=1024, seed=3):
    """a body mask of the asset's shape: random texels inside a disc, so both the body map and the face window see
    covered and uncovered regions"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:size, 0:size]
    disc = (yy - size / 2) ** 2 + (xx - size / 2) ** 2 < (0.48 * size) ** 2
    return (disc & (rng.random((size, size)) < 0.9)).astype(np.float32)


def seeded_uv(batch=1, size=1024, seed=17):
    g = th.Generator().manual_seed(seed)
    return th.randn(batch, 3, size, size, generator=g)
