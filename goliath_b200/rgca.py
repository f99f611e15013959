"""RGCA `PrimDecoder` (ca_code/models/rgca.py:372-620) assembled from the sm_90a pieces: the two 7-layer
weight-normalised untied-bias deconv towers (rows R1, `goliath_b200.nn`), the fused Gaussian heads + SH diffuse
(row R2, `goliath_b200.rgca_heads`) and the SG specular shade (row R3, `goliath_b200.sgutils`).

Same constructor / forward arguments, the same `preds` keys (rgca.py:574-588) and the same parameter names and shapes
as the reference module, so its checkpoints load: `viewmod.0.*`, `encmod.0.*`, `vnocond_mod.{0,2,..,12}.*`,
`vcond_mod.{0,2,..,12}.*`, `albedo`.  `slabsize` (1024 upstream, hard-coded at rgca.py:385) is a parameter here so the
module can be exercised at small sizes.  The environment-map specular branch (`preconv_envmap`, rgca.py:548-556) is
one texture-fetch kernel (csrc/envmap_spec.cu, `goliath_b200.envmap_spec`); the training-only random back-light
outputs `cos_weight` / `color_rand` (rgca.py:590-618) come out of the heads kernel's pass over the diffuse planes
(second light-SH table), so the reference's `backlit_reg` loss finds both keys.

The joint texture + geometry `Encoder` (rgca.py:256-332) and the coarse-geometry `GeomDecoder` (rgca.py:335-369) are
mirrored with the same constructor arguments, state-dict keys and outputs; the encoder's eight stride-2 convolutions run
on the fused sm_90a kernels (`goliath_b200.nn.Conv2dWNUB(.., 4, 2, 1)` with the LeakyReLU in their epilogue), the
`LinearWN` layers, the input affine and the sampling noise are torch."""
from typing import Dict, Optional

import torch as th
import torch.nn as nn
import torch.nn.functional as F

from . import nn as gnn
from .envmap_spec import envmap_specular
from .rgca_heads import PRIMSCALE_RANGE, gaussian_heads, shade_and_compose
from .sh import dir2sh


def _tower(c_in, c_out, slab):
    plan = [(c_in, 256), (256, 128), (128, 128), (128, 64), (64, 32), (32, 16), (16, c_out)]
    layers, size = [], slab >> 6
    for i, (a, b) in enumerate(plan):
        act = nn.LeakyReLU(0.2, inplace=True) if i < len(plan) - 1 else None
        layers += gnn.make_conv_trans(a, b, 4, 2, 1, "wn", act, ub=(size, size))
        size *= 2
    return nn.Sequential(*layers)


class PrimDecoder(nn.Module):
    """A decoder for relightable Gaussians (same role and interface as rgca.PrimDecoder)."""

    def __init__(self, n_embs, geo_fn, color_mean: th.Tensor, n_diff_sh: int = 8, n_color_sh: int = 3, slabsize: int = 1024):
        super().__init__()
        assert (n_diff_sh, n_color_sh) == (8, 3), "the fused heads kernel implements the reference's SH split (8, 3)"
        assert slabsize >= 128 and slabsize & (slabsize - 1) == 0
        self.slabsize, self.n_splats, self.n_embs, self.geo_fn = slabsize, slabsize ** 2, n_embs, geo_fn
        self.base = slabsize >> 7  # 8 upstream
        self.viewmod = nn.Sequential(*gnn.make_linear(3, 8, "wn", nn.LeakyReLU(0.2, inplace=True)))
        self.encmod = nn.Sequential(*gnn.make_linear(n_embs, 256 * self.base * self.base, "wn", nn.LeakyReLU(0.2, inplace=True)))
        self.n_diff_coeffs = 113
        self.diff_sh_degree = n_diff_sh
        self.vnocond_mod = _tower(256, self.n_diff_coeffs + 12, slabsize)
        self.vcond_mod = _tower(256 + 8, 4, slabsize)
        # rgca.py:458-460: Glorot for a LeakyReLU(0.2) network, the two output layers with gain 1
        self.apply(lambda m: gnn.glorot(m, 0.2))
        gnn.glorot(self._last_deconv(self.vnocond_mod), 1.0)
        gnn.glorot(self._last_deconv(self.vcond_mod), 1.0)
        rgb = color_mean / 255.0
        self.albedo = nn.Parameter((2.0 * rgb / 2.2974).permute(1, 2, 0).reshape(1, -1, 3))
        # inference (no_grad) runs the towers on the tensor cores (wgmma + TMA, csrc/deconv_tc.cu); training uses
        # the SIMT kernels that also provide the backward (csrc/deconv_wnub.cu)
        self.use_tensor_cores = True

    @staticmethod
    def _last_deconv(tower):
        """the last ConvTranspose2dWNUB of a tower (a fused-activation placeholder may follow a layer, never the last)"""
        return [m for m in tower if isinstance(m, gnn.ConvTranspose2dWNUB)][-1]

    def _run_tower(self, tower, x):
        if self.use_tensor_cores and not th.is_grad_enabled():
            return gnn.tower_forward_tc(tower, x)
        return tower(x)

    def forward(self, embs, geom, headrel_campos, light_intensity, headrel_light_pos, headrel_light_sh, n_lights,
                preconv_envmap: Optional[th.Tensor] = None, lightrot: Optional[th.Tensor] = None):
        postex = self.geo_fn.to_uv(geom)
        tn = F.normalize(self.geo_fn.to_uv(self.geo_fn.vn(geom)), dim=1)
        x = self.encmod(embs).view(-1, 256, self.base, self.base)
        f_vnocond = self._run_tower(self.vnocond_mod, x)
        view = self.viewmod(F.normalize(headrel_campos, dim=1))[:, :, None, None].expand(-1, -1, self.base, self.base)
        f_vcond = self._run_tower(self.vcond_mod, th.cat([x, view], dim=1))
        rand_sh = light_dir = None
        if self.training:
            with th.no_grad():  # rgca.py:590-613: one random unit-intensity point light per batch item
                B = embs.shape[0]
                light_dir = F.normalize(th.rand(B, 1, 3, device=headrel_light_pos.device, dtype=headrel_light_pos.dtype) - 0.5,
                                        p=2, dim=-1)
                sh_coeffs = dir2sh(self.diff_sh_degree, light_dir)                       # [B,1,81]
                rand_int = th.ones_like(light_intensity[:, :1])                          # [B,1,3]
                rand_sh = (sh_coeffs[:, :, None] * rand_int[..., None]).sum(dim=1).contiguous()  # [B,3,81]
        heads = gaussian_heads(f_vnocond, f_vcond, postex, tn, self.albedo, headrel_light_sh, headrel_campos, PRIMSCALE_RANGE,
                               rand_light_sh=rand_sh)
        if preconv_envmap is not None:
            # rgca.py:548-556: pre-convolved mip pyramid looked up along the rotated reflection vector
            levels = [preconv_envmap] if th.is_tensor(preconv_envmap) else list(preconv_envmap)
            spec_color = envmap_specular(levels, heads["ref_dirs"], heads["sigma"], heads["spec_vis"], lightrot)
            preds = dict(heads)
            preds.update(spec_color=spec_color, color=(heads["diff_color"].clamp(min=0.0) + spec_color).clamp(min=0.0))
        else:
            preds = shade_and_compose(heads, light_intensity, headrel_light_pos, n_lights)
        if self.training:
            with th.no_grad():
                preds["cos_weight"] = (light_dir * preds["spec_nml"]).sum(dim=-1, keepdim=True)
            preds["color_rand"] = preds.pop("diff_color_rand").clamp(min=0.0)
        return preds


class Encoder(nn.Module):
    """A joint encoder for texture and geometry (rgca.Encoder): `geom` [B, n_verts_in, 3] and a 1024x1024 `color`
    texture in [0, 255] -> `embs`, `embs_mu`, `embs_logvar` [B, n_embs]."""

    def __init__(self, n_embs: int, n_verts_in: int, noise_std: float = 1.0, mean_scale: float = 0.1,
                 logvar_scale: float = 0.01):
        super().__init__()
        self.noise_std = noise_std
        self.n_embs = n_embs
        self.mean_scale = mean_scale
        self.logvar_scale = logvar_scale
        self.n_verts_in = n_verts_in
        self.geommod = nn.Sequential(gnn.LinearWN(self.n_verts_in * 3, 256), nn.LeakyReLU(0.2, inplace=True))
        # 1024^2 -> 4^2: the texture size is fixed by the reshape to 256 * 4 * 4 below, as upstream
        texmod = []
        for cin, cout, size in ((3, 32, 512), (32, 32, 256), (32, 64, 128), (64, 64, 64), (64, 128, 32), (128, 128, 16),
                                (128, 256, 8), (256, 256, 4)):
            layer = gnn.Conv2dWNUB(cin, cout, size, size, 4, 2, 1)
            layer.fused_slope = 0.2
            texmod += [layer, gnn.FusedLeakyReLU()]
        self.texmod = nn.Sequential(*texmod)
        self.jointmod = nn.Sequential(gnn.LinearWN(256 + 256 * 4 * 4, 512), nn.LeakyReLU(0.2, inplace=True))
        self.mean = gnn.LinearWN(512, self.n_embs)
        self.logvar = gnn.LinearWN(512, self.n_embs)
        self.apply(lambda m: gnn.glorot(m, 0.2))
        gnn.glorot(self.mean, 1.0)
        gnn.glorot(self.logvar, 1.0)

    def forward(self, geom: th.Tensor, color: th.Tensor) -> Dict[str, th.Tensor]:
        geomout = self.geommod(geom.view(geom.shape[0], -1))
        texout = self.texmod(color / 255.0 - 0.5).view(-1, 256 * 4 * 4)
        encout = self.jointmod(th.cat([geomout, texout], dim=1))
        embs_mu = self.mean(encout) * self.mean_scale
        embs_logvar = self.logvar(encout) * self.logvar_scale
        # the noise is only applied to the input-conditioned values; its scale is exp(logvar), as upstream
        if self.training:
            noise = th.randn_like(embs_mu)
            embs = embs_mu + th.exp(embs_logvar) * noise * self.noise_std
        else:
            embs = embs_mu.clone()
        return dict(embs=embs, embs_mu=embs_mu, embs_logvar=embs_logvar)


class GeomDecoder(nn.Module):
    """A decoder for coarse geometry (rgca.GeomDecoder): `embs` [B, n_embs] -> `face_geom` [B, n_verts, 3]."""

    def __init__(self, n_embs: int, verts_mean: th.Tensor, verts_std: float):
        super().__init__()
        self.verts_std: float = verts_std
        self.register_buffer("verts_mean", verts_mean[None].float())
        self.n_embs = n_embs
        self.n_verts_out = verts_mean.shape[-2]
        self.geommod = nn.Sequential(gnn.LinearWN(self.n_embs, 256), nn.LeakyReLU(0.2, inplace=True),
                                     gnn.LinearWN(256, 3 * self.n_verts_out))
        self.apply(lambda m: gnn.glorot(m, 0.2))
        gnn.glorot(self.geommod[-1], 1.0)

    def forward(self, embs: th.Tensor) -> Dict[str, th.Tensor]:
        geom = self.geommod(embs).view(embs.shape[0], -1, 3)
        geom = geom * self.verts_std + self.verts_mean
        return dict(face_geom=geom)
