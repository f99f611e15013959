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
`LinearWN` layers, the input affine and the sampling noise are torch.

`AutoEncoder` (rgca.py:50-253) binds them into the head avatar's frame: the head-relative light work in one kernel
(`head_lights`, csrc/head_frame.cu), encoder -> geometry decoder -> Gaussian decoder, the splat render
(`render.render_views`, or `gsplat.olat.render_views_shared` for the environment-map frame) and the image finish on
`photo_loss.post_render`."""
import math
from typing import Any, Dict, List, Optional

import torch as th
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
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


def head_lights(head_pose: th.Tensor, campos: th.Tensor, Rt: th.Tensor, light_pos: th.Tensor,
                light_intensity: th.Tensor, lightrot: Optional[th.Tensor] = None) -> Dict[str, th.Tensor]:
    """rgca.py:175-193 in one launch (csrc/head_frame.cu): head_pose [B,3,4] (R | t), campos [B,3], Rt [B,3,4],
    light_pos [B,L,3], light_intensity [B,L,C] with C in {1, 3}, lightrot [B,3,3] or None ->
    headrel_Rt [B,3,4] = Rt @ [head_pose; 0 0 0 1], headrel_campos [B,3], headrel_light_pos [B,L,3],
    headrel_light_sh [B,3,81] (degree-8 SH of the normalised light directions times the intensities, summed over all
    L lights) and lightrot = lightrot @ R (None without one).  fp32 CUDA tensors; no gradient: an input that requires
    grad is refused.  The reduction over L is in a fixed order, so two calls give the same bits."""
    args = {"head_pose": head_pose, "campos": campos, "Rt": Rt, "light_pos": light_pos,
            "light_intensity": light_intensity}
    if lightrot is not None:
        args["lightrot"] = lightrot
    for name, t in args.items():
        if t.requires_grad:
            raise RuntimeError("head_lights: %s requires grad; the light kernel has no backward" % name)
    args = {k: v.contiguous() for k, v in args.items()}
    for name, t in args.items():
        _lib.check_input(t, name)
    B = args["head_pose"].shape[0]
    L = args["light_pos"].shape[1] if args["light_pos"].dim() == 3 else -1
    C = args["light_intensity"].shape[-1] if args["light_intensity"].dim() == 3 else -1
    shapes = {"head_pose": (B, 3, 4), "campos": (B, 3), "Rt": (B, 3, 4), "light_pos": (B, L, 3),
              "light_intensity": (B, L, C), "lightrot": (B, 3, 3)}
    for name, t in args.items():
        if tuple(t.shape) != shapes[name] or C not in (1, 3):
            raise RuntimeError("head_lights: %s must have shape %s with C in {1, 3} (got %s)"
                               % (name, shapes[name], tuple(t.shape)))
    dev = args["head_pose"].device
    f32 = dict(device=dev, dtype=th.float32)
    out = {"headrel_Rt": th.empty(B, 3, 4, **f32), "headrel_campos": th.empty(B, 3, **f32),
           "headrel_light_pos": th.empty(B, L, 3, **f32), "headrel_light_sh": th.empty(B, 3, 81, **f32),
           "lightrot": th.empty(B, 3, 3, **f32) if lightrot is not None else None}
    with th.cuda.device(dev):
        _lib.check(_lib.lib().gb_head_lights_fwd(
            B, L, C, _lib.ptr(args["head_pose"]), _lib.ptr(args["campos"]), _lib.ptr(args["Rt"]),
            _lib.ptr(args["light_pos"]), _lib.ptr(args["light_intensity"]), _lib.ptr(args.get("lightrot")),
            _lib.ptr(out["headrel_Rt"]), _lib.ptr(out["headrel_campos"]), _lib.ptr(out["headrel_light_pos"]),
            _lib.ptr(out["headrel_light_sh"]), _lib.ptr(out["lightrot"]), _lib.stream_ptr(dev)), "head_lights_fwd")
    return out


class AutoEncoder(nn.Module):
    """rgca.AutoEncoder (rgca.py:50-253): the head avatar's frame with the reference's constructor, state-dict keys
    (`geo_fn.*` and `decoder.geo_fn.*` are the same module; there is no v2uv) and output keys, so
    `AutoEncoder(**config.model, assets=assets)` builds from rgca_example.yml and a head checkpoint loads with
    strict=True.  `decoder` may carry `slabsize` (1024 upstream) to run the frame at small sizes.

    `assets` (attributes or dict keys) carries the reference's assets and, because this project does not rasterise the
    UV layout, the four `geo_fn` images a head checkpoint stores, at 1024 x 1024 in the head's flip_uv=True
    orientation: index_image / bary_image [1024,1024,3], face_index_image [1024,1024] and valid_mask
    [1024,1024,1] (slabsize x slabsize when `decoder` sets a slabsize).  Construction raises an error that names any
    missing image.

    Differences from the reference: the intrinsics come from one host copy of K per call (the reference makes four
    `.item()` calls per view); the light work (`head_lights`) has no gradient; the point-light frame's calibration,
    training background and learnable blur run as one `post_render` call; the environment-map frame renders its three
    colour sets from one projection and binning per view.  forward() runs on CUDA only."""

    def __init__(self, encoder, decoder, assets, image_height, image_width, cal=None, n_embs: int = 256,
                 n_diff_sh: int = 8, learn_blur: bool = True, bg_weight: float = 1.0):
        super().__init__()
        from .mesh_vae import _get, _uv_geometry
        from .photo_loss import CalV5, LearnableBlur

        if n_diff_sh != 8:
            raise ValueError("AutoEncoder: n_diff_sh must be 8, the degree of the light kernel and the heads kernel "
                             "(got %r)" % (n_diff_sh,))
        self.height = image_height
        self.width = image_width
        self.n_diff_sh = n_diff_sh
        self.bg_weight = bg_weight
        # the UV images are the slab's texel grid: 1024 x 1024 at the reference's size
        self.geo_fn, _ = _uv_geometry(assets, with_v2uv=False, size=decoder.get("slabsize", 1024))
        self.encoder = Encoder(n_embs=n_embs, n_verts_in=_get(_get(assets, "topology"), "v").shape[0], **encoder)
        self.geomdecoder = GeomDecoder(n_embs=n_embs, verts_std=math.sqrt(_get(assets, "verts_var")),
                                       verts_mean=th.as_tensor(_get(assets, "verts_mean")))
        self.decoder = PrimDecoder(n_embs=n_embs, geo_fn=self.geo_fn,
                                   color_mean=th.as_tensor(_get(assets, "color_mean"), dtype=th.float32),
                                   n_diff_sh=self.n_diff_sh, **decoder)
        cameras = _get(assets, "camera_ids")
        self.learn_blur_enabled = False
        if learn_blur:
            self.learn_blur_enabled = True
            self.learn_blur = LearnableBlur(cameras)
        self.cal_enabled = False
        if cal is not None:
            self.cal_enabled = True
            self.cal = CalV5(**cal, cameras=cameras)

    @staticmethod
    def intrinsics(K: th.Tensor) -> List[tuple]:
        """(fx, fy, cx, cy) per view from one host copy of K [B,3,3]"""
        Kh = K.detach().to("cpu").tolist()
        return [(k[0][0], k[1][1], k[0][2], k[1][2]) for k in Kh]

    def render(self, K: th.Tensor, Rt: th.Tensor, preds: Dict[str, Any], intrinsics_host=None):
        """rgca.py:112-151: rgb [B,3,H,W], alpha [B,1,H,W] (from the detached final T) and
        depth / alpha.clamp(0.05, 1)"""
        from .render import render_views

        if intrinsics_host is None:
            intrinsics_host = self.intrinsics(K)
        return render_views(self.width, self.height, K, Rt, preds, intrinsics_host=intrinsics_host)

    def forward(self, head_pose: th.Tensor, campos: th.Tensor, registration_vertices: th.Tensor, color: th.Tensor,
                light_intensity: th.Tensor, light_pos: th.Tensor, n_lights: th.Tensor, K: th.Tensor, Rt: th.Tensor,
                background: Optional[th.Tensor] = None, is_fully_lit_frame: Optional[th.Tensor] = None,
                camera_id: Optional[List[str]] = None, frame_id: Optional[th.Tensor] = None,
                iteration: Optional[int] = None, preconv_envmap: Optional[th.Tensor] = None,
                lightrot: Optional[th.Tensor] = None, **kwargs) -> Dict[str, Any]:
        from .envmap import compose_envmap
        from .gsplat.olat import render_views_shared
        from .photo_loss import post_render

        B = head_pose.shape[0]
        if (self.cal_enabled or self.learn_blur_enabled) and camera_id is None:
            raise ValueError("AutoEncoder.forward: camera_id is needed while cal_enabled or learn_blur_enabled")
        lights = head_lights(head_pose, campos, Rt, light_pos, light_intensity, lightrot)
        light_intensity = light_intensity.expand(-1, -1, 3)
        headrel_light_sh = lights["headrel_light_sh"]

        enc_preds = self.encoder(registration_vertices, color)
        geom = self.geomdecoder(enc_preds["embs"])["face_geom"]
        dec_preds = self.decoder(enc_preds["embs"], geom, lights["headrel_campos"], light_intensity,
                                 lights["headrel_light_pos"], headrel_light_sh, n_lights, preconv_envmap,
                                 lights["lightrot"])
        # the reference's output keys: the reflection directions the heads kernel hands the shade stay internal
        dec_preds.pop("ref_dirs", None)
        preds = {"geom": geom, "headrel_light_sh": headrel_light_sh, **enc_preds, **dec_preds}

        intrinsics_host = self.intrinsics(K)
        headrel_Rt = lights["headrel_Rt"]
        cal_w = cal_b = grey = bg = None
        if self.cal_enabled:
            cal_w, cal_b, grey = self.cal.rows(self.cal.name_to_idx(camera_id))
        if self.training and background is not None:
            if is_fully_lit_frame is None:
                raise ValueError("AutoEncoder.forward: a training background needs is_fully_lit_frame")
            lit = (is_fully_lit_frame.reshape(B) != 0).to(background.dtype)
            bg = background[:, :3] * lit[:, None, None, None]
        blur_w = self.learn_blur.weights(camera_id) if self.learn_blur_enabled else None

        if preconv_envmap is not None and "envbg" in kwargs:
            colors = th.stack([preds["color"].reshape(B, -1, 3), preds["diff_color"].reshape(B, -1, 3).clamp(min=0.0),
                               preds["spec_color"].reshape(B, -1, 3).clamp(min=0.0)], 1)
            geo = {k: preds[k] for k in ("primpos", "primqvec", "primscale", "opacity")}
            rgbs, alpha, depth = render_views_shared(self.width, self.height, headrel_Rt, geo, colors, intrinsics_host)
            full = rgbs[:, 0]
            if cal_w is not None or bg is not None:
                full = post_render(full, alpha if bg is not None else None, bg, cal_w, cal_b, grey)
            full = compose_envmap(full, alpha, kwargs["envbg"], K, Rt)
            rgb = th.cat([full, rgbs[:, 1], rgbs[:, 2]], -1)
            preds["color"] = preds["spec_color"].clamp(min=0.0)
            if blur_w is not None:
                rgb = post_render(rgb, blur_weights=blur_w)
        else:
            rgb, alpha, depth = self.render(K, headrel_Rt, preds, intrinsics_host)
            if cal_w is not None or bg is not None or blur_w is not None:
                rgb = post_render(rgb, alpha if bg is not None else None, bg, cal_w, cal_b, grey, blur_w)

        preds.update(rgb=rgb, alpha=alpha, depth=depth)
        if self.learn_blur_enabled:
            preds["learn_blur_weights"] = self.learn_blur.reg(camera_id)
        return preds
