"""The drivable body avatar (ca_code/models/mesh_vae_drivable.py) on the GPU, with the reference's constructors and
state-dict keys, so `AutoEncoder(**config.model, assets=assets)` loads a reference checkpoint with strict=True.

It is built from the mesh_vae stages: `Encoder` and `ConvDecoder` are `mesh_vae.Encoder` / `mesh_vae.ConvDecoder` with
the drivable model's constructor and call signature, and the texture, shadow, calibration and render stages are the
same modules.  What is new: the face region is conditioned on a face model's latent code through the frozen
`face.FaceDecoderFrontal` and the texture-conditioned `FaceEncoder` here, and `shadow.PoseToShadow` drives the shadow
from the pose alone, so the frame needs no ambient-occlusion map in eval."""
import numpy as np
import torch
import torch.nn as tnn
import torch.nn.functional as F

from . import _lib
from . import mesh_vae as mv
from .face import FaceDecoderFrontal
from .nn import ConvDownBlock, LinearWN, glorot
from .seams import SeamSampler


class Encoder(mv.Encoder):
    """mesh_vae_drivable.py:387-466: `mesh_vae.Encoder` that lays the unposed vertices out in UV itself (through
    `geo_fn.to_uv`, then the first block's fused resize + bool mask) and has no `mean_scale` (1.0 here)."""

    def __init__(self, geo_fn, n_embs, noise_std, mask, logvar_scale=0.1):
        super().__init__(n_embs, mask, noise_std=noise_std, mean_scale=1.0, logvar_scale=logvar_scale)
        self.geo_fn = geo_fn

    def forward(self, motion, verts_unposed):
        return super().forward(self.geo_fn.to_uv(verts_unposed))


class ConvDecoder(mv.ConvDecoder):
    """mesh_vae_drivable.py:469-653: `mesh_vae.ConvDecoder` without output scales (1.0 here).  forward(motion, embs,
    face_embs, embs_conv=None): a given `embs_conv` replaces the decoded `embs` map.  Unlike the reference, which
    merges the face region into the caller's `embs_conv` in place (:621-624), the caller's tensor is left as it is;
    preds["embs_conv"] is the merged copy."""

    def __init__(self, geo_fn, uv_size, seam_sampler, init_uv_size, n_pose_dims, n_pose_enc_channels, n_embs,
                 n_embs_enc_channels, n_face_embs, n_init_channels, n_min_channels, assets):
        super().__init__(geo_fn, uv_size, seam_sampler, init_uv_size, n_pose_dims, n_pose_enc_channels, n_embs,
                         n_embs_enc_channels, n_face_embs, n_init_channels, n_min_channels, assets, tex_scale=1.0,
                         verts_scale=1.0)

    def forward(self, motion, embs, face_embs, embs_conv=None):
        return super().forward(motion, embs, face_embs, embs_conv)


def face_tex_cond(face_tex, mask):
    """(bilinear(face_tex -> mask's size, align_corners=False) / 255 - 0.5) * mask on csrc/body_drive.cu, forward
    only; face_tex [B, C, Hs, Ws], mask [.., H, W]"""
    face_tex = face_tex.contiguous()
    _lib.check_input(face_tex, "face_tex")
    mask = mask.contiguous()
    _lib.check_input(mask, "tex_cond_mask")
    B, C, Hs, Ws = face_tex.shape
    H, W = mask.shape[-2:]
    if mask.numel() != H * W:
        raise RuntimeError("tex_cond_mask must hold one [H, W] plane")
    out = torch.empty(B, C, H, W, device=face_tex.device)
    _lib.kernels().gb_face_tex_cond_fwd(B, C, Hs, Ws, H, W, face_tex, mask, out)
    return out


class FaceEncoder(tnn.Module):
    """mesh_vae_drivable.py:656-748: the face code in body space from the face decoder's geometry and texture.
    `tex_cond_mask` is a float buffer (the mask interpolated with align_corners=True, never cast to bool); the
    conditioning `(bilinear(face_tex -> 512^2) / 255 - 0.5) * tex_cond_mask` is one kernel (`face_tex_cond`) whose
    output is returned as `face_tex_cond` and read by the first of seven ConvDownBlocks.  No gradient reaches
    `face_tex` (the frame computes it under no_grad): a `face_tex` that requires grad is refused."""

    def __init__(self, noise_std, assets, n_embs=256, uv_size=512, logvar_scale=0.1, n_vert_in=7306 * 3,
                 prefix="face_"):
        super().__init__()
        if uv_size != 512:
            raise ValueError("FaceEncoder: uv_size must be 512 (got %s)" % uv_size)
        self.noise_std, self.n_embs, self.logvar_scale = noise_std, n_embs, logvar_scale
        self.prefix, self.uv_size = prefix, uv_size
        mask = torch.as_tensor(np.asarray(mv._get(assets, "mugsy_face_mask"))[..., 0], dtype=torch.float32)
        self.register_buffer("tex_cond_mask", F.interpolate(mask[None, None], (uv_size, uv_size), mode="bilinear",
                                                            align_corners=True))
        self.conv_blocks = tnn.Sequential(ConvDownBlock(3, 4, 512), ConvDownBlock(4, 8, 256),
                                          ConvDownBlock(8, 16, 128), ConvDownBlock(16, 32, 64),
                                          ConvDownBlock(32, 64, 32), ConvDownBlock(64, 128, 16),
                                          ConvDownBlock(128, 128, 8))
        self.geommod = tnn.Sequential(LinearWN(n_vert_in, 256), tnn.LeakyReLU(0.2, inplace=True))
        self.jointmod = tnn.Sequential(LinearWN(256 + 128 * 4 * 4, 512), tnn.LeakyReLU(0.2, inplace=True))
        self.mu = LinearWN(512, n_embs)
        self.logvar = LinearWN(512, n_embs)
        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.mu, 1.0)
        glorot(self.logvar, 1.0)

    def forward(self, face_geom, face_tex, **kwargs):
        for t, n in ((face_geom, "face_geom"), (face_tex, "face_tex")):
            if not t.is_cuda:
                raise RuntimeError("FaceEncoder runs on CUDA only (no CPU fallback): %s is on %s" % (n, t.device))
        if torch.is_grad_enabled() and face_tex.requires_grad:
            raise RuntimeError("FaceEncoder: the texture conditioning has no backward, and face_tex requires grad")
        B = face_geom.shape[0]
        tex_cond = face_tex_cond(face_tex, self.tex_cond_mask)
        tex_enc = self.conv_blocks(tex_cond).reshape(B, 4 * 4 * 128)
        geom_enc = self.geommod(face_geom.reshape(B, -1))
        x = self.jointmod(torch.cat([tex_enc, geom_enc], dim=1))
        embs_mu = self.mu(x)
        embs_logvar = self.logvar_scale * self.logvar(x)
        if self.training:
            embs = embs_mu + torch.exp(embs_logvar) * torch.randn_like(embs_mu) * self.noise_std
        else:
            embs = embs_mu.clone()
        preds = {"embs": embs, "embs_mu": embs_mu, "embs_logvar": embs_logvar, "tex_cond": tex_cond}
        return {self.prefix + k: v for k, v in preds.items()}


class AutoEncoder(tnn.Module):
    """mesh_vae_drivable.AutoEncoder (mesh_vae_drivable.py:71-384) with the reference's constructor, state-dict keys
    and output keys (including `face_tex_cond` and the nested `face_dec_preds` dict).  `assets` carries the
    reference's assets (`lbs_template_verts`, `lbs_scale`, `tex_mean`, `ao_mean`, `mugsy_face_mask`,
    `face_frontal_view`, ...) and, as for `mesh_vae.AutoEncoder`, the four UV images of `geo_fn`.
    `decoder_face["ckpt"]`, when given, is loaded into the face decoder with strict=False, as the reference does; the
    caller's dict is not modified.

    The shadow follows the reference: in training with `pose_to_shadow`, the ShadowUNet's map plus
    `pose_shadow_map`; in eval with `pose_to_shadow`, the pose alone (`ao` may be None); otherwise the ShadowUNet.

    Render: the reference renders through pytorch3d (render_pytorch3d.RenderLayer), which this project does not
    restate; `rgb` here is `mesh_render.RenderLayer`'s `render` with edge_grad=False (pytorch3d's rasteriser has no
    visibility gradient either).  The two differ in pytorch3d's pixel centres, TexturesUV's align_corners=True
    border sampling, and its vertical flip of the UVs (which cancels against flip_uvs=False).  The `renderer.image_size`
    key is the same, so checkpoints load strictly.

    forward() runs on CUDA only and issues no host synchronisation after the first call.  `encode=False` raises (the
    reference leaves face_embs_body unbound there), as do `pixel_cal` without `cal`, and `learn_blur` or `pixel_cal`
    without `renderer` (the reference fails later on the missing `rgb`).  As in mesh_vae.AutoEncoder,
    `preds["shadow_map"]` is the shadow net's map, not the copy forward_tex impaints in place."""

    forward_tex = mv.TextureComposer.forward
    _check = mv.TextureComposer._check

    def __init__(self, encoder, decoder, decoder_view, encoder_face, decoder_face, shadow_net, upscale_net, assets,
                 pose_to_shadow=None, renderer=None, cal=None, pixel_cal=None, learn_blur: bool = True):
        super().__init__()
        from .lbs import LBSModule
        from .shadow import PoseToShadow, ShadowUNet

        _get = mv._get
        if pixel_cal is not None and cal is None:
            raise ValueError("AutoEncoder: pixel_cal needs cal (its camera indices are cal's)")
        if renderer is None and (learn_blur or pixel_cal is not None):
            raise ValueError("AutoEncoder: learn_blur and pixel_cal act on the rendered rgb, and there is no renderer")
        self.geo_fn, uv = mv._uv_geometry(assets)
        self.lbs_fn = LBSModule(_get(assets, "lbs_model_json"), _get(assets, "lbs_config_dict"),
                                _get(assets, "lbs_template_verts"), _get(assets, "lbs_scale"),
                                _get(assets, "global_scaling"))
        self.seam_sampler = SeamSampler(_get(assets, "seam_data_1024"))
        self.seam_sampler_2k = SeamSampler(_get(assets, "seam_data_2048"))

        tex_mean = mv._gaussian_blur(torch.as_tensor(np.asarray(_get(assets, "tex_mean")), dtype=torch.float32)[None],
                                     kernel_size=11)
        self.register_buffer("tex_mean", F.interpolate(tex_mean, (2048, 2048), mode="bilinear"))
        tex_var = _get(assets, "tex_var")
        self.tex_std = tex_var if tex_var is not None else 64.0

        self.register_buffer("face_cond_mask", torch.as_tensor(
            np.asarray(_get(assets, "face_cond_mask")), dtype=torch.float32)[None, None])
        meye = mv._values_to_uv_cpu(torch.as_tensor(np.asarray(_get(assets, "mouth_eyes_mask_geom"))[None, :, None]),
                                    uv["index_image"], uv["bary_image"])
        self.register_buffer("meye_mask", F.interpolate(meye, (2048, 2048), mode="bilinear"))

        self.decoder = ConvDecoder(geo_fn=self.geo_fn, seam_sampler=self.seam_sampler, **decoder, assets=assets)
        self.encoder = Encoder(geo_fn=self.geo_fn, mask=1.0 - np.asarray(_get(assets, "face_mask")), **encoder)
        self.encoder_face = FaceEncoder(assets=assets, **encoder_face)
        decoder_face = dict(decoder_face)
        ckpt = decoder_face.pop("ckpt", None)
        self.decoder_face = FaceDecoderFrontal(assets=assets, **decoder_face)
        if ckpt is not None:
            self.decoder_face.load_state_dict(torch.load(ckpt, map_location="cpu"), strict=False)
        self.decoder_view = mv.UNetViewDecoder(self.geo_fn, seam_sampler=self.seam_sampler, **decoder_view)
        self.shadow_net = ShadowUNet(ao_mean=_get(assets, "ao_mean"), interp_mode="bilinear", biases=False,
                                     **shadow_net)
        self.pose_to_shadow_enabled = pose_to_shadow is not None
        if self.pose_to_shadow_enabled:
            self.pose_to_shadow = PoseToShadow(**pose_to_shadow)
        self.upscale_net = mv.UpscaleNet(in_channels=6, size=1024, upscale_factor=2, out_channels=3, **upscale_net)
        mv._image_stages(self, _get(assets, "camera_ids"), renderer, cal, pixel_cal, learn_blur)

    def encode(self, geom, lbs_motion, face_embs_hqlp):
        """mesh_vae_drivable.py:265-285: the body code from the unposed registration, the face code in body space
        from the frozen face decoder's output"""
        with torch.no_grad():
            verts_unposed = self.lbs_fn.unpose(geom, lbs_motion)
        enc_preds = self.encoder(motion=lbs_motion, verts_unposed=verts_unposed)
        with torch.no_grad():
            face_dec_preds = self.decoder_face(face_embs_hqlp)
        enc_face_preds = self.encoder_face(**face_dec_preds)
        return {**enc_preds, **enc_face_preds, "face_dec_preds": face_dec_preds}

    def forward(self, lbs_motion, campos, geom=None, ao=None, K=None, Rt=None, image_bg=None, image=None,
                image_mask=None, embs=None, _index=None, face_embs=None, embs_conv=None, tex_seg=None, encode=True,
                iteration=None, **kwargs):
        if not encode:
            raise ValueError("AutoEncoder.forward: encode=False is not supported (the reference leaves "
                             "face_embs_body unbound on that path)")
        enc_preds = self.encode(geom, lbs_motion, face_embs)
        dec_preds = self.decoder(motion=lbs_motion, embs=enc_preds["embs"], face_embs=enc_preds["face_embs"],
                                 embs_conv=embs_conv)
        geom_rec = self.lbs_fn.pose(dec_preds["geom_delta_rec"], lbs_motion)
        dec_view_preds = self.decoder_view(geom_rec=geom_rec, tex_mean_rec=dec_preds["tex_mean_rec"],
                                           camera_pos=campos)
        if self.training and self.pose_to_shadow_enabled:
            shadow_preds = self.shadow_net(ao_map=ao)
            shadow_preds["pose_shadow_map"] = self.pose_to_shadow(lbs_motion)["shadow_map"]
        elif self.pose_to_shadow_enabled:
            shadow_preds = self.pose_to_shadow(lbs_motion)
        else:
            shadow_preds = self.shadow_net(ao_map=ao)
        tex_rec = self.forward_tex(dec_preds["tex_mean_rec"], dec_view_preds["tex_view_rec"],
                                   shadow_preds["shadow_map"])
        cam_idxs = None
        if self.cal_enabled:
            cam_idxs = self.cal.name_to_idx(_index["camera"])
            tex_rec = self.cal(tex_rec, cam_idxs)
        preds = {"geom": geom_rec, "tex_rec": tex_rec, **dec_preds, **shadow_preds, **dec_view_preds, **enc_preds}
        if self.rendering_enabled:
            preds.update(rgb=self.renderer(geom_rec, tex_rec, K=K, Rt=Rt, edge_grad=False)["render"])
        if self.learn_blur_enabled:
            preds["rgb"] = self.learn_blur(preds["rgb"], _index["camera"])
            preds["learn_blur_weights"] = self.learn_blur.reg(_index["camera"])
        if self.pixel_cal_enabled:
            preds["rgb"] = self.pixel_cal(cam_idxs, preds["rgb"])
        return preds
