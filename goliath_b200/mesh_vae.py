"""The body decoder `mesh_vae.ConvDecoder` (ca_code/models/mesh_vae.py:439-630) on the GPU: every `UpConvBlockDeep`
(the 8-64^2 `embs` / `face_embs` branches with groups = 1 and the 128^2-1024^2 trunk with groups = 2) runs on the
fused upsample + grouped weight-normalised convolution kernels of csrc/upconv_wnub.cu, the two 64^2 `ConvBlock`s and the
final 4 -> 3 convolutions on the stride-1 kernels (csrc/conv_wnub.cu, and a channel-slice variant so the final
convolutions read their halves of the 8-channel map in place), the seam sampler and `from_uv` on the gathers of
`goliath_b200.seams` when the caller passes this library's `SeamSampler` / `GeometryModule`.

Constructor, parameter names and shapes, buffers and the Glorot initialisation are the reference's, so a checkpoint of
the reference class loads with strict=True.  `geo_fn` and `seam_sampler` are duck-typed as in the reference: any object
with `from_uv`, and `impaint` / `resample`.  The small pieces stay in torch: the LinearWN layers, tile2d x mask, the
face / body merge and the concatenations.  Forward and backward are free of host synchronisation; CPU tensors raise.

The encoders `mesh_vae.Encoder` / `FaceEncoder` (mesh_vae.py:344-436) run on the fused `ConvDownBlock` kernels of
csrc/downconv_wnub.cu, the first block building its resized, masked input inside its kernels; `encode` is
`AutoEncoder.encode` (mesh_vae.py:230-239) as a function over the LBS module, the geometry module and the encoders.

`AutoEncoder` (mesh_vae.py:72-341) runs the whole frame on these stages with the reference's constructor and keys, and
finishes the render with the depth-discontinuity mask and `CameraPixelBias` on csrc/body_frame.cu."""
import numpy as np
import torch
import torch.nn as tnn
import torch.nn.functional as F
from torch.autograd import Function

from . import _lib
from .geom import depth_discontuity_mask
from .nn import (ConvBlock, ConvDownBlock, Conv2dWNUB, FusedLeakyReLU, LinearWN, UpConvBlockDeep, _wn_chain,
                 _wn_scale, glorot, tile2d)
from .seams import SeamSampler
from .unet import UNetWB


class _ConvSlices(Function):
    """verts_conv on channels [0,c) and tex_conv on channels [c,2c) of x [B,2c,H,W] (mesh_vae.py:615-621), read in
    place; the backward writes both halves of one gx."""

    @staticmethod
    def forward(ctx, x, va, ga, ba, vb, gb, bb):
        x = x.contiguous()
        _lib.check_input(x, "input")
        B, C2, H, W = x.shape
        c, Cout = va.shape[1], va.shape[0]
        if C2 != 2 * c or vb.shape != va.shape or va.shape[2:] != (3, 3):
            raise RuntimeError("the final convolutions need a [B, %d, H, W] map" % (2 * va.shape[1]))
        outs = []
        with torch.cuda.device(x.device):
            for i, (v, g, b) in enumerate(((va, ga, ba), (vb, gb, bb))):
                out = torch.empty(B, Cout, H, W, device=x.device)
                _lib.check(_lib.lib().gb_conv3x3_ub_slice_fwd(
                    B, c, Cout, H, W, x.data_ptr() + 4 * i * c * H * W, C2 * H * W, _lib.ptr(v.contiguous()),
                    _lib.ptr(_wn_scale(v, g)), _lib.ptr(b.contiguous()), _lib.ptr(out), _lib.stream_ptr(x.device)),
                    "conv3x3_ub_slice_fwd")
                outs.append(out)
        ctx.save_for_backward(x, va, ga, vb, gb)
        return tuple(outs)

    @staticmethod
    def backward(ctx, g_a, g_b):
        x, va, ga, vb, gb = ctx.saved_tensors
        B, C2, H, W = x.shape
        c, Cout = va.shape[1], va.shape[0]
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        grads = []
        with torch.cuda.device(x.device):
            for i, (v, g, go) in enumerate(((va, ga, g_a), (vb, gb, g_b))):
                gbias = torch.empty(Cout, H, W, device=x.device)
                gw = torch.zeros_like(v)
                _lib.check(_lib.lib().gb_conv3x3_ub_slice_bwd(
                    B, c, Cout, H, W, x.data_ptr() + 4 * i * c * H * W, C2 * H * W, _lib.ptr(v.contiguous()),
                    _lib.ptr(_wn_scale(v, g)), _lib.ptr(go.contiguous()), _lib.ptr(gbias),
                    None if gx is None else gx.data_ptr() + 4 * i * c * H * W, _lib.ptr(gw),
                    _lib.stream_ptr(x.device)), "conv3x3_ub_slice_bwd")
                grads += list(_wn_chain(v, g, gw)) + [gbias]
        return (gx, *grads)


def _asset(assets, name):
    return assets[name] if isinstance(assets, dict) else getattr(assets, name)


class ConvDecoder(tnn.Module):
    """mesh_vae.py:439-630.  `assets` carries pose_cond_mask [P,S,S], head_cond_mask, face_cond_mask and
    body_cond_mask [S,S] (S = init_uv_size) as attributes or dict keys."""

    def __init__(self, geo_fn, uv_size, seam_sampler, init_uv_size, n_pose_dims, n_pose_enc_channels, n_embs,
                 n_embs_enc_channels, n_face_embs, n_init_channels, n_min_channels, assets, tex_scale: float = 0.001,
                 verts_scale: float = 0.01):
        super().__init__()
        self.geo_fn = geo_fn
        self.tex_scale, self.verts_scale = tex_scale, verts_scale
        self.uv_size, self.init_uv_size = uv_size, init_uv_size
        self.n_pose_dims, self.n_pose_enc_channels = n_pose_dims, n_pose_enc_channels
        self.n_embs, self.n_embs_enc_channels, self.n_face_embs = n_embs, n_embs_enc_channels, n_face_embs
        self.n_blocks = int(np.log2(uv_size // init_uv_size))
        self.sizes = [init_uv_size * 2 ** s for s in range(self.n_blocks + 1)]
        self.n_channels = [max(n_init_channels // 2 ** b, n_min_channels) for b in range(self.n_blocks + 1)]

        self.local_pose_conv_block = ConvBlock(n_pose_dims, n_pose_enc_channels, init_uv_size, kernel_size=1,
                                               padding=0)
        self.embs_fc = tnn.Sequential(LinearWN(n_embs, 4 * 4 * 128), tnn.LeakyReLU(0.2, inplace=True))
        self.embs_conv_block = tnn.Sequential(UpConvBlockDeep(128, 128, 8), UpConvBlockDeep(128, 128, 16),
                                              UpConvBlockDeep(128, 64, 32),
                                              UpConvBlockDeep(64, n_embs_enc_channels, 64))
        self.face_embs_fc = tnn.Sequential(LinearWN(n_face_embs, 4 * 4 * 32), tnn.LeakyReLU(0.2, inplace=True))
        self.face_embs_conv_block = tnn.Sequential(UpConvBlockDeep(32, 64, 8), UpConvBlockDeep(64, 64, 16),
                                                   UpConvBlockDeep(64, n_embs_enc_channels, 32))
        n_groups = 2
        self.joint_conv_block = ConvBlock(n_pose_enc_channels + n_embs_enc_channels, n_init_channels, init_uv_size)
        self.conv_blocks = tnn.ModuleList([
            UpConvBlockDeep(self.n_channels[b] * n_groups, self.n_channels[b + 1] * n_groups, self.sizes[b + 1],
                            groups=n_groups) for b in range(self.n_blocks)])
        self.verts_conv = Conv2dWNUB(self.n_channels[-1], 3, uv_size, uv_size, 3, 1, 1)
        self.tex_conv = Conv2dWNUB(self.n_channels[-1], 3, uv_size, uv_size, 3, 1, 1)

        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.verts_conv, 1.0)
        glorot(self.tex_conv, 1.0)
        self.seam_sampler = seam_sampler

        f32 = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float32)
        # mesh_vae.py:560-575: the head region is removed from the pose condition
        self.register_buffer("pose_cond_mask", (f32(_asset(assets, "pose_cond_mask"))[None]
                                                * (1 - f32(_asset(assets, "head_cond_mask"))[None, None])).to(torch.int32))
        self.register_buffer("face_cond_mask", f32(_asset(assets, "face_cond_mask"))[None, None])
        self.register_buffer("body_cond_mask", f32(_asset(assets, "body_cond_mask"))[None, None])

    def forward(self, pose, embs, face_embs, embs_conv=None):
        """`embs_conv` [B, n_embs_enc_channels, S, S], when given, replaces the decoded `embs` map (as in
        mesh_vae_drivable.py:614-615); the face merge is written into a copy, never into the caller's tensor."""
        for t, n in ((pose, "pose"), (embs if embs_conv is None else embs_conv, "embs"), (face_embs, "face_embs")):
            if not t.is_cuda:
                raise RuntimeError("ConvDecoder runs on CUDA only (no CPU fallback): %s is on %s" % (n, t.device))
        B = pose.shape[0]
        local_pose = pose[:, 6:]
        non_head_mask = (self.body_cond_mask * (1.0 - self.face_cond_mask)).clip(0.0, 1.0)
        pose_masked = tile2d(local_pose, self.init_uv_size) * self.pose_cond_mask
        pose_conv = self.local_pose_conv_block(pose_masked) * non_head_mask
        if embs_conv is None:
            embs_conv = self.embs_conv_block(self.embs_fc(embs).reshape(B, 128, 4, 4))
        else:
            embs_conv = embs_conv.clone()
        face_conv = self.face_embs_conv_block(self.face_embs_fc(face_embs).reshape(B, 32, 4, 4))
        # merging embeddings with spatial masks
        embs_conv[:, :, 32:, :32] = (face_conv * self.face_cond_mask[:, :, 32:, :32]
                                     + embs_conv[:, :, 32:, :32] * non_head_mask[:, :, 32:, :32])
        joint = self.joint_conv_block(torch.cat([pose_conv, embs_conv], 1))
        x = torch.cat([joint, joint], 1)
        for blk in self.conv_blocks:
            x = blk(x)
        x = self.seam_sampler.impaint(x)
        x = self.seam_sampler.resample(x)
        x = self.seam_sampler.resample(x)
        vc, tc = self.verts_conv, self.tex_conv
        verts_uv, tex = _ConvSlices.apply(x, vc.weight_v, vc.weight_g, vc.bias, tc.weight_v, tc.weight_g, tc.bias)
        verts_uv_delta_rec = verts_uv * self.verts_scale
        return {"geom_delta_rec": self.geo_fn.from_uv(verts_uv_delta_rec), "geom_uv_delta_rec": verts_uv_delta_rec,
                "tex_mean_rec": tex * self.tex_scale, "embs_conv": embs_conv, "pose_conv": pose_conv}


class UNetViewDecoder(tnn.Module):
    """mesh_vae.py:633-649.  `geo_fn` carries `vi` [F,3], `index_image` [S,S,3] and `bary_image` [S,S,3] (a
    `goliath_b200.geom.GeometryModule`); the view cosine (compute_view_cos + values_to_uv, geom.py:308-352, zero at
    uncovered texels) runs under no_grad on `hand_mvp.view_cos_uv`, the U-Net on `goliath_b200.unet.UNetWB`."""

    def __init__(self, geo_fn, net_uv_size, seam_sampler, n_init_ftrs=8):
        super().__init__()
        self.geo_fn = geo_fn
        self.net_uv_size = net_uv_size
        self.unet = UNetWB(4, 3, n_init_ftrs=n_init_ftrs, size=net_uv_size)
        self.register_buffer("faces", geo_fn.vi.to(torch.int64), persistent=False)

    def forward(self, geom_rec, tex_mean_rec, camera_pos):
        from .hand_mvp import view_cos_uv

        with torch.no_grad():
            vc = view_cos_uv(geom_rec, self.geo_fn.vi, camera_pos, self.geo_fn.index_image, self.geo_fn.bary_image)
        cond_view = torch.cat([vc, tex_mean_rec], dim=1)
        return {"tex_view_rec": self.unet(cond_view), "cond_view": cond_view}


class UpscaleNet(tnn.Module):
    """mesh_vae.py:652-678: conv_block (3x3 Conv2dWNUB + LeakyReLU, fused) and the 1x1 untied-bias out_block on the
    stride-1 kernels, then torch's pixel_shuffle.  Inside `TextureComposer` the out_block and the pixel shuffle run in
    the composite kernel instead."""

    def __init__(self, in_channels, out_channels, n_ftrs, size=1024, upscale_factor=2):
        super().__init__()
        conv = Conv2dWNUB(in_channels, n_ftrs, size, size, kernel_size=3, padding=1)
        conv.fused_slope = 0.2
        self.conv_block = tnn.Sequential(conv, FusedLeakyReLU())
        self.out_block = Conv2dWNUB(n_ftrs, out_channels * upscale_factor ** 2, size, size, kernel_size=1, padding=0)
        self.pixel_shuffle = tnn.PixelShuffle(upscale_factor=upscale_factor)
        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.out_block, 1.0)

    def forward(self, x):
        if not x.is_cuda:
            raise RuntimeError("UpscaleNet runs on CUDA only (no CPU fallback): the input is on %s" % x.device)
        return self.pixel_shuffle(self.out_block(self.conv_block(x)))


class _TexCompose(Function):
    """P = ((U(T1) + PS(out_block(h))) * tex_std + tex_mean) * S3 on csrc/body_tex.cu (mesh_vae.py:211-222 with
    mesh_vae.py:670-678); the backward recomputes the pre-shadow texture."""

    @staticmethod
    def forward(ctx, t1, h, v, g, bias, tex_mean, s3, tex_std):
        t1, h, s3 = t1.contiguous(), h.contiguous(), s3.contiguous()
        v2, bias = v.reshape(v.shape[0], -1).contiguous(), bias.contiguous()
        tex_mean = tex_mean.contiguous()
        for t, n in ((t1, "T1"), (h, "h"), (v2, "out_block.weight_v"), (bias, "out_block.bias"),
                     (tex_mean, "tex_mean"), (s3, "shadow map")):
            _lib.check_input(t, n)
        B, C, H, W = t1.shape
        if (C != 3 or h.shape != (B, 4, H, W) or v2.shape != (12, 4) or bias.shape != (12, H, W)
                or tex_mean.shape != (1, 3, 2 * H, 2 * W) or s3.shape != (B, 1, 2 * H, 2 * W)):
            raise RuntimeError("texture composite: shapes do not match T1 %s" % (tuple(t1.shape),))
        scale = _wn_scale(v, g)
        out = torch.empty(B, 3, 2 * H, 2 * W, device=t1.device)
        with torch.cuda.device(t1.device):
            _lib.check(_lib.lib().gb_body_tex_compose_fwd(
                B, H, W, _lib.ptr(t1), _lib.ptr(h), _lib.ptr(v2), _lib.ptr(scale), _lib.ptr(bias), float(tex_std),
                _lib.ptr(tex_mean), _lib.ptr(s3), _lib.ptr(out), _lib.stream_ptr(t1.device)), "body_tex_compose_fwd")
        ctx.save_for_backward(t1, h, v, g, bias, tex_mean, s3)
        ctx.tex_std = float(tex_std)
        return out

    @staticmethod
    def backward(ctx, g_out):
        t1, h, v, g, bias, tex_mean, s3 = ctx.saved_tensors
        B, _, H, W = t1.shape
        dev = t1.device
        g_out = g_out.contiguous()
        scale = _wn_scale(v, g)
        g_t1, g_h, g_s3 = torch.empty_like(t1), torch.empty_like(h), torch.empty_like(s3)
        g_bias = torch.empty_like(bias)
        g_w = torch.zeros_like(v)
        L = _lib.lib()
        ws = torch.empty(L.gb_body_tex_compose_workspace_bytes(H, W) // 4, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.gb_body_tex_compose_bwd(
                B, H, W, _lib.ptr(t1), _lib.ptr(h), _lib.ptr(v.reshape(v.shape[0], -1).contiguous()),
                _lib.ptr(scale), _lib.ptr(bias), ctx.tex_std, _lib.ptr(tex_mean), _lib.ptr(s3), _lib.ptr(g_out),
                _lib.ptr(g_t1), _lib.ptr(g_h), _lib.ptr(g_bias), _lib.ptr(g_w), _lib.ptr(g_s3), _lib.ptr(ws),
                _lib.stream_ptr(dev)), "body_tex_compose_bwd")
        gv, gg = _wn_chain(v, g, g_w)
        return g_t1, g_h, gv, gg, g_bias, None, g_s3, None


class TextureComposer(tnn.Module):
    """mesh_vae.AutoEncoder.forward_tex (mesh_vae.py:204-228) with the `upscale_net`, `seam_sampler`,
    `seam_sampler_2k` and `tex_mean` [1,3,2S,2S] of the reference's AutoEncoder under the same key names, so that
    subset of an AutoEncoder checkpoint loads strictly.  `tex_mean` is passed in prepared (the blur and resize of the
    asset's colour mean is one-off asset preparation); `tex_std` is a float as in the reference.

    forward(tex_mean_rec [B,3,S,S], tex_view_rec [B,3,S,S], shadow_map [B,1,2S,2S]) -> tex_rec [B,3,2S,2S]:
      T1 = seam_sampler(tex_mean_rec + tex_view_rec)                 (impaint + resample, one gather)
      h  = upscale_net.conv_block(cat(tex_mean_rec, tex_view_rec))
      S3 = seam_sampler_2k.resample(seam_sampler_2k(shadow_map))
      P  = ((U(T1) + PS(out_block(h))) * tex_std + tex_mean) * S3     (csrc/body_tex.cu, one kernel)
      tex_rec = seam_sampler_2k.resample(seam_sampler_2k(P))
    Unlike the reference, whose impaint writes into the caller's shadow_map through a view, the inputs are left as they
    are; the gradients are the same."""

    def __init__(self, seam_sampler, seam_sampler_2k, tex_mean, tex_std=64.0, n_ftrs=4):
        super().__init__()
        for sampler in (seam_sampler, seam_sampler_2k):
            if not isinstance(sampler, SeamSampler):
                raise TypeError("TextureComposer needs goliath_b200.seams.SeamSampler instances")
        self.upscale_net = UpscaleNet(in_channels=6, out_channels=3, n_ftrs=n_ftrs, size=1024, upscale_factor=2)
        self.seam_sampler = seam_sampler
        self.seam_sampler_2k = seam_sampler_2k
        self.register_buffer("tex_mean", torch.as_tensor(tex_mean, dtype=torch.float32))
        self.tex_std = tex_std
        if self.tex_mean.dim() != 4 or tuple(self.tex_mean.shape[:2]) != (1, 3):
            raise ValueError("tex_mean must be [1, 3, 2S, 2S] (got %s)" % (tuple(self.tex_mean.shape),))

    def _check(self, tex_mean_rec, tex_view_rec, shadow_map):
        """tex_mean must be twice the size of tex_mean_rec, and each sampler built for the maps it receives"""
        S = tex_mean_rec.shape[-1]
        size2 = tuple(self.tex_mean.shape[2:])
        if (tex_mean_rec.shape[-2:] != (S, S) or tex_view_rec.shape != tex_mean_rec.shape
                or size2 != (2 * S, 2 * S) or shadow_map.shape[-2:] != size2):
            raise RuntimeError("TextureComposer: tex_mean %s must be twice the size of tex_mean_rec %s, and the "
                               "shadow map %s of tex_mean's size" % (tuple(self.tex_mean.shape),
                                                                     tuple(tex_mean_rec.shape),
                                                                     tuple(shadow_map.shape)))
        for sampler, size, n in ((self.seam_sampler, (S, S), "seam_sampler"),
                                 (self.seam_sampler_2k, size2, "seam_sampler_2k")):
            got = tuple(sampler.uvs.shape[:2])
            if got != size:
                raise RuntimeError("%s was built for %s maps, it receives %s" % (n, got, size))

    def forward(self, tex_mean_rec, tex_view_rec, shadow_map):
        for t, n in ((tex_mean_rec, "tex_mean_rec"), (tex_view_rec, "tex_view_rec"), (shadow_map, "shadow_map")):
            if not t.is_cuda:
                raise RuntimeError("TextureComposer runs on CUDA only (no CPU fallback): %s is on %s" % (n, t.device))
        self._check(tex_mean_rec, tex_view_rec, shadow_map)
        t1 = self.seam_sampler(tex_mean_rec + tex_view_rec)
        h = self.upscale_net.conv_block(torch.cat([tex_mean_rec, tex_view_rec], dim=1))
        s3 = self.seam_sampler_2k.resample(self.seam_sampler_2k(shadow_map))
        ob = self.upscale_net.out_block
        p = _TexCompose.apply(t1, h, ob.weight_v, ob.weight_g, ob.bias, self.tex_mean, s3, self.tex_std)
        return self.seam_sampler_2k.resample(self.seam_sampler_2k(p))


class Encoder(tnn.Module):
    """mesh_vae.py:344-421: seven ConvDownBlocks (3 -> 8 @ 512 ... 128 -> 128 @ 8) and two LinearWN heads.  The input
    conditioning `verts_scale * bilinear(verts_unposed_uv -> 512^2) * mask` (align_corners=False) is evaluated inside
    the first block's kernels, for any input size and for a strided window of a larger map, so neither the resized map
    nor a crop is written.  `encode` computes verts_unposed_uv under no_grad, so no gradient flows to it: an input
    that requires grad is refused.  The reparameterisation noise is torch's randn_like, drawn as the reference
    draws it."""

    def __init__(self, n_embs: int, mask, noise_std: float = 1.0, mean_scale: float = 0.1, logvar_scale: float = 0.1,
                 verts_scale: float = 1.0):
        super().__init__()
        self.noise_std, self.n_embs = noise_std, n_embs
        self.mean_scale, self.logvar_scale, self.verts_scale = mean_scale, logvar_scale, verts_scale
        self.verts_conv = ConvDownBlock(3, 8, 512)
        if len(mask.shape) != 2:
            raise ValueError("mask must be [H, W] (got %s)" % (tuple(mask.shape),))
        mask = torch.as_tensor(mask[np.newaxis, np.newaxis], dtype=torch.float32)
        self.register_buffer("mask", F.interpolate(mask, size=(512, 512), mode="bilinear").to(torch.bool))
        self.joint_conv_blocks = tnn.Sequential(ConvDownBlock(8, 16, 256), ConvDownBlock(16, 32, 128),
                                                ConvDownBlock(32, 32, 64), ConvDownBlock(32, 64, 32),
                                                ConvDownBlock(64, 128, 16), ConvDownBlock(128, 128, 8))
        self.mu = LinearWN(4 * 4 * 128, n_embs)
        self.logvar = LinearWN(4 * 4 * 128, n_embs)
        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.mu, 1.0)
        glorot(self.logvar, 1.0)

    def forward(self, verts_unposed_uv):
        if not verts_unposed_uv.is_cuda:
            raise RuntimeError("Encoder runs on CUDA only (no CPU fallback): verts_unposed_uv is on %s"
                               % verts_unposed_uv.device)
        if verts_unposed_uv.dim() != 4 or verts_unposed_uv.shape[1] != 3:
            raise RuntimeError("verts_unposed_uv must be [B, 3, H, W] (got %s)" % (tuple(verts_unposed_uv.shape),))
        B = verts_unposed_uv.shape[0]
        x = self.verts_conv(verts_unposed_uv, resize_mask=self.mask, scale=self.verts_scale)
        x = self.joint_conv_blocks(x).reshape(B, -1)
        embs_mu = self.mean_scale * self.mu(x)
        embs_logvar = self.logvar_scale * self.logvar(x)
        if self.training:
            embs = embs_mu + torch.exp(embs_logvar) * torch.randn_like(embs_mu) * self.noise_std
        else:
            embs = embs_mu.clone()
        return {"embs": embs, "embs_mu": embs_mu, "embs_logvar": embs_logvar}


class FaceEncoder(tnn.Module):
    """mesh_vae.py:424-436: an `Encoder` on the [512:, :512] window of the UV position map, read in place."""

    def __init__(self, mask, **kwargs):
        super().__init__()
        if len(mask.shape) != 2 or mask.shape[0] <= 512:
            raise ValueError("mask must be [H, W] with H > 512 (got %s)" % (tuple(mask.shape),))
        self.encoder = Encoder(**kwargs, mask=mask[512:, :512])

    def forward(self, verts_unposed_uv):
        if verts_unposed_uv.dim() != 4 or verts_unposed_uv.shape[2] <= 512:
            raise RuntimeError("verts_unposed_uv must be [B, 3, H, W] with H > 512 (got %s)"
                               % (tuple(verts_unposed_uv.shape),))
        preds = self.encoder(verts_unposed_uv[:, :, 512:, :512])
        return {"face_" + k: v for k, v in preds.items()}


def encode(lbs_fn, geo_fn, encoder, encoder_face, registration_vertices, pose):
    """mesh_vae.AutoEncoder.encode (mesh_vae.py:230-239): unpose the registered vertices and lay them out in UV under
    no_grad, then both encoders; returns the merged dict (embs*, face_embs*).  One stream, no host synchronisation."""
    with torch.no_grad():
        verts_unposed = lbs_fn.unpose(registration_vertices, pose)
        verts_unposed_uv = geo_fn.to_uv(verts_unposed)
    return {**encoder(verts_unposed_uv), **encoder_face(verts_unposed_uv)}


class _PixelBias(Function):
    """rgb + bilinear(bias[idx]) on csrc/body_frame.cu; the bias gradient is a fixed-order gather per texel"""

    @staticmethod
    def forward(ctx, rgb, bias, idx):
        rgb, bias, idx = rgb.contiguous(), bias.contiguous(), idx.contiguous()
        _lib.check_input(rgb, "rgb")
        _lib.check_input(bias, "bias")
        _lib.check_input(idx, "camera indices", torch.int64)
        B, C, H, W = rgb.shape
        if bias.dim() != 4 or bias.shape[1] != 1 or idx.shape != (B,):
            raise RuntimeError("pixel bias: bias must be [n_cams,1,h,w] and the indices [B] (got %s, %s)"
                               % (tuple(bias.shape), tuple(idx.shape)))
        out = torch.empty_like(rgb)
        n, _, Hb, Wb = bias.shape
        with torch.cuda.device(rgb.device):
            _lib.check(_lib.lib().gb_pixel_bias_fwd(B, C, H, W, n, Hb, Wb, _lib.ptr(rgb), _lib.ptr(bias), _lib.ptr(idx),
                                                    _lib.ptr(out), _lib.stream_ptr(rgb.device)), "pixel_bias_fwd")
        ctx.save_for_backward(idx)
        ctx.shapes = (tuple(rgb.shape), tuple(bias.shape))
        return out

    @staticmethod
    def backward(ctx, g_out):
        (idx,) = ctx.saved_tensors
        (B, C, H, W), (n, _, Hb, Wb) = ctx.shapes
        g_bias = None
        if ctx.needs_input_grad[1]:
            g_out = g_out.contiguous()
            g_bias = torch.empty(n, 1, Hb, Wb, device=g_out.device)
            with torch.cuda.device(g_out.device):
                _lib.check(_lib.lib().gb_pixel_bias_bwd(B, C, H, W, n, Hb, Wb, _lib.ptr(idx), _lib.ptr(g_out),
                                                        _lib.ptr(g_bias), _lib.stream_ptr(g_out.device)),
                           "pixel_bias_bwd")
        return g_out if ctx.needs_input_grad[0] else None, g_bias, None


class CameraPixelBias(tnn.Module):
    """mesh_vae.py:51-69 with its parameter `bias` [n_cams, 1, image_width // ds_rate, image_height // ds_rate] (width
    and height swapped, as in the reference) stretched to (image_height, image_width) with torch's half-pixel bilinear
    index.  forward(idxs [B] int64, rgb [B,C,H,W]) -> rgb + bias_up in one kernel (mesh_vae.py:335-339); without rgb it
    returns bias_up [B,1,H,W] as the reference's forward does.  Two backward calls give the same bits."""

    def __init__(self, image_height, image_width, cameras, ds_rate) -> None:
        super().__init__()
        self.image_height, self.image_width = image_height, image_width
        self.cameras = cameras
        self.n_cameras = len(cameras)
        self.register_parameter("bias", tnn.Parameter(
            torch.zeros(self.n_cameras, 1, image_width // ds_rate, image_height // ds_rate)))

    def forward(self, idxs: torch.Tensor, rgb: torch.Tensor = None) -> torch.Tensor:
        if rgb is None:
            rgb = torch.zeros(idxs.shape[0], 1, self.image_height, self.image_width, device=self.bias.device)
        if tuple(rgb.shape[2:]) != (self.image_height, self.image_width):
            raise RuntimeError("CameraPixelBias: the image must be %d x %d (got %s)"
                               % (self.image_height, self.image_width, tuple(rgb.shape)))
        return _PixelBias.apply(rgb, self.bias, idxs)


def _gaussian_blur(img, kernel_size):
    """torchvision.transforms.functional.gaussian_blur(img, kernel_size) with its default sigma
    0.3 ((k - 1) 0.5 - 1) + 0.8 and reflect padding, restated in torch (one-off asset preparation on the CPU)"""
    sigma = 0.3 * ((kernel_size - 1) * 0.5 - 1) + 0.8
    half = (kernel_size - 1) * 0.5
    x = torch.linspace(-half, half, steps=kernel_size, dtype=img.dtype)
    k1 = torch.exp(-0.5 * (x / sigma).pow(2))
    k1 = k1 / k1.sum()
    k2 = torch.mm(k1[:, None], k1[None, :]).expand(img.shape[-3], 1, kernel_size, kernel_size)
    p = kernel_size // 2
    return F.conv2d(F.pad(img, [p, p, p, p], mode="reflect"), k2, groups=img.shape[-3])


def _values_to_uv_cpu(values, index_img, bary_img):
    """geom.values_to_uv (geom.py:308-324) in torch, for the constructor's one-off `meye_mask`"""
    index_mask = torch.all(index_img != -1, dim=-1)
    flat = torch.sum(values[:, index_img[index_mask].to(torch.int64)].permute(0, 3, 1, 2)
                     * bary_img[index_mask].to(torch.float32), dim=-1)
    out = torch.zeros(values.shape[0], values.shape[-1], *index_img.shape[:2], dtype=values.dtype)
    out[:, :, index_mask] = flat
    return out


UV_IMAGES = ("index_image", "bary_image", "face_index_image", "valid_mask")


def _get(obj, name, default=None):
    if isinstance(obj, dict):
        return obj.get(name, default)
    return getattr(obj, name, default)


def _uv_geometry(assets, with_v2uv=True, size=1024):
    """the frame's GeometryModule from `assets.topology` and the four UV images the assets must carry at size x size
    (the head's module has no v2uv: with_v2uv=False); returns (geo_fn, {name: image})"""
    from .geom import GeometryModule

    missing = [k for k in UV_IMAGES if _get(assets, k) is None]
    if missing:
        raise ValueError("AutoEncoder: assets must carry the UV images %s at %d x %d (the reference's "
                         "geo_fn.* buffers); missing: %s" % (", ".join(UV_IMAGES), size, size, ", ".join(missing)))
    uv = {k: torch.as_tensor(np.asarray(_get(assets, k))) for k in UV_IMAGES}
    for k, t in uv.items():
        if tuple(t.shape[:2]) != (size, size):
            raise ValueError("AutoEncoder: assets.%s must be %d x %d (got %s)" % (k, size, size, tuple(t.shape)))
    topo = _get(assets, "topology")
    v2uv = _get(topo, "v2uv") if with_v2uv else None
    geo_fn = GeometryModule(_get(topo, "vi"), uv["index_image"], uv["bary_image"], vt=_get(topo, "vt"), v2uv=v2uv,
                            vti=_get(topo, "vti"), face_index_image=uv["face_index_image"],
                            valid_mask=uv["valid_mask"])
    return geo_fn, uv


def _image_stages(model, cameras, renderer, cal, pixel_cal, learn_blur):
    """the frame's optional image-space modules under the reference's names and order: pixel_cal, learn_blur, cal,
    renderer (a RenderLayer over model.geo_fn's topology)"""
    from .mesh_render import RenderLayer
    from .photo_loss import CalV5, LearnableBlur

    model.pixel_cal_enabled = pixel_cal is not None
    if model.pixel_cal_enabled:
        model.pixel_cal = CameraPixelBias(**pixel_cal, cameras=cameras)
    model.learn_blur_enabled = bool(learn_blur)
    if model.learn_blur_enabled:
        model.learn_blur = LearnableBlur(cameras)
    model.cal_enabled = cal is not None
    if model.cal_enabled:
        model.cal = CalV5(**cal, cameras=cameras)
    model.rendering_enabled = renderer is not None
    if model.rendering_enabled:
        model.renderer = RenderLayer(h=_get(renderer, "image_height"), w=_get(renderer, "image_width"),
                                     vt=model.geo_fn.vt, vi=model.geo_fn.vi, vti=model.geo_fn.vti, flip_uvs=False)


class AutoEncoder(tnn.Module):
    """mesh_vae.AutoEncoder (mesh_vae.py:72-341): the body avatar's frame on this project's stages, with the
    reference's constructor and state-dict keys (the shared geometry module and seam sampler repeat under
    `decoder.*` / `decoder_view.*`), so `AutoEncoder(**config.model, assets=assets)` builds from mesh_vae_example.yml
    and a reference checkpoint loads with strict=True.

    `assets` (attributes or dict keys) carries the reference's assets and, because this project does not rasterise
    the UV layout, the four `geo_fn` images a checkpoint stores: index_image / bary_image [1024,1024,3],
    face_index_image [1024,1024] and valid_mask [1024,1024,1].  `tex_mean` (blur + resize of color_mean) and
    `meye_mask` are prepared in torch on the CPU at construction, as the reference's constructor does.

    forward() runs on CUDA only and issues no host synchronisation after the first call (which builds the cached
    gather and render tables).  Unlike the reference, `preds["shadow_map"]` is the shadow net's map, not the copy
    forward_tex impaints in place; `pose_to_shadow`, `encode=False` and `pixel_cal` without `cal` raise."""

    forward_tex = TextureComposer.forward
    _check = TextureComposer._check

    def __init__(self, encoder, encoder_face, decoder, decoder_view, shadow_net, upscale_net, assets,
                 pose_to_shadow=None, renderer=None, cal=None, pixel_cal=None, learn_blur: bool = True):
        super().__init__()
        from .lbs import LBSModule
        from .shadow import ShadowUNet

        if pose_to_shadow is not None:
            raise NotImplementedError("AutoEncoder: pose_to_shadow (PoseToShadow) is not implemented")
        if pixel_cal is not None and cal is None:
            raise ValueError("AutoEncoder: pixel_cal needs cal (its camera indices are cal's)")
        self.geo_fn, uv = _uv_geometry(assets)
        self.lbs_fn = LBSModule(_get(assets, "lbs_model_json"), _get(assets, "lbs_config_dict"),
                                _get(assets, "template_mesh"), _get(assets, "skeleton_scales"),
                                _get(assets, "global_scaling"))
        self.seam_sampler = SeamSampler(_get(assets, "seam_data_1024"))
        self.seam_sampler_2k = SeamSampler(_get(assets, "seam_data_2048"))

        tex_mean = _gaussian_blur(torch.as_tensor(np.asarray(_get(assets, "color_mean")), dtype=torch.float32)[None],
                                  kernel_size=11)
        self.register_buffer("tex_mean", F.interpolate(tex_mean, (2048, 2048), mode="bilinear"))
        tex_var = _get(assets, "tex_var")
        self.tex_std = tex_var if tex_var is not None else 64.0

        self.register_buffer("face_cond_mask", torch.as_tensor(
            np.asarray(_get(assets, "face_cond_mask")), dtype=torch.float32)[None, None])
        meye = _values_to_uv_cpu(torch.as_tensor(np.asarray(_get(assets, "mouth_eyes_mask_geom"))[None, :, None]),
                                 uv["index_image"], uv["bary_image"])
        self.register_buffer("meye_mask", F.interpolate(meye, (2048, 2048), mode="bilinear"))

        self.decoder = ConvDecoder(geo_fn=self.geo_fn, seam_sampler=self.seam_sampler, **decoder, assets=assets)
        face_mask = np.asarray(_get(assets, "face_mask"))
        self.encoder = Encoder(mask=1.0 - face_mask, **encoder)
        self.encoder_face = FaceEncoder(mask=face_mask, **encoder_face)
        self.decoder_view = UNetViewDecoder(self.geo_fn, seam_sampler=self.seam_sampler, **decoder_view)
        self.shadow_net = ShadowUNet(ao_mean=_get(assets, "ambient_occlusion_mean"), interp_mode="bilinear",
                                     biases=False, **shadow_net)
        self.pose_to_shadow_enabled = False
        self.upscale_net = UpscaleNet(in_channels=6, size=1024, upscale_factor=2, out_channels=3, **upscale_net)

        _image_stages(self, _get(assets, "camera_ids"), renderer, cal, pixel_cal, learn_blur)

    def encode(self, registration_vertices, pose):
        return encode(self.lbs_fn, self.geo_fn, self.encoder, self.encoder_face, registration_vertices, pose)

    def forward(self, pose, campos, registration_vertices=None, ambient_occlusion=None, K=None, Rt=None,
                camera_id=None, frame_id=None, embs=None, encode=True, iteration=None, **kwargs):
        if not encode:
            raise ValueError("AutoEncoder.forward: encode=False is not supported (the reference leaves face_embs "
                             "unbound on that path)")
        enc_preds = self.encode(registration_vertices, pose)
        dec_preds = self.decoder(pose=pose, embs=enc_preds["embs"], face_embs=enc_preds["face_embs"])
        geom_rec = self.lbs_fn.pose(dec_preds["geom_delta_rec"], pose)
        dec_view_preds = self.decoder_view(geom_rec=geom_rec, tex_mean_rec=dec_preds["tex_mean_rec"],
                                           camera_pos=campos)
        shadow_preds = self.shadow_net(ao_map=ambient_occlusion)
        tex_rec = self.forward_tex(dec_preds["tex_mean_rec"], dec_view_preds["tex_view_rec"],
                                   shadow_preds["shadow_map"])
        cam_idxs = None
        if self.cal_enabled:
            cam_idxs = self.cal.name_to_idx(camera_id)
            tex_rec = self.cal(tex_rec, cam_idxs)
        preds = {"geom": geom_rec, "tex_rec": tex_rec, **dec_preds, **shadow_preds, **dec_view_preds, **enc_preds}
        if self.rendering_enabled:
            tex_seg = torch.ones_like(tex_rec[:, :1])
            renders = self.renderer(preds["geom"], tex=torch.cat([tex_rec, tex_seg], dim=1), K=K, Rt=Rt)
            render_depth = renders["depth_img"][:, None].detach()
            preds.update(rgb=renders["render"][:, :3], alpha=renders["render"][:, 3:],
                         depth_disc_mask=depth_discontuity_mask(render_depth), depth=render_depth)
        if self.learn_blur_enabled:
            preds["rgb"] = self.learn_blur(preds["rgb"], camera_id)
            preds["learn_blur_weights"] = self.learn_blur.reg(camera_id)
        if self.pixel_cal_enabled:
            preds["rgb"] = self.pixel_cal(cam_idxs, preds["rgb"])
        return preds
