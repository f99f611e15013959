"""The body decoder `mesh_vae.ConvDecoder` (ca_code/models/mesh_vae.py:439-630) on the GPU: every `UpConvBlockDeep`
(the 8-64^2 `embs` / `face_embs` branches with groups = 1 and the 128^2-1024^2 trunk with groups = 2) runs on the
fused upsample + grouped weight-normalised convolution kernels of csrc/upconv_wnub.cu, the two 64^2 `ConvBlock`s and the
final 4 -> 3 convolutions on the stride-1 kernels (csrc/conv_wnub.cu, and a channel-slice variant so the final
convolutions read their halves of the 8-channel map in place), the seam sampler and `from_uv` on the gathers of
`goliath_b200.seams` when the caller passes this library's `SeamSampler` / `GeometryModule`.

Constructor, parameter names and shapes, buffers and the Glorot initialisation are the reference's, so a checkpoint of
the reference class loads with strict=True.  `geo_fn` and `seam_sampler` are duck-typed as in the reference: any object
with `from_uv`, and `impaint` / `resample`.  The small pieces stay in torch: the LinearWN layers, tile2d x mask, the
face / body merge and the concatenations.  Forward and backward are free of host synchronisation; CPU tensors raise."""
import numpy as np
import torch
import torch.nn as tnn
from torch.autograd import Function

from . import _lib
from .nn import ConvBlock, Conv2dWNUB, LinearWN, UpConvBlockDeep, _wn_chain, _wn_scale, glorot, tile2d


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

    def forward(self, pose, embs, face_embs):
        for t, n in ((pose, "pose"), (embs, "embs"), (face_embs, "face_embs")):
            if not t.is_cuda:
                raise RuntimeError("ConvDecoder runs on CUDA only (no CPU fallback): %s is on %s" % (n, t.device))
        B = pose.shape[0]
        local_pose = pose[:, 6:]
        non_head_mask = (self.body_cond_mask * (1.0 - self.face_cond_mask)).clip(0.0, 1.0)
        pose_masked = tile2d(local_pose, self.init_uv_size) * self.pose_cond_mask
        pose_conv = self.local_pose_conv_block(pose_masked) * non_head_mask
        embs_conv = self.embs_conv_block(self.embs_fc(embs).reshape(B, 128, 4, 4))
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
