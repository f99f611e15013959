"""`ShadowUNet` (ca_code/nn/shadow.py:22-188), the body avatar's ambient-occlusion-to-shadow U-Net, on the GPU: the
eight 3x3 layers run on `gb_conv2d_wnub_*` with untied biases and the LeakyReLU fused, and `shadow_pred` on the same
kernel with a tied (`biases=False`, `Conv2dWN`) or untied bias.  The resizes and the `sigmoid(. + beta)` stay in torch
with the reference's modes and corner conventions.  Constructor, parameter and buffer names and shapes are the
reference's, so its checkpoints load with strict=True.

Initialisation: the reference applies `blocks.weights_initializer`, whose `kaiming_uniform_(m.weight.data)` writes into
the weight-normalised layer's derived `weight` tensor and leaves `weight_v` / `weight_g` as the constructor made them.
So `weight_v` keeps nn.Conv2d's default init (bounded by 1/sqrt(fan_in)), `weight_g` is the whole-tensor norm of
`weight_v` (the effective weight equals `weight_v`), and every bias is zero — which is what the layers' constructors
here already produce.  CUDA only; CPU tensors raise.

`PoseToShadow` (ca_code/nn/shadow.py:429-471), the drivable body's shadow from the pose alone, runs its transposed
convolutions on the fused layer kernels and sigmoid(. + beta) with the resize on csrc/body_drive.cu."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

from . import _lib
from .nn import Conv2dWN, Conv2dWNUB, ConvTranspose2dWNUB, FusedLeakyReLU, LinearWN, glorot


def _conv3x3(cin, cout, size, slope):
    conv = Conv2dWNUB(cin, cout, kernel_size=3, height=size, width=size, stride=1, padding=1)
    conv.fused_slope = float(slope)
    return nn.Sequential(conv, FusedLeakyReLU())


class ShadowUNet(nn.Module):
    def __init__(self, uv_size, ao_mean, shadow_size, lrelu_slope=0.2, beta=1.0, n_dims=64, interp_mode="bilinear",
                 biases=True, trainable_mean=False):
        super().__init__()
        self.uv_size = uv_size
        self.shadow_size = shadow_size
        ao_mean = F.interpolate(torch.as_tensor(ao_mean)[np.newaxis], size=(shadow_size, shadow_size))[0]
        if not trainable_mean:
            self.register_buffer("ao_mean", ao_mean)
        else:
            self.register_parameter("ao_mean", nn.Parameter(ao_mean))
        self.depth = 3
        self.lrelu_slope = lrelu_slope
        self.interp_mode = interp_mode
        self.align_corners = False if interp_mode == "bilinear" else None
        self.n_enc_dims = [(1, n_dims), (n_dims, n_dims), (n_dims, n_dims), (n_dims, n_dims)]
        self.sizes = [shadow_size // (2 ** i) for i in range(len(self.n_enc_dims))]
        self.enc_layers = nn.ModuleList([_conv3x3(*self.n_enc_dims[i], size, lrelu_slope)
                                         for i, size in enumerate(self.sizes)])
        self.n_dec_dims = [(n_dims, n_dims), (n_dims * 2, n_dims), (n_dims * 2, n_dims), (n_dims * 2, n_dims)]
        self.dec_layers = nn.ModuleList([_conv3x3(*self.n_dec_dims[i], self.sizes[-i - 1], lrelu_slope)
                                         for i in range(len(self.sizes))])
        if biases:
            self.shadow_pred = Conv2dWNUB(self.n_dec_dims[-1][-1], 1, kernel_size=3, height=self.sizes[0],
                                          width=self.sizes[0], stride=1, padding=1)
        else:
            self.shadow_pred = Conv2dWN(self.n_dec_dims[-1][-1], 1, kernel_size=3, stride=1, padding=1)
        self.beta = beta

    def forward(self, ao_map):
        if not ao_map.is_cuda:
            raise RuntimeError("ShadowUNet runs on CUDA only (no CPU fallback): ao_map is on %s" % ao_map.device)
        if ao_map.shape[-2:] != (self.shadow_size, self.shadow_size):
            ao_map = F.interpolate(ao_map, size=(self.shadow_size, self.shadow_size))
        x = ao_map - self.ao_mean
        enc_acts = []
        for i, layer in enumerate(self.enc_layers):
            x = layer(x)
            enc_acts.append(x)
            if i < len(self.sizes) - 1:
                x = F.interpolate(x, scale_factor=0.5, mode="bilinear", recompute_scale_factor=True,
                                  align_corners=True)
        for i, layer in enumerate(self.dec_layers):
            if i > 0:
                x_prev = enc_acts[-i - 1]
                x = F.interpolate(x, size=x_prev.shape[2:4], mode="bilinear", align_corners=True)
                x = torch.cat([x, x_prev], dim=1)
            x = layer(x)
        shadow_map_lowres = torch.sigmoid(self.shadow_pred(x) + self.beta)
        shadow_map = F.interpolate(shadow_map_lowres, (self.uv_size, self.uv_size), mode=self.interp_mode,
                                   align_corners=self.align_corners)
        return {"shadow_map": shadow_map, "ao_map": ao_map, "shadow_map_lowres": shadow_map_lowres}


class _PoseShadow(Function):
    """bilinear(sigmoid(x + beta) -> size x size, align_corners=False) on csrc/body_drive.cu; the backward is a
    fixed-order gather per low-resolution texel"""

    @staticmethod
    def forward(ctx, x, beta, size):
        x = x.contiguous()
        _lib.check_input(x, "input")
        B, C, h, w = x.shape
        out = torch.empty(B, C, size, size, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().gb_pose_shadow_fwd(B * C, h, w, size, size, _lib.ptr(x), float(beta), _lib.ptr(out),
                                                     _lib.stream_ptr(x.device)), "pose_shadow_fwd")
        ctx.save_for_backward(x)
        ctx.beta = float(beta)
        return out

    @staticmethod
    def backward(ctx, g_out):
        (x,) = ctx.saved_tensors
        B, C, h, w = x.shape
        g_out = g_out.contiguous()
        g_x = torch.empty_like(x)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().gb_pose_shadow_bwd(B * C, h, w, g_out.shape[2], g_out.shape[3], _lib.ptr(x),
                                                     ctx.beta, _lib.ptr(g_out), _lib.ptr(g_x),
                                                     _lib.stream_ptr(x.device)), "pose_shadow_bwd")
        return g_x, None, None


def pose_shadow(x, beta, size):
    """bilinear(sigmoid(x + beta) -> size x size, align_corners=False) for x [B, C, h, w]; two backward calls give the
    same bits"""
    return _PoseShadow.apply(x, beta, size)


class PoseToShadow(nn.Module):
    """ca_code/nn/shadow.py:429-471: the shadow map from the pose alone.  `fc_block` is a LinearWN (cuBLAS) +
    LeakyReLU, `conv_block` five ConvTranspose2dWNUB (4^2 -> 128^2) on the fused layer kernels with the LeakyReLU in
    their epilogue (`FusedLeakyReLU` keeps the reference's indices), and sigmoid(. + beta) with the resize to
    `uv_size` one kernel each way (`pose_shadow`).  Keys and Glorot initialisation are the reference's."""

    def __init__(self, n_pose_dims, uv_size, beta=1.0) -> None:
        super().__init__()
        self.n_pose_dims, self.uv_size = n_pose_dims, uv_size
        self.fc_block = nn.Sequential(LinearWN(n_pose_dims, 256 * 4 * 4), nn.LeakyReLU(0.2))
        layers = []
        for cin, cout, size in ((256, 256, 8), (256, 128, 16), (128, 128, 32), (128, 64, 64)):
            layer = ConvTranspose2dWNUB(cin, cout, size, size, 4, 2, 1)
            layer.fused_slope = 0.2
            layers += [layer, FusedLeakyReLU()]
        self.conv_block = nn.Sequential(*layers, ConvTranspose2dWNUB(64, 1, 128, 128, 4, 2, 1))
        self.beta = beta
        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.conv_block[-1], 1.0)

    def forward(self, pose: torch.Tensor):
        if not pose.is_cuda:
            raise RuntimeError("PoseToShadow runs on CUDA only (no CPU fallback): pose is on %s" % pose.device)
        x = self.conv_block(self.fc_block(pose).reshape(-1, 256, 4, 4))
        return {"shadow_map": pose_shadow(x, self.beta, self.uv_size)}
