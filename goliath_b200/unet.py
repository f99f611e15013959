"""`UNetWB` (ca_code/nn/unet.py:14-93) on the GPU: the five stride-2 4x4 down layers run on `gb_conv4x4s2_wnub_*`
and the five transposed up layers on `gb_deconv4x4s2_wnub_*`, both with the LeakyReLU fused into the kernel, and the
1x1 untied-bias `out` layer on `gb_conv2d_wnub_*`.  Constructor, parameter names and shapes and the Glorot
initialisation are the reference's, so its checkpoints load with strict=True; the `FusedLeakyReLU` placeholders keep the
Sequential indices.  The skip additions stay in torch: the kernels' backward reads the post-activation output to get
the LeakyReLU slope, so an add fused into the epilogue would break it.  CUDA only; CPU tensors raise."""
import torch
import torch.nn as nn

from .nn import Conv2dWNUB, ConvTranspose2dWNUB, FusedLeakyReLU, glorot


def _down(cin, cout, size):
    conv = Conv2dWNUB(cin, cout, size, size, 4, 2, 1)
    conv.fused_slope = 0.2
    return nn.Sequential(conv, FusedLeakyReLU())


def _up(cin, cout, size):
    conv = ConvTranspose2dWNUB(cin, cout, size, size, 4, 2, 1)
    conv.fused_slope = 0.2
    return nn.Sequential(conv, FusedLeakyReLU())


class UNetWB(nn.Module):
    """unet.py:14-93: `size` is the input (and output) size; the input is [B, in_channels, size, size]."""

    def __init__(self, in_channels: int, out_channels: int, size: int, n_init_ftrs: int = 8, out_scale: float = 0.1):
        super().__init__()
        self.out_scale = out_scale
        F = n_init_ftrs
        self.size = size
        self.down1 = _down(in_channels, F, size // 2)
        self.down2 = _down(F, 2 * F, size // 4)
        self.down3 = _down(2 * F, 4 * F, size // 8)
        self.down4 = _down(4 * F, 8 * F, size // 16)
        self.down5 = _down(8 * F, 16 * F, size // 32)
        self.up1 = _up(16 * F, 8 * F, size // 16)
        self.up2 = _up(8 * F, 4 * F, size // 8)
        self.up3 = _up(4 * F, 2 * F, size // 4)
        self.up4 = _up(2 * F, F, size // 2)
        self.up5 = _up(F, F, size)
        self.out = Conv2dWNUB(F + in_channels, out_channels, size, size, kernel_size=1, padding=0)
        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.out, 1.0)

    def forward(self, x):
        if not x.is_cuda:
            raise RuntimeError("UNetWB runs on CUDA only (no CPU fallback): the input is on %s" % x.device)
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
        return self.out(torch.cat([x, x1], dim=1)) * self.out_scale
