"""Decoder building blocks with the reference's names, parameter names and shapes (ca_code/nn/layers.py), so its
checkpoints load (`weight_v`, `weight_g`, `bias`): `ConvTranspose2dWNUB`, `LinearWN`, `make_conv_trans`,
`make_linear`.  Weight norm is the reference's non-standard one: g per output channel, norm of v over the WHOLE tensor
(layers.py:200-204,468-480; SURVEY.md §0.6):  w = g * v / ||v||_F.

The stride-2 4x4 transposed convolution + untied bias + LeakyReLU runs as ONE hand-written sm_90a kernel in the
forward, and its backward as three more (activation/bias gradient, data gradient, weight gradient) — no cuDNN
(csrc/deconv_wnub.cu).  The stride-2 4x4 convolution of the RGCA encoder (`Conv2dWNUB(.., 4, 2, 1)`) runs on the same
kernels with the two sides of the layer exchanged.  Round-1 status: fp32 SIMT kernels; LinearWN is a plain library
GEMM (cuBLAS via F.linear).

The body model's residual blocks run as fused blocks instead of layer by layer: `UpConvBlockDeep` (decoder,
csrc/upconv_wnub.cu) and `ConvDownBlock` (encoders, csrc/downconv_wnub.cu)."""
import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

from . import _lib


class _Deconv4x4s2WNUB(Function):
    @staticmethod
    def forward(ctx, x, weight_v, weight_g, bias, slope):
        x, weight_v = x.contiguous(), weight_v.contiguous()
        _lib.check_input(x, "input")
        _lib.check_input(weight_v, "weight_v")
        B, Cin, Hi, Wi = x.shape
        Cout = weight_v.shape[1]
        if weight_v.shape != (Cin, Cout, 4, 4):
            raise RuntimeError("weight_v must be [Cin, Cout, 4, 4]")
        vnorm = weight_v.norm()
        scale = (weight_g.reshape(-1) / vnorm).contiguous()
        b = None if bias is None else bias.contiguous()
        if b is not None and b.shape != (Cout, 2 * Hi, 2 * Wi):
            raise RuntimeError("untied bias must be [Cout, 2*Hi, 2*Wi]")
        out = torch.empty(B, Cout, 2 * Hi, 2 * Wi, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().gb_deconv4x4s2_wnub_fwd(
                B, Cin, Cout, Hi, Wi, _lib.ptr(x), _lib.ptr(weight_v), _lib.ptr(scale), _lib.ptr(b),
                float(slope if slope is not None else 1.0), int(slope is not None), _lib.ptr(out),
                _lib.stream_ptr(x.device)), "deconv4x4s2_wnub_fwd")
        ctx.save_for_backward(x, weight_v, weight_g, out)
        ctx.slope = slope
        ctx.has_bias = bias is not None
        return out

    @staticmethod
    def backward(ctx, gout):
        x, v, g, out = ctx.saved_tensors
        B, Cin, Hi, Wi = x.shape
        Cout = v.shape[1]
        dev = x.device
        gout = gout.contiguous()
        vnorm = v.norm()
        scale = (g.reshape(-1) / vnorm).contiguous()
        # the untied bias has one entry per output element, so with B == 1 its gradient IS the pre-activation gradient:
        # alias instead of writing it a second time; without an activation the pre-activation gradient is gout itself
        alias_bias = ctx.has_bias and B == 1
        if B == 1 and ctx.slope is None:
            gz = gout                                    # nothing to compute, nothing to copy
        else:
            gz = torch.empty_like(out)                   # scratch: gradient w.r.t. the pre-activation
        gb = None
        if ctx.has_bias and not alias_bias:
            gb = torch.empty(Cout, 2 * Hi, 2 * Wi, device=dev, dtype=torch.float32)
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gw = torch.zeros_like(v)                         # d L / d (effective weight), accumulated by the kernel
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_deconv4x4s2_wnub_bwd(
                B, Cin, Cout, Hi, Wi, _lib.ptr(x), _lib.ptr(v), _lib.ptr(scale), _lib.ptr(out), _lib.ptr(gout),
                float(ctx.slope if ctx.slope is not None else 1.0), int(ctx.slope is not None), _lib.ptr(gz), _lib.ptr(gb),
                _lib.ptr(gx), _lib.ptr(gw), _lib.stream_ptr(dev)), "deconv4x4s2_wnub_bwd")
        if alias_bias:
            gb = gz.view(Cout, 2 * Hi, 2 * Wi)
        # weight-norm chain rule on the small [Cin,Cout,4,4] tensors:  w = g * v / n,  n = ||v||_F
        w = g * v / vnorm
        gg = (gw * v).sum(dim=(0, 2, 3), keepdim=True) / vnorm
        gv = g * gw / vnorm - (gw * w).sum() * v / (vnorm * vnorm)
        return gx, gv, gg.view_as(g), gb, None


class ConvTranspose2dWNUB(nn.Module):
    """ConvTranspose2d(k=4, s=2, p=1) with weight norm and untied bias (layers.py:331-397,478-480)."""

    def __init__(self, in_channels, out_channels, height, width, kernel_size=4, stride=2, padding=1, bias=True):
        super().__init__()
        if (kernel_size, stride, padding) != (4, 2, 1):
            raise NotImplementedError("the fused kernel covers the decoder towers' k=4, s=2, p=1 layers")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.weight_v = nn.Parameter(torch.empty(in_channels, out_channels, 4, 4))
        self.weight_g = nn.Parameter(torch.ones(1, out_channels, 1, 1))
        self.bias = nn.Parameter(torch.zeros(out_channels, height, width)) if bias else None
        self.fused_slope: Optional[float] = None  # set by make_conv_trans when a LeakyReLU follows the layer
        nn.init.kaiming_uniform_(self.weight_v, a=math.sqrt(5))
        with torch.no_grad():
            self.weight_g.fill_(float(self.weight_v.norm()))  # weight == weight_v at init (layers.py:236-242)

    @property
    def weight(self):
        return self.weight_g * self.weight_v / self.weight_v.norm()

    def forward(self, input, slope: Optional[float] = None):
        """`slope` (or `fused_slope`) fuses the LeakyReLU that follows the layer into the same kernel."""
        slope = self.fused_slope if slope is None else slope
        return _Deconv4x4s2WNUB.apply(input, self.weight_v, self.weight_g, self.bias, slope)


class _ConvS1WN(Function):
    """stride-1 KxK conv + weight-norm scale + tied/untied bias [+ LeakyReLU], csrc/conv_wnub.cu."""

    @staticmethod
    def forward(ctx, x, weight_v, weight_g, bias, slope):
        x, weight_v = x.contiguous(), weight_v.contiguous()
        _lib.check_input(x, "input")
        _lib.check_input(weight_v, "weight_v")
        B, Cin, H, W = x.shape
        Cout, K = weight_v.shape[0], weight_v.shape[2]
        if weight_v.shape != (Cout, Cin, K, K) or K not in (1, 3):
            raise RuntimeError("weight_v must be [Cout, Cin, K, K] with K in (1, 3)")
        mode = 0
        b = None
        if bias is not None:
            b = bias.contiguous()
            if b.shape == (Cout,):
                mode = 1
            elif b.shape == (Cout, H, W):
                mode = 2
            else:
                raise RuntimeError("bias must be [Cout] or [Cout, H, W]")
        scale = (weight_g.reshape(-1) / weight_v.norm()).contiguous()
        out = torch.empty(B, Cout, H, W, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().gb_conv2d_wnub_fwd(
                B, Cin, Cout, H, W, K, _lib.ptr(x), _lib.ptr(weight_v), _lib.ptr(scale), _lib.ptr(b), mode,
                float(slope if slope is not None else 1.0), int(slope is not None), _lib.ptr(out),
                _lib.stream_ptr(x.device)), "conv2d_wnub_fwd")
        ctx.save_for_backward(x, weight_v, weight_g, out)
        ctx.slope, ctx.mode = slope, mode
        return out

    @staticmethod
    def backward(ctx, gout):
        x, v, g, out = ctx.saved_tensors
        B, Cin, H, W = x.shape
        Cout, K = v.shape[0], v.shape[2]
        dev = x.device
        gout = gout.contiguous()
        vnorm = v.norm()
        scale = (g.reshape(-1) / vnorm).contiguous()
        gz = torch.empty_like(out)
        gb = None
        if ctx.mode == 1:
            gb = torch.zeros(Cout, device=dev, dtype=torch.float32)
        elif ctx.mode == 2:
            gb = torch.empty(Cout, H, W, device=dev, dtype=torch.float32)
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gw = torch.zeros_like(v)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_conv2d_wnub_bwd(
                B, Cin, Cout, H, W, K, _lib.ptr(x), _lib.ptr(v), _lib.ptr(scale), _lib.ptr(out), _lib.ptr(gout),
                float(ctx.slope if ctx.slope is not None else 1.0), int(ctx.slope is not None), ctx.mode, _lib.ptr(gz),
                _lib.ptr(gb), _lib.ptr(gx), _lib.ptr(gw), _lib.stream_ptr(dev)), "conv2d_wnub_bwd")
        # weight-norm chain rule, g per OUTPUT channel (dim 0), norm over the whole tensor
        w = g * v / vnorm
        gg = (gw * v).sum(dim=(1, 2, 3), keepdim=True) / vnorm
        gv = g * gw / vnorm - (gw * w).sum() * v / (vnorm * vnorm)
        return gx, gv, gg.view_as(g), gb, None


class _Conv4x4s2WN(Function):
    """stride-2 4x4 conv (padding 1) + weight-norm scale + untied bias [+ LeakyReLU], csrc/deconv_wnub.cu."""

    @staticmethod
    def forward(ctx, x, weight_v, weight_g, bias, slope):
        x, weight_v = x.contiguous(), weight_v.contiguous()
        _lib.check_input(x, "input")
        _lib.check_input(weight_v, "weight_v")
        B, Cin, H, W = x.shape
        Cout = weight_v.shape[0]
        if weight_v.shape != (Cout, Cin, 4, 4):
            raise RuntimeError("weight_v must be [Cout, Cin, 4, 4]")
        if H % 2 or W % 2:
            raise RuntimeError("a k=4, s=2, p=1 layer needs an even input size (got %dx%d)" % (H, W))
        Ho, Wo = H // 2, W // 2
        b = None if bias is None else bias.contiguous()
        if b is not None and b.shape != (Cout, Ho, Wo):
            raise RuntimeError("untied bias must be [Cout, H/2, W/2]")
        scale = (weight_g.reshape(-1) / weight_v.norm()).contiguous()
        out = torch.empty(B, Cout, Ho, Wo, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().gb_conv4x4s2_wnub_fwd(
                B, Cin, Cout, Ho, Wo, _lib.ptr(x), _lib.ptr(weight_v), _lib.ptr(scale), _lib.ptr(b),
                float(slope if slope is not None else 1.0), int(slope is not None), _lib.ptr(out),
                _lib.stream_ptr(x.device)), "conv4x4s2_wnub_fwd")
        ctx.save_for_backward(x, weight_v, weight_g, out)
        ctx.slope = slope
        ctx.has_bias = bias is not None
        return out

    @staticmethod
    def backward(ctx, gout):
        x, v, g, out = ctx.saved_tensors
        B, Cin = x.shape[:2]
        Cout, Ho, Wo = out.shape[1:]
        dev = x.device
        gout = gout.contiguous()
        vnorm = v.norm()
        scale = (g.reshape(-1) / vnorm).contiguous()
        # as in _Deconv4x4s2WNUB: with B == 1 the untied-bias gradient is the pre-activation gradient, and without an
        # activation that is gout itself
        alias_bias = ctx.has_bias and B == 1
        gz = gout if B == 1 and ctx.slope is None else torch.empty_like(out)
        gb = None
        if ctx.has_bias and not alias_bias:
            gb = torch.empty(Cout, Ho, Wo, device=dev, dtype=torch.float32)
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gw = torch.zeros_like(v)                         # d L / d (effective weight), accumulated by the kernel
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_conv4x4s2_wnub_bwd(
                B, Cin, Cout, Ho, Wo, _lib.ptr(x), _lib.ptr(v), _lib.ptr(scale), _lib.ptr(out), _lib.ptr(gout),
                float(ctx.slope if ctx.slope is not None else 1.0), int(ctx.slope is not None), _lib.ptr(gz), _lib.ptr(gb),
                _lib.ptr(gx), _lib.ptr(gw), _lib.stream_ptr(dev)), "conv4x4s2_wnub_bwd")
        if alias_bias:
            gb = gz.view(Cout, Ho, Wo)
        # weight-norm chain rule, g per OUTPUT channel (dim 0), norm over the whole tensor (as _ConvS1WN)
        w = g * v / vnorm
        gg = (gw * v).sum(dim=(1, 2, 3), keepdim=True) / vnorm
        gv = g * gw / vnorm - (gw * w).sum() * v / (vnorm * vnorm)
        return gx, gv, gg.view_as(g), gb, None


class Conv2dWNUB(nn.Module):
    """Conv2d with weight norm and untied bias (layers.py:276-327,472): stride 1, k in {1,3}, "same" padding (hand-MVP
    decoders), or k=4, s=2, p=1 (the RGCA encoder, rgca.py:281-298), where (height, width) is the OUTPUT size and the
    input must be [B, Cin, 2*height, 2*width].
    Constructor argument order is the reference's: (in, out, height, width, kernel_size, stride, padding)."""

    def __init__(self, in_channels, out_channels, height, width, kernel_size=3, stride=1, padding=1, bias=True):
        super().__init__()
        strided = (kernel_size, stride, padding) == (4, 2, 1)
        if not strided and (stride != 1 or kernel_size not in (1, 3) or padding != (kernel_size - 1) // 2):
            raise NotImplementedError("the fused kernels cover stride-1 'same' 1x1 / 3x3 layers and k=4, s=2, p=1 layers")
        self.in_channels, self.out_channels, self.kernel_size = in_channels, out_channels, (kernel_size, kernel_size)
        self.stride = (stride, stride)
        self._out_size = (height, width)
        self.weight_v = nn.Parameter(torch.empty(out_channels, in_channels, kernel_size, kernel_size))
        self.weight_g = nn.Parameter(torch.ones(out_channels, 1, 1, 1))
        self.bias = nn.Parameter(torch.zeros(out_channels, height, width)) if bias else None
        self.fused_slope: Optional[float] = None
        nn.init.kaiming_uniform_(self.weight_v, a=math.sqrt(5))
        with torch.no_grad():
            self.weight_g.fill_(float(self.weight_v.norm()))

    @property
    def weight(self):
        return self.weight_g * self.weight_v / self.weight_v.norm()

    def forward(self, input, slope: Optional[float] = None):
        slope = self.fused_slope if slope is None else slope
        if self.stride[0] == 2:
            h, w = self._out_size
            if input.dim() != 4 or tuple(input.shape[1:]) != (self.in_channels, 2 * h, 2 * w):
                raise RuntimeError("input must be [B, %d, %d, %d] (got %s)" % (self.in_channels, 2 * h, 2 * w,
                                                                              tuple(input.shape)))
            return _Conv4x4s2WN.apply(input, self.weight_v, self.weight_g, self.bias, slope)
        return _ConvS1WN.apply(input, self.weight_v, self.weight_g, self.bias, slope)


class Conv2dWN(Conv2dWNUB):
    """th.nn.Conv2d with the reference's weight norm and a tied bias [Cout] (layers.py:470; ConvBlock.conv_resize)."""

    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, padding=0, bias=True):
        if stride != 1:
            raise NotImplementedError("the fused kernels cover stride-1 'same' 1x1 / 3x3 tied-bias layers")
        super().__init__(in_channels, out_channels, 1, 1, kernel_size, stride, padding, bias=False)
        self.bias = nn.Parameter(torch.zeros(out_channels)) if bias else None


def tile2d(x, size: int):
    """[N,F] -> [N,F,size,size] (blocks.py:731-743)."""
    return x[:, :, None, None].expand(-1, -1, size, size)


class ConvBlock(nn.Module):
    """blocks.py:232-280: 1x1 Conv2dWN skip + two Conv2dWNUB with LeakyReLU (fused into the conv kernels)."""

    def __init__(self, in_channels, out_channels, size, lrelu_slope=0.2, kernel_size=3, padding=1, wnorm_dim=0):
        super().__init__()
        assert wnorm_dim == 0
        self.conv_resize = Conv2dWN(in_channels, out_channels, kernel_size=1)
        self.conv1 = Conv2dWNUB(in_channels, in_channels, size, size, kernel_size, 1, padding)
        self.conv2 = Conv2dWNUB(in_channels, out_channels, size, size, kernel_size, 1, padding)
        self.conv1.fused_slope = self.conv2.fused_slope = float(lrelu_slope)
        self.lrelu1, self.lrelu2 = FusedLeakyReLU(), FusedLeakyReLU()

    def forward(self, x):
        x_skip = self.conv_resize(x)
        return self.conv2(self.conv1(x)) + x_skip


class LinearWN(nn.Module):
    """nn.Linear with the reference's weight norm (layers.py:468): weight_g [out,1], weight_v [out,in]."""

    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.weight_v = nn.Parameter(torch.empty(out_features, in_features))
        self.weight_g = nn.Parameter(torch.ones(out_features, 1))
        self.bias = nn.Parameter(torch.zeros(out_features)) if bias else None
        nn.init.kaiming_uniform_(self.weight_v, a=math.sqrt(5))
        with torch.no_grad():
            self.weight_g.fill_(float(self.weight_v.norm()))

    @property
    def weight(self):
        return self.weight_g * self.weight_v / self.weight_v.norm()

    def forward(self, input):
        return F.linear(input, self.weight, self.bias)  # plain library GEMM (cuBLAS)


class FusedLeakyReLU(nn.Identity):
    """Placeholder for the LeakyReLU that the preceding ConvTranspose2dWNUB already applied in its epilogue; it keeps
    the Sequential indices (and therefore the checkpoint key names) identical to the reference's [layer, act] lists."""


def _pad32(c):
    return (c + 31) // 32 * 32


# which layers of a tower run on the tensor cores; TC_MIN_CIN can be lowered to 16 to put the last (16 -> 125) layer
# on them too (its K dimension is then half zero padding)
TC_MIN_CIN = 32


def _tc_layer_ok(cin, cout):
    return cout <= 256 and cin >= TC_MIN_CIN


def tower_forward_tc(tower: nn.Sequential, x: torch.Tensor) -> torch.Tensor:
    """Inference forward of a deconv tower (Sequential of ConvTranspose2dWNUB [+ FusedLeakyReLU]) on the tensor cores
    (csrc/deconv_tc.cu: wgmma tf32 with 3xTF32 split, TMA-fed, register accumulators).  Activations stay NHWC
    (hi/lo split) between tensor-core layers (channels padded to 32, N padded to 16 inside the kernel); only layers
    with Cout > 256 would fall back to the SIMT kernel.
    No autograd: use the module's normal forward for training."""
    assert not torch.is_grad_enabled(), "tower_forward_tc is the inference path"
    L = _lib.lib()
    dev = x.device
    layers = [m for m in tower if isinstance(m, ConvTranspose2dWNUB)]
    cur_nchw, cur_hi, cur_lo, cur_c = x.contiguous(), None, None, x.shape[1]
    B, _, H, W = x.shape
    with torch.cuda.device(dev):
        st = _lib.stream_ptr(dev)
        for i, layer in enumerate(layers):
            Cin, Cout = layer.in_channels, layer.out_channels
            # with Cin = 16 the layer is pure output/bias bandwidth and the per-pixel NCHW epilogue of the tensor-core
            # kernel loses to the SIMT kernel (bench.py decoder object, 16 -> 125 @ 1024^2 on an H100 SXM at 400 W:
            # 0.92 ms SIMT, 1.05 ms tensor cores), so it stays SIMT
            tc_ok = _tc_layer_ok(Cin, Cout)
            nxt = layers[i + 1] if i + 1 < len(layers) else None
            nxt_tc = nxt is not None and _tc_layer_ok(nxt.in_channels, nxt.out_channels)
            bias = None if layer.bias is None else layer.bias.contiguous()
            slope = layer.fused_slope
            # frozen-parameter cache: weight-norm scale and the prepared tensor-core weight matrices are functions of
            # (weight_v, weight_g) only; they are rebuilt when either tensor is modified in place or replaced
            key = (layer.weight_v.data_ptr(), layer.weight_v._version, layer.weight_g.data_ptr(), layer.weight_g._version)
            cache = getattr(layer, "_tc_cache", None)
            fresh = cache is None or cache[0] != key
            if fresh:
                scale = (layer.weight_g.reshape(-1) / layer.weight_v.norm()).contiguous()
                ws = torch.empty(L.gb_deconv_tc_weight_bytes(_pad32(Cin), Cout) // 4, device=dev) if tc_ok else None
                layer._tc_cache = (key, scale, ws)
            else:
                _, scale, ws = cache
            if tc_ok:
                cpad = _pad32(Cin)
                if cur_hi is None:  # enter the NHWC hi/lo format
                    cur_hi = torch.empty(B, H, W, cpad, device=dev)
                    cur_lo = torch.empty(B, H, W, cpad, device=dev)
                    _lib.check(L.gb_nchw_to_nhwc_split(B, Cin, cpad, H, W, _lib.ptr(cur_nchw), _lib.ptr(cur_hi),
                                                       _lib.ptr(cur_lo), st), "nchw_to_nhwc_split")
                    cur_c = cpad
                assert cur_c == cpad, "channel padding mismatch between consecutive tensor-core layers"
                ldc = _pad32(Cout)
                # padded output channels must be zero for the next layer's K loop
                o_hi = (torch.zeros if ldc != Cout else torch.empty)(B, 2 * H, 2 * W, ldc, device=dev) if nxt_tc else None
                o_lo = (torch.zeros if ldc != Cout else torch.empty)(B, 2 * H, 2 * W, ldc, device=dev) if nxt_tc else None
                o_nchw = None if nxt_tc else torch.empty(B, Cout, 2 * H, 2 * W, device=dev)
                _lib.check(L.gb_deconv4x4s2_tc_fwd(
                    B, Cin, cpad, Cout, H, W, _lib.ptr(cur_hi), _lib.ptr(cur_lo),
                    _lib.ptr(layer.weight_v.contiguous()) if fresh else None, _lib.ptr(ws), _lib.ptr(scale), _lib.ptr(bias), float(slope if slope is not None else 1.0),
                    int(slope is not None), _lib.ptr(o_hi), _lib.ptr(o_lo), ldc, _lib.ptr(o_nchw), st), "deconv4x4s2_tc_fwd")
                cur_hi, cur_lo, cur_c, cur_nchw = o_hi, o_lo, ldc, o_nchw
            else:
                assert cur_nchw is not None
                out = torch.empty(B, Cout, 2 * H, 2 * W, device=dev)
                _lib.check(L.gb_deconv4x4s2_wnub_fwd(
                    B, Cin, Cout, H, W, _lib.ptr(cur_nchw), _lib.ptr(layer.weight_v.contiguous()), _lib.ptr(scale),
                    _lib.ptr(bias), float(slope if slope is not None else 1.0), int(slope is not None), _lib.ptr(out), st),
                    "deconv4x4s2_wnub_fwd")
                cur_nchw, cur_hi, cur_lo = out, None, None
            H, W = 2 * H, 2 * W
    assert cur_nchw is not None, "a tower must end with a layer that produces NCHW output"
    return cur_nchw


def make_conv_trans(n_in, n_out, fs, stride, pad, mode, act=None, ub=None, bias=True):
    """layers.py:27-47 with trans=True, ub=(H,W).  Returns [layer] or [layer, act] like the reference; a LeakyReLU is
    executed inside the layer's kernel and replaced by a parameter-free placeholder at the same list position."""
    assert mode == "wn" and ub is not None
    layer = ConvTranspose2dWNUB(n_in, n_out, ub[0], ub[1], fs, stride, pad, bias=bias)
    if act is None:
        return [layer]
    if isinstance(act, nn.LeakyReLU):
        layer.fused_slope = float(act.negative_slope)
        return [layer, FusedLeakyReLU()]
    return [layer, act]


def make_linear(n_in, n_out, mode, act=None, bias=True):
    assert mode == "wn"
    layers = [LinearWN(n_in, n_out, bias=bias)]
    if act is not None:
        layers.append(act)
    return layers


def glorot(m: nn.Module, alpha: float = 1.0) -> None:
    """Initialisation used by the decoders (layers.py:605-650): uniform with the Glorot std scaled for a LeakyReLU of
    slope `alpha`; a stride-2 transposed kernel gets its four sub-pixel phases tied at init; bias zero.  For the
    weight-normalised layers of this module the direction tensor receives the sample and g its Frobenius norm, i.e.
    the effective weight equals the sample."""
    gain = math.sqrt(2.0 / (1.0 + alpha ** 2))
    if isinstance(m, (Conv2dWNUB,)):
        k = m.kernel_size[0] * m.kernel_size[1]
        fan = (m.in_channels + m.out_channels) * k
    elif isinstance(m, ConvTranspose2dWNUB):
        fan = (m.in_channels + m.out_channels) * 4  # 4x4 kernel, stride 2: k*k // 4
    elif isinstance(m, LinearWN):
        fan = m.weight_v.shape[0] + m.weight_v.shape[1]
    else:
        return
    bound = gain * math.sqrt(2.0 / fan) * math.sqrt(3.0)
    with torch.no_grad():
        m.weight_v.uniform_(-bound, bound)
        if isinstance(m, ConvTranspose2dWNUB):
            base = m.weight_v[:, :, 0::2, 0::2].clone()
            m.weight_v[:, :, 0::2, 1::2] = base
            m.weight_v[:, :, 1::2, 0::2] = base
            m.weight_v[:, :, 1::2, 1::2] = base
        m.weight_g.fill_(float(m.weight_v.norm()))
        if m.bias is not None:
            m.bias.zero_()


def _wn_chain(v, g, gw):
    """weight-norm chain rule (g per output channel, norm over the whole tensor) from the effective-weight gradient"""
    vnorm = v.norm()
    w = g * v / vnorm
    gg = (gw * v).sum(dim=tuple(range(1, v.dim())), keepdim=True) / vnorm
    gv = g * gw / vnorm - (gw * w).sum() * v / (vnorm * vnorm)
    return gv, gg.view_as(g)


def _wn_scale(v, g):
    return (g.reshape(-1) / v.norm()).contiguous()


class _UpConvBlock(Function):
    """UpConvBlockDeep forward / backward on csrc/upconv_wnub.cu (two kernels forward, eight backward)."""

    @staticmethod
    def forward(ctx, x, v1, g1, b1, v2, g2, b2, vr, gr, br, slope, groups):
        x = x.contiguous()
        _lib.check_input(x, "input")
        for t, n in ((v1, "conv1.weight_v"), (v2, "conv2.weight_v"), (vr, "conv_resize.weight_v"),
                     (b1, "conv1.bias"), (b2, "conv2.bias"), (br, "conv_resize.bias")):
            _lib.check_input(t, n)
        B, Cin, Hi, Wi = x.shape
        Cout = v2.shape[0]
        H, W = 2 * Hi, 2 * Wi
        if (v1.shape != (Cin, Cin // groups, 3, 3) or v2.shape != (Cout, Cin // groups, 3, 3)
                or vr.shape != (Cout, Cin // groups, 1, 1) or b1.shape != (Cin, H, W) or b2.shape != (Cout, H, W)):
            raise RuntimeError("UpConvBlockDeep: parameter shapes do not match an input of %s" % (tuple(x.shape),))
        s1, s2, sr = _wn_scale(v1, g1), _wn_scale(v2, g2), _wn_scale(vr, gr)
        dev = x.device
        h1 = torch.empty(B, Cin, H, W, device=dev)
        out = torch.empty(B, Cout, H, W, device=dev)
        train = any(ctx.needs_input_grad)
        mask = torch.empty(B, Cout, H, W, device=dev, dtype=torch.uint8) if train else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_upconv_block_fwd(
                B, Cin, Cout, groups, Hi, Wi, _lib.ptr(x), _lib.ptr(v1), _lib.ptr(s1), _lib.ptr(b1), _lib.ptr(v2),
                _lib.ptr(s2), _lib.ptr(b2), _lib.ptr(vr), _lib.ptr(sr), _lib.ptr(br), float(slope), _lib.ptr(h1),
                _lib.ptr(out), _lib.ptr(mask), _lib.stream_ptr(dev)), "upconv_block_fwd")
        if train:
            ctx.save_for_backward(x, v1, g1, v2, g2, vr, gr, h1, mask)
        ctx.slope, ctx.groups = float(slope), groups
        return out

    @staticmethod
    def backward(ctx, gout):
        x, v1, g1, v2, g2, vr, gr, h1, mask = ctx.saved_tensors
        B, Cin, Hi, Wi = x.shape
        Cout = v2.shape[0]
        H, W = 2 * Hi, 2 * Wi
        dev = x.device
        gout = gout.contiguous()
        s1, s2, sr = _wn_scale(v1, g1), _wn_scale(v2, g2), _wn_scale(vr, gr)
        need_gx = ctx.needs_input_grad[0]
        gz2 = torch.empty(B, Cout, H, W, device=dev)
        gz1 = torch.empty(B, Cin, H, W, device=dev)
        gu = torch.empty(B, Cin, H, W, device=dev) if need_gx else None
        gx = torch.empty_like(x) if need_gx else None
        gb1 = torch.empty(Cin, H, W, device=dev)
        gb2 = torch.empty(Cout, H, W, device=dev)
        gbr = torch.zeros(Cout, device=dev)
        gw1, gw2, gwr = torch.zeros_like(v1), torch.zeros_like(v2), torch.zeros_like(vr)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_upconv_block_bwd(
                B, Cin, Cout, ctx.groups, Hi, Wi, _lib.ptr(x), _lib.ptr(v1), _lib.ptr(s1), _lib.ptr(v2), _lib.ptr(s2),
                _lib.ptr(vr), _lib.ptr(sr), _lib.ptr(h1), _lib.ptr(mask), _lib.ptr(gout), ctx.slope, _lib.ptr(gz2),
                _lib.ptr(gz1), _lib.ptr(gu), _lib.ptr(gb1), _lib.ptr(gb2), _lib.ptr(gbr), _lib.ptr(gw1), _lib.ptr(gw2),
                _lib.ptr(gwr), _lib.ptr(gx), _lib.stream_ptr(dev)), "upconv_block_bwd")
        gv1, gg1 = _wn_chain(v1, g1, gw1)
        gv2, gg2 = _wn_chain(v2, g2, gw2)
        gvr, ggr = _wn_chain(vr, gr, gwr)
        return gx, gv1, gg1, gb1, gv2, gg2, gb2, gvr, ggr, gbr, None, None


def _grouped(m, groups):
    """give a weight-norm conv the reference's grouped weight_v [Cout, Cin/groups, k, k] (its kernel is the block's)"""
    m.groups = groups
    if groups != 1:
        m.weight_v = nn.Parameter(torch.empty(m.out_channels, m.in_channels // groups, *m.kernel_size))
        nn.init.kaiming_uniform_(m.weight_v, a=math.sqrt(5))
        with torch.no_grad():
            m.weight_g.fill_(float(m.weight_v.norm()))
    return m


class UpConvBlockDeep(nn.Module):
    """blocks.py:382-434: bilinear x2 upsample (align_corners=True), grouped weight-normalised 1x1 skip with tied bias,
    two grouped 3x3 Conv2dWNUB + LeakyReLU; the whole block runs on the two fused kernels of csrc/upconv_wnub.cu, and
    `lrelu1` / `lrelu2` are parameter-free placeholders.  `size` is the OUTPUT size; the input is [B, Cin, size/2,
    size/2].  Parameter names and shapes are the reference's."""

    def __init__(self, in_channels, out_channels, size, lrelu_slope=0.2, wnorm_dim=0, groups=1):
        super().__init__()
        if wnorm_dim != 0:
            raise NotImplementedError("only wnorm_dim = 0 (g per output channel) is supported")
        if in_channels % groups or out_channels % groups or size % 2:
            raise ValueError("channels must divide into groups and size must be even")
        self.size, self.groups, self.lrelu_slope = size, groups, float(lrelu_slope)
        self.conv_resize = _grouped(Conv2dWN(in_channels, out_channels, kernel_size=1), groups)
        self.conv1 = _grouped(Conv2dWNUB(in_channels, in_channels, size, size, 3, 1, 1), groups)
        self.lrelu1 = FusedLeakyReLU()
        self.conv2 = _grouped(Conv2dWNUB(in_channels, out_channels, size, size, 3, 1, 1), groups)
        self.lrelu2 = FusedLeakyReLU()

    def forward(self, x):
        if x.dim() != 4 or x.shape[2] * 2 != self.size or x.shape[3] * 2 != self.size:
            raise RuntimeError("UpConvBlockDeep(size=%d) needs a [B, C, %d, %d] input (got %s)"
                               % (self.size, self.size // 2, self.size // 2, tuple(x.shape)))
        c1, c2, cr = self.conv1, self.conv2, self.conv_resize
        return _UpConvBlock.apply(x, c1.weight_v, c1.weight_g, c1.bias, c2.weight_v, c2.weight_g, c2.bias,
                                  cr.weight_v, cr.weight_g, cr.bias, self.lrelu_slope, self.groups)


class _DownConvBlock(Function):
    """ConvDownBlock forward / backward on csrc/downconv_wnub.cu (two kernels forward, ten or eleven backward).  With
    `cond_mask` the block's input is cond_scale * bilinear(x -> mask's size) * cond_mask, built inside the kernels."""

    @staticmethod
    def forward(ctx, x, v1, g1, b1, v2, g2, b2, vr, gr, br, slope, groups, cond_mask, cond_scale):
        if x.dim() != 4 or not x.is_cuda or x.dtype != torch.float32:
            raise RuntimeError("input must be a float32 CUDA tensor [B, C, H, W]")
        if cond_mask is None or x.stride(3) != 1 or min(x.stride()) < 1:
            x = x.contiguous()  # a window of a larger map is read in place only by the fused resize
        for t, n in ((v1, "conv1.weight_v"), (v2, "conv2.weight_v"), (vr, "conv_resize.weight_v"),
                     (b1, "conv1.bias"), (b2, "conv2.bias"), (br, "conv_resize.bias")):
            _lib.check_input(t, n)
        B, Cin, Hs, Ws = x.shape
        Cout = v2.shape[0]
        if cond_mask is None:
            H, W = Hs, Ws
        else:
            _lib.check_input(cond_mask, "mask", torch.bool)
            H, W = cond_mask.shape[-2:]
            if cond_mask.numel() != H * W:
                raise RuntimeError("mask must hold one [H, W] plane")
        if (H % 2 or W % 2 or v1.shape != (Cin, Cin // groups, 3, 3) or v2.shape != (Cout, Cin // groups, 3, 3)
                or vr.shape != (Cout, Cin // groups, 1, 1) or b1.shape != (Cin, H, W)
                or b2.shape != (Cout, H // 2, W // 2) or br.shape != (Cout,)):
            raise RuntimeError("ConvDownBlock: parameter shapes do not match an input of %s" % (tuple(x.shape),))
        s1, s2, sr = _wn_scale(v1, g1), _wn_scale(v2, g2), _wn_scale(vr, gr)
        dev = x.device
        h1 = torch.empty(B, Cin, H, W, device=dev)
        out = torch.empty(B, Cout, H // 2, W // 2, device=dev)
        train = any(ctx.needs_input_grad)
        mask = torch.empty(B, Cout, H // 2, W // 2, device=dev, dtype=torch.uint8) if train else None
        ctx.xargs = (B, Cin, Cout, groups, H, W)
        ctx.cond = (x.stride(0), x.stride(1), x.stride(2), Hs, Ws)
        ctx.cond_scale = float(cond_scale)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_downconv_block_fwd(
                *ctx.xargs, _lib.ptr(x), *ctx.cond, _lib.ptr(cond_mask), ctx.cond_scale, _lib.ptr(v1), _lib.ptr(s1),
                _lib.ptr(b1), _lib.ptr(v2), _lib.ptr(s2), _lib.ptr(b2), _lib.ptr(vr), _lib.ptr(sr), _lib.ptr(br),
                float(slope), _lib.ptr(h1), _lib.ptr(out), _lib.ptr(mask), _lib.stream_ptr(dev)), "downconv_block_fwd")
        if train:
            ctx.save_for_backward(x, v1, g1, v2, g2, vr, gr, h1, mask, cond_mask)
        ctx.slope = float(slope)
        return out

    @staticmethod
    def backward(ctx, gout):
        x, v1, g1, v2, g2, vr, gr, h1, mask, cond_mask = ctx.saved_tensors
        B, Cin, Cout, groups, H, W = ctx.xargs
        dev = x.device
        gout = gout.contiguous()
        s1, s2, sr = _wn_scale(v1, g1), _wn_scale(v2, g2), _wn_scale(vr, gr)
        need_gx = ctx.needs_input_grad[0]
        if need_gx and cond_mask is not None:
            raise RuntimeError("ConvDownBlock: the fused resize + mask of the input has no backward")
        L = _lib.lib()
        gz2 = torch.empty(B, Cout, H // 2, W // 2, device=dev)
        gz1 = torch.empty(B, Cin, H, W, device=dev)
        gx = torch.empty(B, Cin, H, W, device=dev) if need_gx else None
        gb1 = torch.empty(Cin, H, W, device=dev)
        gb2 = torch.empty(Cout, H // 2, W // 2, device=dev)
        gbr = torch.empty(Cout, device=dev)
        gw1, gw2, gwr = torch.empty_like(v1), torch.empty_like(v2), torch.empty_like(vr)
        ws = torch.empty(L.gb_downconv_block_bwd_workspace_bytes(*ctx.xargs) // 4, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.gb_downconv_block_bwd(
                *ctx.xargs, _lib.ptr(x), *ctx.cond, _lib.ptr(cond_mask), ctx.cond_scale, _lib.ptr(v1), _lib.ptr(s1),
                _lib.ptr(v2), _lib.ptr(s2), _lib.ptr(vr), _lib.ptr(sr), _lib.ptr(h1), _lib.ptr(mask), _lib.ptr(gout),
                ctx.slope, _lib.ptr(gz2), _lib.ptr(gz1), _lib.ptr(gb1), _lib.ptr(gb2), _lib.ptr(gbr), _lib.ptr(gw1),
                _lib.ptr(gw2), _lib.ptr(gwr), _lib.ptr(gx), _lib.ptr(ws), _lib.stream_ptr(dev)), "downconv_block_bwd")
        gv1, gg1 = _wn_chain(v1, g1, gw1)
        gv2, gg2 = _wn_chain(v2, g2, gw2)
        gvr, ggr = _wn_chain(vr, gr, gwr)
        return gx, gv1, gg1, gb1, gv2, gg2, gb2, gvr, ggr, gbr, None, None, None, None


def _block_only(*args, **kwargs):
    raise NotImplementedError("a stride-2 layer of ConvDownBlock runs inside the block's kernels only")


def _strided(m):
    """mark a weight-norm conv as a stride-2 layer of ConvDownBlock: a holder of the reference's parameters"""
    m.stride = (2, 2)
    m.forward = _block_only
    return m


class ConvDownBlock(nn.Module):
    """blocks.py:327-379: grouped weight-normalised 1x1 stride-2 skip with tied bias, 3x3 Conv2dWNUB + LeakyReLU at the
    input size, 3x3 stride-2 Conv2dWNUB + LeakyReLU; the whole block runs on the two fused kernels of
    csrc/downconv_wnub.cu, and `lrelu1` / `lrelu2` are parameter-free placeholders.  `size` is the INPUT size; the
    output is [B, Cout, size/2, size/2].  Parameter names and shapes are the reference's.

    forward(x, resize_mask=None, scale=1.0): with a bool `resize_mask` [.., size, size] the block's input is
    scale * bilinear(x -> size x size, align_corners=False) * resize_mask, computed inside the kernels from x
    [B, Cin, Hs, Ws], which may be a strided window of a larger map (unit stride along a row); that input is never
    written, and no gradient reaches x through it (asking for one raises)."""

    def __init__(self, in_channels, out_channels, size, lrelu_slope=0.2, groups=1, wnorm_dim=0):
        super().__init__()
        if wnorm_dim != 0:
            raise NotImplementedError("only wnorm_dim = 0 (g per output channel) is supported")
        if in_channels % groups or out_channels % groups or size % 2:
            raise ValueError("channels must divide into groups and size must be even")
        self.size, self.groups, self.lrelu_slope = size, groups, float(lrelu_slope)
        self.conv_resize = _strided(_grouped(Conv2dWN(in_channels, out_channels, kernel_size=1), groups))
        self.conv1 = _grouped(Conv2dWNUB(in_channels, in_channels, size, size, 3, 1, 1), groups)
        self.lrelu1 = FusedLeakyReLU()
        self.conv2 = _strided(_grouped(Conv2dWNUB(in_channels, out_channels, size // 2, size // 2, 3, 1, 1), groups))
        self.lrelu2 = FusedLeakyReLU()

    def forward(self, x, resize_mask=None, scale: float = 1.0):
        if resize_mask is None:
            if x.dim() != 4 or tuple(x.shape[2:]) != (self.size, self.size):
                raise RuntimeError("ConvDownBlock(size=%d) needs a [B, C, %d, %d] input (got %s)"
                                   % (self.size, self.size, self.size, tuple(x.shape)))
        else:
            if resize_mask.dtype != torch.bool or tuple(resize_mask.shape[-2:]) != (self.size, self.size):
                raise RuntimeError("resize_mask must be a bool [.., %d, %d] tensor" % (self.size, self.size))
            if torch.is_grad_enabled() and x.requires_grad:
                raise RuntimeError("ConvDownBlock: the fused resize + mask of the input has no backward, and the input "
                                   "requires grad")
        c1, c2, cr = self.conv1, self.conv2, self.conv_resize
        return _DownConvBlock.apply(x, c1.weight_v, c1.weight_g, c1.bias, c2.weight_v, c2.weight_g, c2.bias,
                                    cr.weight_v, cr.weight_g, cr.bias, self.lrelu_slope, self.groups, resize_mask,
                                    scale)
