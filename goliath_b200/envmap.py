"""Environment-map background of the relighting frame (ca_code/utils/envmap.py) on sm_90a kernels
(csrc/envmap_compose.cu):

* `rotate_envmap_mat(image, rot_mat)` (envmap.py:141-166): the environment map seen through a rotation, one texel per
  thread; batched when given [B,3,He,We] and [B,3,3].
* `compose_envmap(render, alpha, envbg, K, Rt)` (envmap.py:325-345): the blurred environment behind the render and the
  200x200 mirror ball in the bottom-right corner, two kernels (bicubic lookup + horizontal blur pass; vertical blur
  pass + composite).  K and Rt are read on the device, so the call never synchronises with the host.  The gradient
  goes to `render` only: alpha is detached in the reference (rgca.py:137,144) and envbg, K, Rt are data.

Same signatures and results as the reference; no CPU fallback."""
import torch
from torch.autograd import Function

from . import _lib

BALL = 200  # envmap_to_mirrorball(200, 200, ...) pasted at [-200:, -200:]


def rotate_envmap_mat(image: torch.Tensor, rot_mat: torch.Tensor) -> torch.Tensor:
    """image [3,He,We] and rot_mat [3,3] -> [3,He,We], or batched [B,3,He,We] and [B,3,3] -> [B,3,He,We].
    No gradient (the relighting loop rotates data once per frame)."""
    batched = image.dim() == 4
    if not batched and (image.dim() != 3 or rot_mat.shape != (3, 3)):
        raise RuntimeError("rotate_envmap_mat: image must be [3,He,We] with rot_mat [3,3], or [B,3,He,We] with [B,3,3]")
    if image.requires_grad and torch.is_grad_enabled():
        raise RuntimeError("rotate_envmap_mat: no gradient is implemented for the environment map")
    img = (image if batched else image[None]).contiguous()
    rot = (rot_mat if batched else rot_mat[None]).contiguous()
    _lib.check_input(img, "image")
    _lib.check_input(rot, "rot_mat")
    B, _, He, We = img.shape
    if img.shape[1] != 3 or rot.shape != (B, 3, 3) or He < 1 or We < 1:
        raise RuntimeError("rotate_envmap_mat: image must be [B,3,He,We] and rot_mat [B,3,3]")
    out = torch.empty_like(img)
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().gb_envmap_rotate(B, He, We, _lib.ptr(img), _lib.ptr(rot), _lib.ptr(out),
                                               _lib.stream_ptr(img.device)), "envmap_rotate")
    return out if batched else out[0]


class _ComposeEnvmap(Function):
    @staticmethod
    def forward(ctx, render, alpha, envbg, K, Rt):
        if render.dim() != 4 or render.shape[1] != 3:
            raise RuntimeError("compose_envmap: render must be [B,3,H,W]")
        B, _, H, W = render.shape
        if H < BALL or W < BALL:
            raise RuntimeError("compose_envmap: the image must be at least %dx%d for the mirror ball (got %dx%d)"
                               % (BALL, BALL, H, W))
        if alpha.shape != (B, 1, H, W):
            raise RuntimeError("compose_envmap: alpha must be [B,1,H,W] = %s" % ((B, 1, H, W),))
        if envbg.dim() != 4 or envbg.shape[0] != B or envbg.shape[1] != 3:
            raise RuntimeError("compose_envmap: envbg must be [B,3,He,We] with B = %d" % B)
        if K.shape != (B, 3, 3) or Rt.dim() != 3 or Rt.shape[0] != B or Rt.shape[1] < 3 or Rt.shape[2] < 3:
            raise RuntimeError("compose_envmap: K must be [B,3,3] and Rt [B,>=3,>=3] with B = %d" % B)
        ins = [t.contiguous() for t in (render, alpha, envbg, K, Rt)]
        for t, n in zip(ins, ("render", "alpha", "envbg", "K", "Rt")):
            _lib.check_input(t, n)
        render, alpha, envbg, K, Rt = ins
        if len({t.device for t in ins}) != 1:
            raise RuntimeError("compose_envmap: all tensors must be on one device")
        out = torch.empty_like(render)
        hblur = torch.empty_like(render)
        with torch.cuda.device(render.device):
            _lib.check(_lib.lib().gb_envmap_compose_fwd(
                B, H, W, envbg.shape[2], envbg.shape[3], _lib.ptr(render), _lib.ptr(alpha), _lib.ptr(envbg), _lib.ptr(K),
                _lib.ptr(Rt), Rt.shape[1], Rt.shape[2], _lib.ptr(hblur), _lib.ptr(out), _lib.stream_ptr(render.device)),
                "envmap_compose_fwd")
        ctx.bhw = (B, H, W)
        return out

    @staticmethod
    def backward(ctx, g_out):
        B, H, W = ctx.bhw
        g_out = g_out.contiguous()
        g_render = torch.empty_like(g_out)
        with torch.cuda.device(g_out.device):
            _lib.check(_lib.lib().gb_envmap_compose_bwd(B, H, W, _lib.ptr(g_out), _lib.ptr(g_render),
                                                        _lib.stream_ptr(g_out.device)), "envmap_compose_bwd")
        return g_render, None, None, None, None


def compose_envmap(render: torch.Tensor, alpha: torch.Tensor, envbg: torch.Tensor, K: torch.Tensor,
                   Rt: torch.Tensor) -> torch.Tensor:
    """render [B,3,H,W] (H, W >= 200), alpha [B,1,H,W], envbg [B,3,He,We], K [B,3,3], Rt [B,>=3,>=3] (world camera;
    its [:3,:3] rotates the rays).  Returns render + (1 - alpha) * clamp(blurred environment, 0, 1) with the mirror
    ball blended into the bottom-right 200x200 corner.  Differentiable w.r.t. render only."""
    return _ComposeEnvmap.apply(render, alpha, envbg, K, Rt)
