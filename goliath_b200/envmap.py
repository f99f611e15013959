"""Environment-map background of the relighting frame (ca_code/utils/envmap.py) on sm_90a kernels
(csrc/envmap_compose.cu):

* `rotate_envmap_mat(image, rot_mat)` (envmap.py:141-166): the environment map seen through a rotation, one texel per
  thread; batched when given [B,3,He,We] and [B,3,3].
* `compose_envmap(render, alpha, envbg, K, Rt)` (envmap.py:325-345): the blurred environment behind the render and the
  200x200 mirror ball in the bottom-right corner, two kernels (bicubic lookup + horizontal blur pass; vertical blur
  pass + composite).  K and Rt are read on the device, so the call never synchronises with the host.  The gradient
  goes to `render` only: alpha is detached in the reference (rgca.py:137,144) and envbg, K, Rt are data.
* `prefilter_envmap_sg(sigma, v, env_tex, num_samples, xi=None, seed=None)` (envmap.py:305-323): the Monte-Carlo
  spherical-Gaussian prefilter of the environment-spin mip chain, one warp per texel (csrc/envmap_prefilter.cu).

Same signatures and results as the reference; no CPU fallback."""
import ctypes

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
    _lib.kernels().gb_envmap_rotate(B, He, We, img, rot, out)
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
        _lib.kernels().gb_envmap_compose_fwd(
            B, H, W, envbg.shape[2], envbg.shape[3], render, alpha, envbg, K, Rt, Rt.shape[1], Rt.shape[2], hblur,
            out)
        ctx.bhw = (B, H, W)
        return out

    @staticmethod
    def backward(ctx, g_out):
        B, H, W = ctx.bhw
        g_out = g_out.contiguous()
        g_render = torch.empty_like(g_out)
        _lib.kernels().gb_envmap_compose_bwd(B, H, W, g_out, g_render)
        return g_render, None, None, None, None


def compose_envmap(render: torch.Tensor, alpha: torch.Tensor, envbg: torch.Tensor, K: torch.Tensor,
                   Rt: torch.Tensor) -> torch.Tensor:
    """render [B,3,H,W] (H, W >= 200), alpha [B,1,H,W], envbg [B,3,He,We], K [B,3,3], Rt [B,>=3,>=3] (world camera;
    its [:3,:3] rotates the rays).  Returns render + (1 - alpha) * clamp(blurred environment, 0, 1) with the mirror
    ball blended into the bottom-right 200x200 corner.  Differentiable w.r.t. render only."""
    return _ComposeEnvmap.apply(render, alpha, envbg, K, Rt)


def _prefilter_levels(levels, num_samples, seed=None):
    """levels: list of (sigma, v [B,3,H,W], env_tex [B,3,He,We], xi [S,B,2,H,W] or None), all run in one launch.
    Returns the prefiltered [B,3,H,W] of each level."""
    q = len(levels)
    if not 1 <= q <= 8:
        raise RuntimeError("prefilter_envmap_sg: 1..8 levels per launch")
    if int(num_samples) < 1:
        raise RuntimeError("prefilter_envmap_sg: num_samples must be >= 1")
    with_xi = levels[0][3] is not None
    B = levels[0][1].shape[0]
    hw, sig, vs, envs, xis, outs = [], [], [], [], [], []
    for sigma, v, env_tex, xi in levels:
        if not float(sigma) > 0.0:
            raise RuntimeError("prefilter_envmap_sg: sigma must be > 0 (got %r)" % (sigma,))
        if v.dim() != 4 or v.shape[0] != B or v.shape[1] != 3:
            raise RuntimeError("prefilter_envmap_sg: v must be [B,3,H,W]")
        if env_tex.dim() != 4 or env_tex.shape[:2] != v.shape[:2]:
            raise RuntimeError("prefilter_envmap_sg: env_tex must be [B,3,He,We] with the B of v")
        H, W = v.shape[2:]
        if (xi is not None) != with_xi:
            raise RuntimeError("prefilter_envmap_sg: xi must be given for every level or for none")
        if xi is not None:
            if xi.dim() == 4 and B == 1:
                xi = xi[:, None]
            if tuple(xi.shape) != (int(num_samples), B, 2, H, W):
                raise RuntimeError("prefilter_envmap_sg: xi must be [num_samples,2,H,W] (B = 1) or [num_samples,B,2,H,W]"
                                   " = %s (got %s)" % ((int(num_samples), B, 2, H, W), tuple(xi.shape)))
        ts = [t.contiguous() for t in (v, env_tex) + ((xi,) if xi is not None else ())]
        for t, n in zip(ts, ("v", "env_tex", "xi")):
            _lib.check_input(t, n)
        if len({t.device for t in ts + vs[:1]}) != 1:
            raise RuntimeError("prefilter_envmap_sg: all tensors must be on one device")
        vs.append(ts[0])
        envs.append(ts[1])
        xis.append(ts[2] if xi is not None else None)
        outs.append(torch.empty_like(ts[0]))
        hw += [H, W, env_tex.shape[2], env_tex.shape[3]]
        sig.append(float(sigma))
    if seed is None:
        seed = int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item())  # torch's default CPU generator
    ptrs = lambda ts: (ctypes.c_void_p * q)(*[t.data_ptr() for t in ts])
    # every image reaches the kernel through a host array of device pointers, so no tensor argument names the device
    with torch.cuda.device(vs[0].device):
        _lib.kernels().gb_envmap_prefilter_sg(
            B, q, (ctypes.c_int32 * (4 * q))(*[int(x) for x in hw]), (ctypes.c_float * q)(*sig), ptrs(vs), ptrs(envs),
            ptrs(xis) if with_xi else None, int(num_samples), int(seed) & (2 ** 64 - 1), ptrs(outs))
    return outs


def prefilter_envmap_sg(sigma: float, v: torch.Tensor, env_tex: torch.Tensor, num_samples: int = 1,
                        xi: torch.Tensor = None, seed: int = None) -> torch.Tensor:
    """prefilterEnvmapSG: v [B,3,H,W] (unit directions), env_tex [B,3,He,We] -> [B,3,H,W], the mean of `num_samples`
    bilinear lookups (border padding, align_corners=False) of env_tex along importance_sample_sg's directions around v
    for a spherical Gaussian of width sigma (radians).

    The draws come from a counter-based Philox stream keyed by `seed`; without one, the seed is drawn from torch's
    default CPU generator, so torch.manual_seed reproduces a run.  `xi` [num_samples,B,2,H,W] (or [num_samples,2,H,W]
    with B = 1) replaces the draws with the ones given: the tensors the reference's th.rand_like(v[:, :2]) returns, one
    per sample, for checking the arithmetic sample for sample.  No gradient."""
    return _prefilter_levels([(sigma, v, env_tex, xi)], num_samples, seed)[0]
