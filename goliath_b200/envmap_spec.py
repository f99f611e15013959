"""Environment-map specular branch of the RGCA decoder (ca_code/models/rgca.py:548-556) as one sm_90a kernel each way
(csrc/envmap_spec.cu): rotate the reflection vector by `lightrot`, `dir2uv` (ca_code/utils/envmap.py:284-292),
`mipmap_grid_sample` of the pre-convolved pyramid at level `sigma * 5` (ca_code/utils/mipmap_sampler.py:13-66),
`clamp(max=1) * spec_vis`.  Gradients: ref_dirs and spec_vis (the mip level is selected under no_grad upstream; the
environment map is a constant of the relighting loop and receives none)."""
import ctypes
from typing import List

import torch
from torch.autograd import Function

from . import _lib

LEVEL_SCALE = 5.0  # rgca.py:552  miplevel = sigma * 5


def _level_args(levels: List[torch.Tensor], B: int):
    q = len(levels)
    if not 1 <= q <= 8:
        raise RuntimeError("envmap_specular: 1..8 mip levels expected")
    lv = []
    for i, t in enumerate(levels):
        _lib.check_input(t, "preconv_envmap[%d]" % i)
        if t.dim() != 4 or t.shape[0] != B or t.shape[1] != 3:
            raise RuntimeError("preconv_envmap[%d] must be [B,3,H,W]" % i)
        lv.append(t)
    ptrs = (ctypes.c_void_p * q)(*[t.data_ptr() for t in lv])
    hw = (ctypes.c_int32 * (2 * q))(*[int(v) for t in lv for v in t.shape[2:]])
    return lv, ptrs, hw


class _EnvmapSpec(Function):
    @staticmethod
    def forward(ctx, ref_dirs, sigma, spec_vis, lightrot, level_scale, *levels):
        ins = [t.contiguous() for t in (ref_dirs, sigma, spec_vis, lightrot)]
        for t, n in zip(ins, ("ref_dirs", "sigma", "spec_vis", "lightrot")):
            _lib.check_input(t, n)
        ref_dirs, sigma, spec_vis, lightrot = ins
        B, G = ref_dirs.shape[0], ref_dirs.shape[1]
        if sigma.numel() != B * G or spec_vis.numel() != B * G or lightrot.shape != (B, 3, 3):
            raise RuntimeError("envmap_specular: sigma / spec_vis must be [B,G(,1)], lightrot [B,3,3]")
        lv, ptrs, hw = _level_args([t.contiguous() for t in levels], B)
        spec = torch.empty(B, G, 3, device=ref_dirs.device, dtype=torch.float32)
        with torch.cuda.device(ref_dirs.device):
            _lib.check(_lib.lib().gb_envmap_spec_fwd(B, G, len(lv), ptrs, hw, _lib.ptr(ref_dirs), _lib.ptr(sigma),
                                                     _lib.ptr(spec_vis), _lib.ptr(lightrot), float(level_scale),
                                                     _lib.ptr(spec), _lib.stream_ptr(ref_dirs.device)), "envmap_spec_fwd")
        ctx.save_for_backward(ref_dirs, sigma, spec_vis, lightrot, *lv)
        ctx.meta = (B, G, float(level_scale), spec_vis.shape)
        return spec

    @staticmethod
    def backward(ctx, g_spec):
        ref_dirs, sigma, spec_vis, lightrot, *lv = ctx.saved_tensors
        B, G, level_scale, vis_shape = ctx.meta
        lv, ptrs, hw = _level_args(list(lv), B)
        g_spec = g_spec.contiguous()
        g_dirs = torch.empty_like(ref_dirs)
        g_vis = torch.empty(vis_shape, device=ref_dirs.device, dtype=torch.float32)
        with torch.cuda.device(ref_dirs.device):
            _lib.check(_lib.lib().gb_envmap_spec_bwd(B, G, len(lv), ptrs, hw, _lib.ptr(ref_dirs), _lib.ptr(sigma),
                                                     _lib.ptr(spec_vis), _lib.ptr(lightrot), level_scale, _lib.ptr(g_spec),
                                                     _lib.ptr(g_dirs), _lib.ptr(g_vis), _lib.stream_ptr(ref_dirs.device)),
                       "envmap_spec_bwd")
        return (g_dirs, None, g_vis, None, None) + (None,) * len(lv)


def envmap_specular(preconv_envmap: List[torch.Tensor], ref_dirs, sigma, spec_vis, lightrot,
                    level_scale: float = LEVEL_SCALE) -> torch.Tensor:
    """preconv_envmap: list of q mip levels [B,3,H_l,W_l]; ref_dirs [B,G,3]; sigma [B,G]; spec_vis [B,G,1]; lightrot
    [B,3,3].  Returns spec_color [B,G,3] = mipmap_grid_sample(...).clamp(max=1) * spec_vis."""
    return _EnvmapSpec.apply(ref_dirs, sigma, spec_vis, lightrot, level_scale, *preconv_envmap)
