"""Row R2 (SURVEY.md §8a): the Gaussian heads + SH diffuse + reflection direction block of the RGCA PrimDecoder
(ca_code/models/rgca.py:506-546) and the colour compose (:557-575) as ONE fused sm_90a kernel per direction
(csrc/rgca_heads.cu) instead of ~60 eager element-wise kernels and a [B,G,3,81] temporary.

`gaussian_heads(...)` returns a dict with the reference's `preds` key names and shapes (rgca.py:574-588);
`shade_and_compose(...)` adds the SG specular term and the final colour exactly as rgca.py:557-575 does."""
from typing import Dict

import torch
from torch.autograd import Function

from . import _lib
from .sgutils import evaluate_gaussian

PRIMSCALE_RANGE = (0.1, 20.0)  # ca_code/models/rgca.py:47
_OUT = ("primpos", "primqvec", "primscale", "primscale_preclip", "opacity", "sigma", "spec_vis", "spec_dnml", "spec_nml",
        "diff_color", "ref_dirs", "primnmlbase")


class _GaussianHeads(Function):
    @staticmethod
    def forward(ctx, f_vnocond, f_vcond, postex, tn, albedo, light_sh, campos, scale_lo, scale_hi, light_sh2=None):
        ins = [t.contiguous() for t in (f_vnocond, f_vcond, postex, tn, albedo, light_sh, campos)]
        names = ("f_vnocond", "f_vcond", "postex", "tn", "albedo", "light_sh", "campos")
        for t, n in zip(ins, names):
            _lib.check_input(t, n)
        f_vnocond, f_vcond, postex, tn, albedo, light_sh, campos = ins
        B, C, H, W = f_vnocond.shape
        G = H * W
        if C != 125 or f_vcond.shape[1] != 4 or light_sh.shape[1:] != (3, 81) or albedo.numel() != G * 3:
            raise RuntimeError("gaussian_heads expects f_vnocond [B,125,H,W], f_vcond [B,4,H,W], light_sh [B,3,81], "
                               "albedo [1,H*W,3]")
        dev = f_vnocond.device
        e = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)
        outs = dict(primpos=e(B, G, 3), primqvec=e(B, G, 4), primscale=e(B, G, 3), primscale_preclip=e(B, G, 3),
                    opacity=e(B, G, 1), sigma=e(B, G), spec_vis=e(B, G, 1), spec_dnml=e(B, G, 3), spec_nml=e(B, G, 3),
                    diff_color=e(B, G, 3), ref_dirs=e(B, G, 3), primnmlbase=e(B, G, 3))
        shsum = e(B, G, 3)
        shsum2 = None
        if light_sh2 is not None:  # second light-SH table evaluated in the same pass (rgca.py:590-616)
            light_sh2 = light_sh2.contiguous()
            _lib.check_input(light_sh2, "light_sh2")
            if light_sh2.shape != light_sh.shape:
                raise RuntimeError("light_sh2 must have the shape of light_sh [B,3,81]")
            shsum2 = e(B, G, 3)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_rgca_heads_fwd(
                B, G, *[_lib.ptr(t) for t in ins], float(scale_lo), float(scale_hi),
                *[_lib.ptr(outs[k]) for k in _OUT], _lib.ptr(shsum), _lib.ptr(light_sh2), _lib.ptr(shsum2),
                _lib.stream_ptr(dev)), "rgca_heads_fwd")
        ctx.save_for_backward(*ins, shsum)
        ctx.light_sh2 = light_sh2  # constant (no gradient): built under no_grad upstream
        ctx.scale = (float(scale_lo), float(scale_hi))
        ctx.shape = (B, C, H, W)
        ctx.set_materialize_grads(False)
        return tuple(outs[k] for k in _OUT) + (shsum2,)

    @staticmethod
    def backward(ctx, *gouts):
        g_shsum2 = gouts[-1]
        gouts = gouts[:-1]
        f_vnocond, f_vcond, postex, tn, albedo, light_sh, campos, shsum = ctx.saved_tensors
        B, C, H, W = ctx.shape
        G = H * W
        dev = f_vnocond.device
        gouts = [None if g is None else g.contiguous() for g in gouts]
        g_fn = torch.empty_like(f_vnocond)
        g_fv = torch.empty_like(f_vcond)
        g_pt = torch.empty_like(postex)
        g_tn = torch.empty_like(tn)
        g_al = torch.empty(B, G, 3, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_rgca_heads_bwd(
                B, G, _lib.ptr(f_vnocond), _lib.ptr(f_vcond), _lib.ptr(postex), _lib.ptr(tn), _lib.ptr(albedo),
                _lib.ptr(light_sh), _lib.ptr(campos), ctx.scale[0], ctx.scale[1], _lib.ptr(shsum),
                *[_lib.ptr(g) for g in gouts], _lib.ptr(g_fn), _lib.ptr(g_fv), _lib.ptr(g_pt), _lib.ptr(g_tn),
                _lib.ptr(g_al), _lib.ptr(ctx.light_sh2 if g_shsum2 is not None else None),
                _lib.ptr(None if g_shsum2 is None or ctx.light_sh2 is None else g_shsum2.contiguous()),
                _lib.stream_ptr(dev)), "rgca_heads_bwd")
        g_albedo = g_al.sum(0, keepdim=True).view_as(albedo) if ctx.needs_input_grad[4] else None
        return g_fn, g_fv, g_pt, g_tn, g_albedo, None, None, None, None, None


def gaussian_heads(f_vnocond, f_vcond, postex, tn, albedo, headrel_light_sh, headrel_campos,
                   primscale_range=PRIMSCALE_RANGE, rand_light_sh=None) -> Dict[str, torch.Tensor]:
    """f_vnocond [B,125,H,W] and f_vcond [B,4,H,W] are the decoder towers' raw outputs (rgca.py:495,503), postex the UV
    position map, tn the UNIT normal map (rgca.py:483-491), albedo the [1,H*W,3] parameter, headrel_light_sh [B,3,81],
    headrel_campos [B,3].  Returns the reference's per-Gaussian tensors plus `ref_dirs`.  With `rand_light_sh`
    [B,3,81] (the training-mode random back light, rgca.py:590-616) the result also holds `diff_color_rand` [B,G,3] =
    (diff_shs * rand_light_sh[:, None]).sum(-1), computed in the same pass over the 113 diffuse planes."""
    outs = _GaussianHeads.apply(f_vnocond, f_vcond, postex, tn, albedo, headrel_light_sh, headrel_campos,
                                primscale_range[0], primscale_range[1], rand_light_sh)
    d = dict(zip(_OUT, outs[:-1]))
    if rand_light_sh is not None:
        d["diff_color_rand"] = outs[-1]
    return d


class _ShadeCompose(Function):
    """normalise + SG shade + `spec * spec_vis` + `clamp(clamp(diff, 0) + spec, 0)` as one kernel each way
    (csrc/sg_shade.cu, FUSED instantiations)."""

    @staticmethod
    def forward(ctx, ref_dirs, sigma, light_values, light_pts, prim_pts, n_lights, diff_color, spec_vis, w_type, want_spec):
        ins = [t.contiguous() for t in (ref_dirs, sigma, light_values, light_pts, prim_pts, diff_color, spec_vis)]
        for t, n in zip(ins, ("ref_dirs", "sigma", "light_values", "light_pts", "prim_pts", "diff_color", "spec_vis")):
            _lib.check_input(t, n)
        ref_dirs, sigma, light_values, light_pts, prim_pts, diff_color, spec_vis = ins
        n_lights = n_lights.int().contiguous()
        N, D, L = ref_dirs.shape[0], ref_dirs.shape[1], light_values.shape[1]
        if spec_vis.numel() != N * D or sigma.numel() != N * D or diff_color.shape != (N, D, 3):
            raise RuntimeError("shade_compose: sigma / spec_vis must be [N,D(,1)] and diff_color [N,D,3]")
        dev = ref_dirs.device
        color = torch.empty(N, D, 3, device=dev, dtype=torch.float32)
        spec = torch.empty(N, D, 3, device=dev, dtype=torch.float32) if want_spec else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_sg_shade_compose_fwd(
                _lib.ptr(ref_dirs), _lib.ptr(sigma), _lib.ptr(light_values), _lib.ptr(light_pts), _lib.ptr(prim_pts),
                _lib.ptr(n_lights), _lib.ptr(diff_color), _lib.ptr(spec_vis), _lib.ptr(color), _lib.ptr(spec), N, D, L,
                int(w_type), _lib.stream_ptr(dev)), "sg_shade_compose_fwd")
        ctx.save_for_backward(ref_dirs, sigma, light_values, light_pts, prim_pts, n_lights, diff_color, spec_vis, color)
        ctx.meta = (N, D, L, int(w_type), sigma.shape, spec_vis.shape)
        ctx.set_materialize_grads(False)
        return (color, spec) if want_spec else (color, None)

    @staticmethod
    def backward(ctx, g_color, g_spec):
        ref_dirs, sigma, light_values, light_pts, prim_pts, n_lights, diff_color, spec_vis, color = ctx.saved_tensors
        N, D, L, w_type, sig_shape, vis_shape = ctx.meta
        dev = ref_dirs.device
        f32 = dict(device=dev, dtype=torch.float32)
        if g_color is None:
            g_color = torch.zeros(N, D, 3, **f32)
        g_color = g_color.contiguous()
        g_spec = None if g_spec is None else g_spec.contiguous()
        g_dirs, g_sig = torch.empty(N, D, 3, **f32), torch.empty(sig_shape, **f32)
        g_diff, g_vis = torch.empty(N, D, 3, **f32), torch.empty(vis_shape, **f32)
        g_light = torch.zeros_like(light_values) if ctx.needs_input_grad[2] else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_sg_shade_compose_bwd(
                _lib.ptr(ref_dirs), _lib.ptr(sigma), _lib.ptr(light_values), _lib.ptr(light_pts), _lib.ptr(prim_pts),
                _lib.ptr(n_lights), _lib.ptr(diff_color), _lib.ptr(spec_vis), _lib.ptr(color), _lib.ptr(g_color),
                _lib.ptr(g_spec), _lib.ptr(g_dirs), _lib.ptr(g_sig), _lib.ptr(g_diff), _lib.ptr(g_vis), _lib.ptr(g_light),
                N, D, L, w_type, _lib.stream_ptr(dev)), "sg_shade_compose_bwd")
        return g_dirs, g_sig, g_light, None, None, None, g_diff, g_vis, None, None


def shade_compose(ref_dirs, sigma, light_intensity, light_pos, primpos, n_lights, diff_color, spec_vis, w_type: int = 0,
                  return_spec: bool = False):
    """Fused form of rgca.py:557-575: `spec = evaluate_gaussian(ref_dirs, sigma, ...) * spec_vis`,
    `color = (diff_color.clamp(min=0) + spec).clamp(min=0)`.  ref_dirs [N,D,3] un-normalised, sigma [N,D], spec_vis
    [N,D,1] or [N,D], diff_color [N,D,3].  Returns color (and spec_color when asked).  Gradients: ref_dirs, sigma,
    light_intensity, diff_color, spec_vis — the same set the unfused chain differentiates."""
    color, spec = _ShadeCompose.apply(ref_dirs, sigma, light_intensity, light_pos, primpos, n_lights, diff_color, spec_vis,
                                      w_type, return_spec)
    return (color, spec) if return_spec else color


def shade_and_compose(heads: Dict[str, torch.Tensor], light_intensity, headrel_light_pos, n_lights,
                      fused: bool = True) -> Dict[str, torch.Tensor]:
    """rgca.py:557-575 (point-light branch): SG specular via evaluate_gaussian, times spec_vis, plus clamped diffuse.
    fused=True runs it as one kernel each way (`shade_compose`); fused=False is the reference's op-by-op chain."""
    if fused:
        color, spec_color = shade_compose(heads["ref_dirs"], heads["sigma"], light_intensity, headrel_light_pos,
                                          heads["primpos"], n_lights, heads["diff_color"], heads["spec_vis"],
                                          return_spec=True)
        out = dict(heads)
        out.update(spec_color=spec_color, color=color)
        return out
    spec_color = evaluate_gaussian(heads["ref_dirs"].contiguous(), heads["sigma"].contiguous(), light_intensity.contiguous(),
                                   headrel_light_pos.contiguous(), heads["primpos"].contiguous(), n_lights.int(),
                                   w_type=0) * heads["spec_vis"]
    color = heads["diff_color"].clamp(min=0.0) + spec_color
    out = dict(heads)
    out.update(spec_color=spec_color, color=color.clamp(min=0.0))
    return out
