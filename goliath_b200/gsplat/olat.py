"""render_shared — one view, C colour sets against ONE projection and ONE tile binning (BASELINE config 3, SURVEY.md section 8d:
"32 OLAT lights x 16 views": 32 lighting conditions of a view share geometry, EWA projection, tile lists and the
transmittance of every pixel; only the colours differ).

The reference reaches this case as a batch of B = C renders through rgca.AutoEncoder.render (ca_code/models/rgca.py:112-151,
driven by ca_code/utils/light_decorator.py:167), i.e. C projections, 2C binnings and 2C blends per view.  Here a view is
projected and binned once (gsplat/fused.py machinery, csrc/splat_bin_tiles.cu); condition 0 is blended with the depth
channel (4 channels); the further conditions go FOUR AT A TIME through blend kernels that walk the tile lists once per
group — alphas, transmittances, culling and (backward) the whole v_sigma machinery are shared by the four colour sets
(csrc/splat_blend_mom.cu, gb_rasterize_multi_*; "wide" 80-byte records whose colour part is rewritten per group).
MODE = "single" keeps the one-condition-per-pass formulation (in-place recolouring of the 48-byte records + 3-channel
blends) for A/B timing and the tests.  The backward mirrors the forward: geometry gradients (xy, conic, opacity)
accumulate over the conditions in the same buffers, colour gradients land per condition, one projection backward."""
import os
from typing import Dict, Optional, Sequence

import torch
from torch.autograd import Function

from .. import _lib
from .fused import _bin_tiles, _blend_grads, _blend_plan
from .project import _project_bwd, _project_fwd
from .utils import _tile_bounds

MODE = os.environ.get("GOLIATH_B200_OLAT", "multi")  # "multi": four conditions per blend pass; "single": one


class _RenderShared(Function):
    @staticmethod
    def forward(ctx, means3d, scales, quats, opacity, colors, viewmat, background, glob_scale, fx, fy, cx, cy, img_height,
                img_width, clip_thresh, capacity):
        ins = [t.contiguous() for t in (means3d, scales, quats, opacity, colors, viewmat, background)]
        for t, n in zip(ins, ("means3d", "scales", "quats", "opacity", "colors", "viewmat", "background")):
            _lib.check_input(t, n)
        means3d, scales, quats, opacity, colors, viewmat, background = ins
        if colors.dim() != 3 or colors.shape[1:] != (means3d.size(0), 3):
            raise RuntimeError("render_shared: colors must be [C,G,3]")
        C, G = colors.shape[0], means3d.size(0)
        dev = means3d.device
        L = _lib.kernels()
        if not L.gb_bin_tiles_supported(G):
            raise RuntimeError("render_shared: %d Gaussians exceed the bucket binning's range (gb_bin_tiles_supported)" % G)
        f32 = dict(device=dev, dtype=torch.float32)
        i32 = dict(device=dev, dtype=torch.int32)
        H, W, BW = int(img_height), int(img_width), 16
        out4 = torch.empty(H, W, 4, **f32)
        rgb = torch.empty(C, H, W, 3, **f32)
        final_Ts = torch.empty(H, W, **f32)
        final_idx = torch.empty(H, W, **i32)
        scratch_T, scratch_idx = torch.empty(H, W, **f32), torch.empty(H, W, **i32)  # conditions > 0 rewrite the same values
        bg4 = torch.cat([background, background[:1]])
        xys, depths, radii, conics, comp, num_tiles_hit, cov3d = _project_fwd(
            means3d, scales, quats, viewmat, glob_scale, fx, fy, cx, cy, H, W, BW, clip_thresh)
        n_isect = None
        if capacity is None:  # reference-like exact buffers: one host sync for the intersection count
            n_isect = int(num_tiles_hit.sum().item())
            cap = max(n_isect, 1)
        else:
            cap = int(capacity)
        tb = _tile_bounds(H, W, BW)
        plan = _blend_plan(tb[0] * tb[1])
        gids = torch.empty(cap, **i32)
        records = torch.empty(cap, 12, **f32)
        n_dev = torch.empty(1, **i32)
        bins, order = _bin_tiles(xys, depths, radii, conics, colors[0], opacity, comp, H, W, cap, plan, (gids, records),
                                 n_out=n_dev)
        plan.fwd(H, W, 4, bins, order, records, bg4, out4, final_Ts, final_idx)
        if n_isect == 0:
            # as render_fused(capacity=None): the reference's final_Ts = 0 when nothing is drawn, so alpha = 1
            final_Ts.zero_()
            final_idx.zero_()
        rgb[0].copy_(out4[..., :3])
        multi = MODE == "multi" and C > 1
        wide = None
        if multi:
            wide = torch.empty(cap, 20, **f32)
            L.gb_records_widen(cap, n_dev, records, wide)
            stage = torch.empty(4, H, W, 3, **f32)  # a group's four images (the last group may be partial)
            for c in range(1, C, 4):
                nk = min(4, C - c)
                L.gb_records_set_colors4(cap, n_dev, gids, colors[c], nk, G, wide)
                dst = rgb[c:c + 4] if nk == 4 else stage
                L.gb_rasterize_multi_fwd(H, W, bins, order, plan.sched, wide, background, dst)
                if nk < 4:
                    rgb[c:c + nk].copy_(stage[:nk])
        else:
            for c in range(1, C):
                L.gb_records_set_colors(cap, n_dev, gids, colors[c], depths, records)
                plan.fwd(H, W, 3, bins, order, records, background, rgb[c], scratch_T, scratch_idx)
        ctx.save_for_backward(means3d, scales, quats, opacity, colors, viewmat, bg4, cov3d, depths, radii, conics, comp, gids,
                              bins, order, records, n_dev, final_Ts, final_idx)
        ctx.wide = wide  # scratch of the multi-condition passes (colour part rewritten per group in the backward)
        ctx.meta = (C, G, H, W, cap, float(glob_scale), float(fx), float(fy), plan)
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)
        return rgb, out4[..., 3], 1 - final_Ts, radii

    @staticmethod
    def backward(ctx, v_rgb, v_depth, v_alpha, _v_radii):
        (means3d, scales, quats, opacity, colors, viewmat, bg4, cov3d, depths, radii, conics, comp, gids, bins, order, records,
         n_dev, final_Ts, final_idx) = ctx.saved_tensors
        C, G, H, W, cap, glob_scale, fx, fy, plan = ctx.meta
        dev = means3d.device
        L = _lib.kernels()
        f32 = dict(device=dev, dtype=torch.float32)
        v_rgb = torch.zeros(C, H, W, 3, **f32) if v_rgb is None else v_rgb.contiguous()
        v_out4 = torch.empty(H, W, 4, **f32)
        v_out4[..., :3] = v_rgb[0]
        if v_depth is None:
            v_out4[..., 3].zero_()
        else:
            v_out4[..., 3] = v_depth
        wide = ctx.wide
        v_colors = (torch.empty if wide is not None else torch.zeros)(C, G, 3, **f32)  # multi: every table is overwritten

        def blend(v_out4, v_alpha, v_xy, v_conic, v_col4, v_opeff):
            zero_alpha = None  # the conditions after the first carry no alpha gradient
            bg3 = bg4[:3].contiguous()
            if wide is not None:
                # four conditions per pass: colour gradients arrive interleaved [G,12] and are split per group
                v12 = torch.zeros(G, 12, **f32)
                stage = torch.zeros(4, H, W, 3, **f32)
                for c in range(1, C, 4):
                    nk = min(4, C - c)
                    L.gb_records_set_colors4(cap, n_dev, gids, colors[c], nk, G, wide)
                    src = v_rgb[c:c + 4]
                    if nk < 4:
                        stage[:nk].copy_(v_rgb[c:c + nk])
                        src = stage
                    L.gb_rasterize_multi_bwd(H, W, gids, bins, order, plan.sched, wide, bg3, final_Ts, final_idx, src,
                                             v_xy, v_conic, v12, v_opeff)
                    L.gb_colors12_unpack(G, nk, v12, v_colors[c])
            else:
                # the records hold the colours of condition C-1 (left by the forward): walk the conditions downwards
                for c in range(C - 1, 0, -1):
                    if c != C - 1:
                        L.gb_records_set_colors(cap, n_dev, gids, colors[c], depths, records)
                    plan.bwd(H, W, 3, gids, bins, order, records, bg3, final_Ts, final_idx, v_rgb[c], zero_alpha, v_xy,
                             v_conic, v_colors[c], v_opeff)
                if C > 1:
                    L.gb_records_set_colors(cap, n_dev, gids, colors[0], depths, records)
            plan.bwd(H, W, 4, gids, bins, order, records, bg4, final_Ts, final_idx, v_out4, v_alpha, v_xy, v_conic,
                     v_col4, v_opeff)

        v_xy, v_conic, _, v_opacity, v_comp, v_dep = _blend_grads(H, W, v_out4, v_alpha, opacity, comp, blend, v_colors[0])
        g_mean, g_scale, g_quat = _project_bwd(means3d, scales, quats, viewmat, cov3d, radii, conics, comp, glob_scale,
                                               fx, fy, v_xy, v_dep, v_conic, v_comp)
        return (g_mean, g_scale, g_quat, v_opacity, v_colors) + (None,) * 11


def render_shared(means3d, scales, glob_scale, quats, viewmat, fx, fy, cx, cy, img_height, img_width, opacity, colors,
                  background, clip_thresh=0.01, capacity=None):
    """colors [C,G,3]: C colour sets of the same Gaussians.  Returns (rgb [C,H,W,3], depth_raw [H,W] (blended depth,
    not yet divided by alpha), alpha [H,W], radii [G] i32).  capacity as in gsplat.fused.render_fused."""
    return _RenderShared.apply(means3d, scales, quats, opacity, colors, viewmat, background, glob_scale, fx, fy, cx, cy,
                               img_height, img_width, clip_thresh, capacity)


def render_views_shared(width: int, height: int, Rt: torch.Tensor, geom: Dict[str, torch.Tensor], colors: torch.Tensor,
                        intrinsics_host: Sequence, capacity: Optional[int] = None, background: Optional[torch.Tensor] = None):
    """V views x C lighting conditions of ONE decoded avatar per view-batch item (the OLAT case of the reference's
    rgca.AutoEncoder.render, rgca.py:112-151, called with B = V*C).  geom: primpos/primqvec/primscale/opacity [V,G,*];
    colors [V,C,G,3]; Rt [V,3,4]; intrinsics_host: V tuples (fx, fy, cx, cy).  Returns rgb [V,C,3,H,W] (a permuted view
    of the blended [V,C,H,W,3], as the reference returns `out_color.permute(2,0,1)`), alpha [V,1,H,W] (detached, as
    rgca.py:137), depth [V,1,H,W] = blended depth / alpha.clamp(0.05, 1)."""
    from ..render import _issue_views, _per_view

    V = Rt.shape[0]
    bg = torch.zeros(3, device=Rt.device) if background is None else background
    gp, gs, gq, go = (_per_view(geom["primpos"], V, 3), _per_view(geom["primscale"], V, 3),
                      _per_view(geom["primqvec"], V, 4), _per_view(geom["opacity"], V, 1))
    cols = [colors.reshape(colors.shape[1:])] if V == 1 else list(torch.unbind(colors, 0))

    def render_view(v):
        fx, fy, cx, cy = intrinsics_host[v]
        rgb, depth_raw, alpha, _ = render_shared(gp[v], gs[v], 1.0, gq[v], Rt[v], fx, fy, cx, cy, height, width, go[v],
                                                 cols[v], bg, 0.1, capacity)
        a = alpha.detach()
        return rgb, a, depth_raw / a.clamp(0.05, 1.0)

    rgbs, alphas, depths = zip(*_issue_views(Rt.device, V, capacity, render_view))
    return (torch.stack(rgbs).permute(0, 1, 4, 2, 3), torch.stack([a[None] for a in alphas]),
            torch.stack([d[None] for d in depths]))
