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
from typing import Dict, List, Optional, Sequence

import torch
from torch.autograd import Function

from .. import _lib
from .fused import _overflow_flag
from .utils import _tile_bounds, _workspace

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
        L = _lib.lib()
        if not L.gb_bin_tiles_supported(G):
            raise RuntimeError("render_shared: %d Gaussians exceed the bucket binning's range (gb_bin_tiles_supported)" % G)
        f32 = dict(device=dev, dtype=torch.float32)
        i32 = dict(device=dev, dtype=torch.int32)
        cov3d, xys, depths = torch.empty(G, 6, **f32), torch.empty(G, 2, **f32), torch.empty(G, **f32)
        radii, conics, comp = torch.empty(G, **i32), torch.empty(G, 3, **f32), torch.empty(G, **f32)
        num_tiles_hit = torch.empty(G, **i32)
        H, W, BW = int(img_height), int(img_width), 16
        out4 = torch.empty(H, W, 4, **f32)
        rgb = torch.empty(C, H, W, 3, **f32)
        final_Ts = torch.empty(H, W, **f32)
        final_idx = torch.empty(H, W, **i32)
        scratch_T, scratch_idx = torch.empty(H, W, **f32), torch.empty(H, W, **i32)  # conditions > 0 rewrite the same values
        bg4 = torch.cat([background, background[:1]])
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            _lib.check(L.gb_project_gaussians_fwd(
                G, _lib.ptr(means3d), _lib.ptr(scales), float(glob_scale), _lib.ptr(quats), _lib.ptr(viewmat), float(fx),
                float(fy), float(cx), float(cy), H, W, BW, float(clip_thresh), _lib.ptr(cov3d), _lib.ptr(xys),
                _lib.ptr(depths), _lib.ptr(radii), _lib.ptr(conics), _lib.ptr(comp), _lib.ptr(num_tiles_hit), st),
                "project_gaussians_forward")
            n_isect = None
            if capacity is None:  # reference-like exact buffers: one host sync for the intersection count
                n_isect = int(num_tiles_hit.sum().item())
                cap = max(n_isect, 1)
            else:
                cap = int(capacity)
            tb = _tile_bounds(H, W, BW)
            T = tb[0] * tb[1]
            sched = 1 if L.gb_get_blend_mode() in (2, 4) else 0
            gids = torch.empty(cap, **i32)
            order = torch.empty(L.gb_tile_schedule_ints(T) if sched else T, **i32)
            records = torch.empty(cap, 12, **f32)
            bins = torch.empty(T, 2, **i32)
            n_dev = torch.empty(1, **i32)
            ws = _workspace(dev, L.gb_bin_tiles_workspace_bytes(G, T, cap))
            col0 = colors[0]
            _lib.check(L.gb_bin_tiles_pack(G, _lib.ptr(xys), _lib.ptr(depths), _lib.ptr(radii), _lib.ptr(conics),
                                           _lib.ptr(col0), _lib.ptr(opacity), _lib.ptr(comp), H, W, BW, cap, _lib.ptr(bins),
                                           _lib.ptr(order), sched, _lib.ptr(gids), _lib.ptr(records), _lib.ptr(n_dev),
                                           _lib.ptr(_overflow_flag(dev)), _lib.ptr(ws), st), "bin_tiles_pack")
            ras_fwd = L.gb_rasterize_sched_fwd if sched else L.gb_rasterize_packed_fwd
            _lib.check(ras_fwd(H, W, 4, _lib.ptr(bins), _lib.ptr(order), _lib.ptr(records), _lib.ptr(bg4), _lib.ptr(out4),
                               _lib.ptr(final_Ts), _lib.ptr(final_idx), st), "rasterize_packed_forward")
            if n_isect == 0:
                # as render_fused(capacity=None): the reference's final_Ts = 0 when nothing is drawn, so alpha = 1
                final_Ts.zero_()
                final_idx.zero_()
            rgb[0].copy_(out4[..., :3])
            multi = MODE == "multi" and C > 1
            wide = None
            if multi:
                wide = torch.empty(cap, 20, **f32)
                _lib.check(L.gb_records_widen(cap, _lib.ptr(n_dev), _lib.ptr(records), _lib.ptr(wide), st), "records_widen")
                stage = torch.empty(4, H, W, 3, **f32)  # a group's four images (the last group may be partial)
                for c in range(1, C, 4):
                    nk = min(4, C - c)
                    _lib.check(L.gb_records_set_colors4(cap, _lib.ptr(n_dev), _lib.ptr(gids), _lib.ptr(colors[c]), nk, G,
                                                        _lib.ptr(wide), st), "records_set_colors4")
                    dst = rgb[c:c + 4] if nk == 4 else stage
                    _lib.check(L.gb_rasterize_multi_fwd(H, W, _lib.ptr(bins), _lib.ptr(order), sched, _lib.ptr(wide),
                                                        _lib.ptr(background), _lib.ptr(dst), st), "rasterize_multi_forward")
                    if nk < 4:
                        rgb[c:c + nk].copy_(stage[:nk])
            else:
                for c in range(1, C):
                    _lib.check(L.gb_records_set_colors(cap, _lib.ptr(n_dev), _lib.ptr(gids), _lib.ptr(colors[c]), _lib.ptr(depths),
                                                       _lib.ptr(records), st), "records_set_colors")
                    _lib.check(ras_fwd(H, W, 3, _lib.ptr(bins), _lib.ptr(order), _lib.ptr(records), _lib.ptr(background),
                                       _lib.ptr(rgb[c]), _lib.ptr(scratch_T), _lib.ptr(scratch_idx), st),
                               "rasterize_packed_forward")
        ctx.save_for_backward(means3d, scales, quats, opacity, colors, viewmat, bg4, cov3d, depths, radii, conics, comp, gids,
                              bins, order, records, n_dev, final_Ts, final_idx)
        ctx.wide = wide  # scratch of the multi-condition passes (colour part rewritten per group in the backward)
        ctx.meta = (C, G, H, W, cap, float(glob_scale), float(fx), float(fy), sched)
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)
        return rgb, out4[..., 3], 1 - final_Ts, radii

    @staticmethod
    def backward(ctx, v_rgb, v_depth, v_alpha, _v_radii):
        (means3d, scales, quats, opacity, colors, viewmat, bg4, cov3d, depths, radii, conics, comp, gids, bins, order, records,
         n_dev, final_Ts, final_idx) = ctx.saved_tensors
        C, G, H, W, cap, glob_scale, fx, fy, sched = ctx.meta
        dev = means3d.device
        L = _lib.lib()
        f32 = dict(device=dev, dtype=torch.float32)
        v_rgb = torch.zeros(C, H, W, 3, **f32) if v_rgb is None else v_rgb.contiguous()
        v_out4 = torch.empty(H, W, 4, **f32)
        v_out4[..., :3] = v_rgb[0]
        if v_depth is None:
            v_out4[..., 3].zero_()
        else:
            v_out4[..., 3] = v_depth
        v_alpha = None if v_alpha is None else v_alpha.contiguous()  # NULL: no gradient through alpha
        zero_alpha = None  # the conditions after the first carry no alpha gradient
        acc = torch.zeros(G * 10, **f32)  # v_xy | v_conic | v_col4 (condition 0) | v_opacity_eff: one fill
        v_xy, v_conic = acc[:2 * G].view(G, 2), acc[2 * G:5 * G].view(G, 3)
        v_col4, v_opeff = acc[5 * G:9 * G].view(G, 4), acc[9 * G:]
        v_colors = (torch.empty if ctx.wide is not None else torch.zeros)(C, G, 3, **f32)  # multi: every table is overwritten
        v_opacity = torch.empty(G, 1, **f32)
        v_comp, v_dep = torch.empty(G, **f32), torch.empty(G, **f32)
        g_cov2d, g_cov3d = torch.empty(G, 3, **f32), torch.empty(G, 6, **f32)
        g_mean, g_scale, g_quat = torch.empty(G, 3, **f32), torch.empty(G, 3, **f32), torch.empty(G, 4, **f32)
        bg3 = bg4[:3].contiguous()
        with torch.cuda.device(dev):
            st = _lib.stream_ptr(dev)
            ras_bwd = L.gb_rasterize_sched_bwd if sched else L.gb_rasterize_packed_bwd
            wide = ctx.wide
            if wide is not None:
                # four conditions per pass: colour gradients arrive interleaved [G,12] and are split per group
                v12 = torch.zeros(G, 12, **f32)
                stage = torch.zeros(4, H, W, 3, **f32)
                for c in range(1, C, 4):
                    nk = min(4, C - c)
                    _lib.check(L.gb_records_set_colors4(cap, _lib.ptr(n_dev), _lib.ptr(gids), _lib.ptr(colors[c]), nk, G,
                                                        _lib.ptr(wide), st), "records_set_colors4")
                    src = v_rgb[c:c + 4]
                    if nk < 4:
                        stage[:nk].copy_(v_rgb[c:c + nk])
                        src = stage
                    _lib.check(L.gb_rasterize_multi_bwd(H, W, _lib.ptr(gids), _lib.ptr(bins), _lib.ptr(order), sched,
                                                        _lib.ptr(wide), _lib.ptr(bg3), _lib.ptr(final_Ts), _lib.ptr(final_idx),
                                                        _lib.ptr(src), _lib.ptr(v_xy), _lib.ptr(v_conic), _lib.ptr(v12),
                                                        _lib.ptr(v_opeff), st), "rasterize_multi_backward")
                    _lib.check(L.gb_colors12_unpack(G, nk, _lib.ptr(v12), _lib.ptr(v_colors[c]), st), "colors12_unpack")
            else:
                # the records hold the colours of condition C-1 (left by the forward): walk the conditions downwards
                for c in range(C - 1, 0, -1):
                    if c != C - 1:
                        _lib.check(L.gb_records_set_colors(cap, _lib.ptr(n_dev), _lib.ptr(gids), _lib.ptr(colors[c]),
                                                           _lib.ptr(depths), _lib.ptr(records), st), "records_set_colors")
                    _lib.check(ras_bwd(H, W, 3, _lib.ptr(gids), _lib.ptr(bins), _lib.ptr(order), _lib.ptr(records), _lib.ptr(bg3),
                                       _lib.ptr(final_Ts), _lib.ptr(final_idx), _lib.ptr(v_rgb[c]), _lib.ptr(zero_alpha),
                                       _lib.ptr(v_xy), _lib.ptr(v_conic), _lib.ptr(v_colors[c]), _lib.ptr(v_opeff), st),
                               "rasterize_packed_backward")
                if C > 1:
                    _lib.check(L.gb_records_set_colors(cap, _lib.ptr(n_dev), _lib.ptr(gids), _lib.ptr(colors[0]), _lib.ptr(depths),
                                                       _lib.ptr(records), st), "records_set_colors")
            _lib.check(ras_bwd(H, W, 4, _lib.ptr(gids), _lib.ptr(bins), _lib.ptr(order), _lib.ptr(records), _lib.ptr(bg4),
                               _lib.ptr(final_Ts), _lib.ptr(final_idx), _lib.ptr(v_out4), _lib.ptr(v_alpha), _lib.ptr(v_xy),
                               _lib.ptr(v_conic), _lib.ptr(v_col4), _lib.ptr(v_opeff), st), "rasterize_packed_backward")
            _lib.check(L.gb_splat_grad_unpack(G, _lib.ptr(v_col4), _lib.ptr(v_opeff), _lib.ptr(opacity), _lib.ptr(comp),
                                              _lib.ptr(v_colors[0]), _lib.ptr(v_opacity), _lib.ptr(v_comp), _lib.ptr(v_dep),
                                              st), "splat_grad_unpack")
            _lib.check(L.gb_project_gaussians_bwd(
                G, _lib.ptr(means3d), _lib.ptr(scales), glob_scale, _lib.ptr(quats), _lib.ptr(viewmat), fx, fy,
                _lib.ptr(cov3d), _lib.ptr(radii), _lib.ptr(conics), _lib.ptr(comp), _lib.ptr(v_xy), _lib.ptr(v_dep),
                _lib.ptr(v_conic), _lib.ptr(v_comp), _lib.ptr(g_cov2d), _lib.ptr(g_cov3d), _lib.ptr(g_mean),
                _lib.ptr(g_scale), _lib.ptr(g_quat), st), "project_gaussians_backward")
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
    from ..render import _nullctx, view_streams

    V = Rt.shape[0]
    bg = torch.zeros(3, device=Rt.device) if background is None else background
    rgbs: List[torch.Tensor] = []
    alphas: List[torch.Tensor] = []
    depths: List[torch.Tensor] = []
    # independent views on a small pool of side streams (see render.render_views): their kernels overlap on the device
    pool = view_streams(Rt.device, V) if (capacity is not None and V > 1) else None
    main = torch.cuda.current_stream(Rt.device) if pool else None
    def per_view(x, last):  # views with a view / stack backward (`x[v]` would zero-fill a full-batch gradient per field)
        return [x.reshape(-1, last)] if V == 1 else [t.reshape(-1, last) for t in torch.unbind(x, 0)]
    gp, gs, gq, go = (per_view(geom["primpos"], 3), per_view(geom["primscale"], 3), per_view(geom["primqvec"], 4),
                      per_view(geom["opacity"], 1))
    cols = [colors.reshape(colors.shape[1:])] if V == 1 else list(torch.unbind(colors, 0))
    for v in range(V):
        fx, fy, cx, cy = intrinsics_host[v]
        side = pool[v % len(pool)] if pool else None
        if side is not None and v < len(pool):
            side.wait_stream(main)
        with (torch.cuda.stream(side) if side is not None else _nullctx()):
            rgb, depth_raw, alpha, _ = render_shared(gp[v], gs[v], 1.0, gq[v], Rt[v], fx, fy, cx, cy, height, width, go[v], cols[v],
                                                     bg, 0.1, capacity)
            a = alpha.detach()
            dep = depth_raw / a.clamp(0.05, 1.0)
        if side is not None:
            for t_ in (rgb, a, dep):
                t_.record_stream(main)
        rgbs.append(rgb)
        alphas.append(a[None])
        depths.append(dep[None])
    if pool:
        for side in pool[:min(V, len(pool))]:
            main.wait_stream(side)
    return torch.stack(rgbs).permute(0, 1, 4, 2, 3), torch.stack(alphas), torch.stack(depths)
