"""render_fused — project -> bin/sort -> pack -> one 4-channel blend, as a single autograd node (SURVEY.md §8f-1).

Equivalent, output for output, to the reference's call sequence in ca_code/utils/render_gsplat.py:41-106
(project_gaussians, rasterize rgb with opacity * compensation, rasterize depth-as-colour) — same kernels, same
arithmetic — but without the tensors that sequence materialises between the calls (`opacity * compensation[:, None]`,
`depths[:, None].expand(-1, 3)`, the second binning) and without their autograd glue in the backward."""
import os
from typing import NamedTuple

import torch
from torch.autograd import Function

from .. import _lib
from .project import _project_bwd, _project_fwd
from .utils import _tile_bounds, _workspace, bin_and_sort_gaussians, compute_cumulative_intersects, key_bits

# sync-free mode: per-device overflow flag (int32 on the device, set by the bin-edges kernel when the intersection
# count exceeded the capacity of the buffers) — read it with check_overflow() at a point where a sync is acceptable
_OVERFLOW = {}

# binning of the sync-free path: "buckets" (csrc/splat_bin_tiles.cu) or "keysort" (csrc/splat_bin.cu, the gsplat-shaped
# pipeline: cumsum -> keys -> radix sort -> bin edges -> pack); identical outputs, the switch exists for A/B timing
BINNING = os.environ.get("GOLIATH_B200_BINNING", "buckets")
# sync-free path on the bucket binning: "1" runs it as _RenderBuckets (ranked or packed records, see RANKED; with ranked
# records render_views has the blend kernels finish the view), "0" as _RenderFused (packed records).  The name is
# kept from when the first choice was two autograd nodes, projection | binning + blend.
SPLIT = os.environ.get("GOLIATH_B200_RENDER_SPLIT", "1") != "0"
# records of the bucket path: "ranked" (default: the blend stages records by Gaussian id from the per-Gaussian table,
# G x 48 B, with 16-byte cp.async gathers) or "packed" (sorted 48-byte records materialised by the binning's gather,
# cap x 48 B).  On an H100 the by-id table (14.4 MB at 300k Gaussians) stays in the 50 MB L2 between the binning and
# the two blends, the sorted records (52 MB on the bench head scene) do not.  Measured on an H100 SXM at a 700 W power
# limit (scripts/profile_head_step.py): the ranked blends cost ~2 us (forward) and ~10 us (backward) more than the
# packed ones, the record gather they make unnecessary cost ~50 us, and the bench head step takes 0.557 instead of
# 0.592 ms.  The ranked path also holds 4x less memory per view for the backward.  "packed" is kept for A/B timing;
# _RenderFused and OLAT always use packed records.
RANKED = os.environ.get("GOLIATH_B200_RECORDS", "ranked") == "ranked"


def _overflow_flag(dev):
    f = _OVERFLOW.get(dev.index)
    if f is None:
        f = torch.zeros(1, dtype=torch.int32, device=dev)
        _OVERFLOW[dev.index] = f
    return f


def check_overflow(device=None) -> bool:
    """True if any sync-free render on `device` since the last check dropped intersections (capacity too small).
    Synchronises; call it once per step / per epoch, not per render."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    f = _OVERFLOW.get(dev.index)
    if f is None:
        return False
    hit = bool(f.item())
    if hit:
        f.zero_()
    return hit


class _BlendPlan(NamedTuple):
    sched: int  # 1: the tile order is an SM-affine schedule (gb_tile_schedule) the blend kernels draw their tiles from
    order_len: int  # int32 entries of the tile order
    fwd: object  # gb_rasterize_{sched,packed}_fwd
    bwd: object  # gb_rasterize_{sched,packed}_bwd
    ranked: bool  # _RenderBuckets blends id-staged records (gb_rasterize_ranked_*, see RANKED)


def _blend_plan(T, schedule=True):
    """How the blend mode (gb_get_blend_mode) maps to a tile order and to the rasterize entry points of a render over T
    tiles.  Blend modes 2 and 4 take an SM-affine schedule; `schedule=False` (the exact path, whose tile order is always
    gb_tile_order) keeps the launch-order tiles in every mode."""
    L = _lib.kernels()
    mode = L.gb_get_blend_mode()
    sched = 1 if schedule and mode in (2, 4) else 0
    return _BlendPlan(sched, L.gb_tile_schedule_ints(T) if sched else T,
                      L.gb_rasterize_sched_fwd if sched else L.gb_rasterize_packed_fwd,
                      L.gb_rasterize_sched_bwd if sched else L.gb_rasterize_packed_bwd,
                      RANKED and not sched and mode == 3)


def _bin_tiles(xys, depths, radii, conics, colors, opacity, comp, H, W, cap, plan, outs, ranked=False, n_out=None,
               colors_ready=None):
    """Bucket binning (csrc/splat_bin_tiles.cu) on the current stream, into the caller's `outs`: (gids [cap], records
    [cap,12]) for gb_bin_tiles_pack_ev, or with `ranked` (ranks [cap], bucket [cap], records [G,12], gids [G]) for
    gb_bin_tiles_buckets, which leaves each tile unsorted for gb_rasterize_ranked_fwd_sort_lists.  `n_out` (device int32) receives the intersection count, `colors_ready` is the raw handle of
    an event to wait for before the colours are read; either may be None.  Returns (bins [T,2], order)."""
    G = xys.size(0)
    dev = xys.device
    L = _lib.kernels()
    tb = _tile_bounds(H, W, 16)
    T = tb[0] * tb[1]
    bins = torch.empty(T, 2, device=dev, dtype=torch.int32)
    order = torch.empty(plan.order_len, device=dev, dtype=torch.int32)
    ws = _workspace(dev, L.gb_bin_tiles_workspace_bytes(G, T, cap))
    args = (G, xys, depths, radii, conics, colors, opacity, comp, H, W, 16, cap, bins, order)
    tail = (n_out, _overflow_flag(dev), ws, colors_ready)
    if ranked:  # launch-order tiles (the ranked plan never takes the SM-affine schedule)
        L.gb_bin_tiles_buckets(*args, *outs, *tail)
    else:
        L.gb_bin_tiles_pack_ev(*args, plan.sched, *outs, *tail)
    return bins, order


def _blend_grads(H, W, v_out4, v_alpha, opacity, comp, blend, v_colors=None):
    """Gradients through a blend.  `blend(v_out4, v_alpha, v_xy, v_conic, v_col4, v_opeff)` issues the rasterize
    backward(s) on the current stream; they accumulate atomically into the last four arrays, which are zeroed here with
    one fill.  gb_splat_grad_unpack then turns v_col4 / v_opeff into the gradients of the colours (into `v_colors` when
    given), opacity, compensation and depth.  Returns (v_xy, v_conic, v_colors, v_opacity, v_comp, v_depth)."""
    G = comp.size(0)
    dev = comp.device
    f32 = dict(device=dev, dtype=torch.float32)
    v_out4 = torch.zeros(H, W, 4, **f32) if v_out4 is None else v_out4.contiguous()
    v_alpha = None if v_alpha is None else v_alpha.contiguous()  # NULL: no gradient through alpha (no zero fill)
    acc = torch.zeros(G * 10, **f32)  # the four atomically-accumulated gradient arrays, one fill
    v_xy, v_conic = acc[:2 * G].view(G, 2), acc[2 * G:5 * G].view(G, 3)
    v_col4, v_opeff = acc[5 * G:9 * G].view(G, 4), acc[9 * G:]
    v_colors = torch.empty(G, 3, **f32) if v_colors is None else v_colors
    v_opacity, v_comp, v_depth = torch.empty(G, 1, **f32), torch.empty(G, **f32), torch.empty(G, **f32)
    blend(v_out4, v_alpha, v_xy, v_conic, v_col4, v_opeff)
    _lib.kernels().gb_splat_grad_unpack(G, v_col4, v_opeff, opacity, comp, v_colors, v_opacity, v_comp, v_depth)
    return v_xy, v_conic, v_colors, v_opacity, v_comp, v_depth


class _RenderFused(Function):
    @staticmethod
    def forward(ctx, means3d, scales, quats, opacity, colors, viewmat, background, glob_scale, fx, fy, cx, cy, img_height,
                img_width, clip_thresh, capacity):
        ins = [t.contiguous() for t in (means3d, scales, quats, opacity, colors, viewmat, background)]
        for t, n in zip(ins, ("means3d", "scales", "quats", "opacity", "colors", "viewmat", "background")):
            _lib.check_input(t, n)
        means3d, scales, quats, opacity, colors, viewmat, background = ins
        G = means3d.size(0)
        if G == 0:
            capacity = None  # nothing to bin: the exact path below returns the background (no device-side count to read)
        dev = means3d.device
        L = _lib.kernels()
        f32 = dict(device=dev, dtype=torch.float32)
        i32 = dict(device=dev, dtype=torch.int32)
        H, W, BW = int(img_height), int(img_width), 16
        out4 = torch.empty(H, W, 4, **f32)
        final_Ts = torch.empty(H, W, **f32)
        final_idx = torch.empty(H, W, **i32)
        bg4 = torch.cat([background, background[:1]])
        xys, depths, radii, conics, comp, num_tiles_hit, cov3d = _project_fwd(
            means3d, scales, quats, viewmat, glob_scale, fx, fy, cx, cy, H, W, BW, clip_thresh)
        tb = _tile_bounds(H, W, BW)
        T = tb[0] * tb[1]
        plan = _blend_plan(T, schedule=capacity is not None)
        if capacity is not None:
            # ---- sync-free path: the count never visits the host; buffers hold `capacity` intersections
            cap = num_intersects = int(capacity)  # "some": the backward walks the bins, not the count
            gids = torch.empty(cap, **i32)
            records = torch.empty(cap, 12, **f32)
            if BINNING == "buckets" and L.gb_bin_tiles_supported(G):
                # per-tile buckets, each sorted by (depth, id) in shared memory (csrc/splat_bin_tiles.cu): same
                # bins, ids and records as the key sort below, without sorting the intersection keys globally
                bins, order = _bin_tiles(xys, depths, radii, conics, colors, opacity, comp, H, W, cap, plan,
                                         (gids, records))
            else:
                order = torch.empty(plan.order_len, **i32)
                cum = torch.empty_like(num_tiles_hit)
                ws = _workspace(dev, max(L.gb_cumsum_workspace_bytes(G), L.gb_sort_workspace_bytes(cap)))
                L.gb_cumsum_i32(G, num_tiles_hit, cum, ws)
                n_dev = cum.data_ptr() + 4 * (G - 1)
                isect = torch.empty(cap, device=dev, dtype=torch.int64)
                gids_u = torch.empty(cap, **i32)
                isect_s = torch.empty(cap, device=dev, dtype=torch.int64)
                bins = torch.zeros(T, 2, **i32)
                L.gb_map_gaussian_to_intersects_dn(G, xys, depths, radii, cum, H, W, BW, cap, isect, gids_u)
                L.gb_sort_intersects_dn(cap, n_dev, isect, gids_u, isect_s, gids, key_bits(T), ws)
                L.gb_get_tile_bin_edges_dn(cap, n_dev, isect_s, bins, _overflow_flag(dev))
                (L.gb_tile_schedule if plan.sched else L.gb_tile_order)(T, bins, order)
                L.gb_pack_records_fused_dn(cap, n_dev, gids, xys, conics, colors, depths, opacity, comp, records)
        else:
            num_intersects, cum = compute_cumulative_intersects(num_tiles_hit)
            if num_intersects < 1:
                # reference behaviour with nothing to draw (gsplat 0.1.11 rasterize.py): background, final_Ts = 0
                out4.copy_(bg4.expand(H, W, 4))
                final_Ts.zero_()
                final_idx.zero_()
                gids = bins = order = records = torch.empty(0, **i32)
            else:
                _, _, _, gids, bins = bin_and_sort_gaussians(G, num_intersects, xys, depths, radii, cum, tb, BW)
                order = torch.empty(T, **i32)
                records = torch.empty(num_intersects, 12, **f32)
                L.gb_tile_order(T, bins, order)
                L.gb_pack_records_fused(num_intersects, gids, xys, conics, colors, depths, opacity, comp, records)
        if capacity is not None or num_intersects >= 1:
            plan.fwd(H, W, 4, bins, order, records, bg4, out4, final_Ts, final_idx)
        ctx.save_for_backward(means3d, scales, quats, opacity, viewmat, bg4, cov3d, radii, conics, comp, gids, bins, order,
                              records, final_Ts, final_idx)
        ctx.meta = (H, W, num_intersects, float(glob_scale), float(fx), float(fy), plan)
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)
        return out4, 1 - final_Ts, radii

    @staticmethod
    def backward(ctx, v_out4, v_alpha, _v_radii):
        (means3d, scales, quats, opacity, viewmat, bg4, cov3d, radii, conics, comp, gids, bins, order, records, final_Ts,
         final_idx) = ctx.saved_tensors
        H, W, num_intersects, glob_scale, fx, fy, plan = ctx.meta

        def blend(*grads):
            if num_intersects >= 1:
                plan.bwd(H, W, 4, gids, bins, order, records, bg4, final_Ts, final_idx, *grads)

        v_xy, v_conic, v_colors, v_opacity, v_comp, v_depth = _blend_grads(H, W, v_out4, v_alpha, opacity, comp, blend)
        g_mean, g_scale, g_quat = _project_bwd(means3d, scales, quats, viewmat, cov3d, radii, conics, comp, glob_scale,
                                               fx, fy, v_xy, v_depth, v_conic, v_comp)
        return (g_mean, g_scale, g_quat, v_opacity, v_colors) + (None,) * 11


def _acc_parts(acc, G):
    """(v_rgbd [G,4], v_xy [G,2], v_conic [G,3], v_opacity_eff [G]): the blend backward's accumulator as
    gb_project_gaussians_fwd_acc lays it out and zeroes it, and gb_splat_project_bwd reads it."""
    return acc[:4 * G].view(G, 4), acc[4 * G:6 * G].view(G, 2), acc[6 * G:9 * G].view(G, 3), acc[9 * G:]


class _RenderBuckets(Function):
    """The sync-free render on the bucket binning (csrc/splat_bin_tiles.cu) as one autograd node: projection ->
    binning -> blend.  The projection kernel also zeroes the blend backward's accumulator, and the backward turns it
    into every input gradient with one per-Gaussian kernel (gb_splat_project_bwd).  `colors` may still be in flight on
    another stream: `colors_event` (torch.cuda.Event recorded after the kernel that writes them) is waited for inside
    the binning, just before the colours are first read.

    `finish` (ranked records only, see RANKED): the blend kernels also finish the view as render._FinishView does, and
    the node returns (rgb [3,H,W], alpha [1,H,W] (no gradient), depth [1,H,W], radii); without it (out4 [H,W,4],
    alpha [H,W], radii)."""

    @staticmethod
    def forward(ctx, means3d, scales, quats, opacity, colors, viewmat, background, glob_scale, fx, fy, cx, cy,
                img_height, img_width, clip_thresh, capacity, colors_event, finish):
        names = ("means3d", "scales", "quats", "opacity", "colors", "viewmat", "background")
        ins = [t.contiguous() for t in (means3d, scales, quats, opacity, colors, viewmat, background)]
        for t, n in zip(ins, names):
            _lib.check_input(t, n)
        means3d, scales, quats, opacity, colors, viewmat, background = ins
        G = means3d.size(0)
        dev = means3d.device
        L = _lib.kernels()
        f32 = dict(device=dev, dtype=torch.float32)
        i32 = dict(device=dev, dtype=torch.int32)
        H, W = int(img_height), int(img_width)
        tb = _tile_bounds(H, W, 16)
        cap = int(capacity)
        plan = _blend_plan(tb[0] * tb[1])
        if finish and not plan.ranked:
            raise ValueError("the blend kernels finish the view only with ranked records (see blend_finishes_view)")
        acc = torch.empty(10 * G, **f32)
        xys, depths, radii, conics, comp, _, cov3d = _project_fwd(means3d, scales, quats, viewmat, glob_scale, fx, fy,
                                                                  cx, cy, H, W, 16, clip_thresh, grad_acc=acc)
        final_Ts = torch.empty(H, W, **f32)
        final_idx = torch.empty(H, W, **i32)
        ev = None
        if colors_event is not None:
            ev = colors_event.cuda_event
            colors.record_stream(torch.cuda.current_stream(dev))
        # id-staged records (the default with the mom blend and launch-order tiles): the blend gathers each stage
        # from the by-id table, the sorted 48-byte records are never materialised (csrc/splat_blend_mom.cu, RANKED)
        if plan.ranked:
            gids = torch.empty(G, **i32)            # identity (the C ABI's rank_to_gid)
            ranks = torch.empty(cap, **i32)         # per tile: depth keys, then (after the forward) ids in blend order
            bucket = torch.empty(cap, **i32)        # per tile: Gaussian ids in arbitrary order
            records = torch.empty(G, 12, **f32)     # one record per Gaussian, by id
            outs = (ranks, bucket, records, gids)
        else:
            gids = torch.empty(cap, **i32)
            ranks = gids  # unused
            records = torch.empty(cap, 12, **f32)
            outs = (gids, records)
        bins, order = _bin_tiles(xys, depths, radii, conics, colors, opacity, comp, H, W, cap, plan, outs,
                                 ranked=plan.ranked, colors_ready=ev)
        hit_list = hit_count = None
        bg = background if finish else torch.cat([background, background[:1]])
        if plan.ranked:
            # each forward CTA sorts its tile's bucket into `ranks` before it blends the tile, and stores each
            # pixel warp's hits (sorted indices; 8 x cap int32 needs no device-side count) so that the backward
            # walks them instead of culling every tile again
            hit_list = torch.empty(8 * cap, **i32)
            hit_count = torch.empty(16 * tb[0] * tb[1] + 2, **i32)
            head = (bins, order, depths, bucket, ranks, records, bg)
            tail = (final_Ts, final_idx, hit_list, hit_count)
            if finish:
                rgb, a_img, depth = torch.empty(3, H, W, **f32), torch.empty(1, H, W, **f32), torch.empty(1, H, W, **f32)
                L.gb_rasterize_ranked_fwd_sort_finish(H, W, *head, rgb, a_img, depth, *tail)
            else:
                out4 = torch.empty(H, W, 4, **f32)
                L.gb_rasterize_ranked_fwd_sort_lists(H, W, 4, *head, out4, *tail)
        else:
            out4 = torch.empty(H, W, 4, **f32)
            plan.fwd(H, W, 4, bins, order, records, bg, out4, final_Ts, final_idx)
        alpha = a_img if finish else None
        ctx.save_for_backward(means3d, scales, quats, opacity, viewmat, bg, cov3d, radii, conics, comp, acc, gids, bins,
                              order, records, final_Ts, final_idx, ranks, hit_list, hit_count, alpha)
        ctx.meta = (H, W, float(glob_scale), float(fx), float(fy), plan, finish)
        ctx.acc_used = False
        ctx.set_materialize_grads(False)
        if finish:
            ctx.mark_non_differentiable(a_img, radii)
            return rgb, a_img, depth, radii
        ctx.mark_non_differentiable(radii)
        return out4, 1 - final_Ts, radii

    @staticmethod
    def backward(ctx, *grads):
        (means3d, scales, quats, opacity, viewmat, bg, cov3d, radii, conics, comp, acc, gids, bins, order, records,
         final_Ts, final_idx, ranks, hit_list, hit_count, alpha) = ctx.saved_tensors
        H, W, glob_scale, fx, fy, plan, finish = ctx.meta
        G = means3d.size(0)
        dev = means3d.device
        L = _lib.kernels()
        f32 = dict(device=dev, dtype=torch.float32)
        if ctx.acc_used:  # a second backward through this graph (retain_graph): the projection zeroed acc only once
            acc.zero_()
        ctx.acc_used = True
        v_col4, v_xy, v_conic, v_opeff = _acc_parts(acc, G)
        v_colors, v_opacity = torch.empty(G, 3, **f32), torch.empty(G, 1, **f32)
        g_mean, g_scale, g_quat = torch.empty(G, 3, **f32), torch.empty(G, 3, **f32), torch.empty(G, 4, **f32)
        accs = (v_xy, v_conic, v_col4, v_opeff)
        if finish:
            g_rgb, _, g_depth, _ = (None if g is None else g.contiguous() for g in grads)
            L.gb_rasterize_ranked_bwd_lists_finish(
                H, W, ranks, bins, hit_list, hit_count, records, bg, final_Ts, final_idx, alpha, g_rgb, g_depth,
                *accs)
        else:
            v_out4, v_alpha, _ = grads
            v_out4 = torch.zeros(H, W, 4, **f32) if v_out4 is None else v_out4.contiguous()
            v_alpha = None if v_alpha is None else v_alpha.contiguous()  # NULL: no gradient through alpha
            if plan.ranked:
                L.gb_rasterize_ranked_bwd_lists(
                    H, W, 4, ranks, bins, hit_list, hit_count, records, bg, final_Ts, final_idx, v_out4, v_alpha,
                    *accs)
            else:
                plan.bwd(H, W, 4, gids, bins, order, records, bg, final_Ts, final_idx, v_out4, v_alpha, *accs)
        L.gb_splat_project_bwd(
            G, means3d, scales, glob_scale, quats, viewmat, fx, fy, cov3d, radii, conics, comp, opacity, acc,
            v_colors, v_opacity, g_mean, g_scale, g_quat)
        return (g_mean, g_scale, g_quat, v_opacity, v_colors) + (None,) * 13


def _bucket_path(G, capacity):
    """render_fused takes the sync-free bucket path (_RenderBuckets)."""
    return (capacity is not None and SPLIT and BINNING == "buckets" and G > 0
            and bool(_lib.kernels().gb_bin_tiles_supported(G)))


def blend_finishes_view(G, capacity):
    """True when render_fused(..., finish=True) may be called for G Gaussians: the sync-free bucket path with ranked
    records, whose blend kernels write the finished view."""
    return _bucket_path(G, capacity) and _blend_plan(1).ranked


def render_fused(means3d, scales, glob_scale, quats, viewmat, fx, fy, cx, cy, img_height, img_width, opacity, colors,
                 background, clip_thresh=0.01, capacity=None, colors_event=None, finish=False):
    """Returns (out4 [H,W,4] = rgb + depth, alpha [H,W], radii [G] i32).  block_width is 16.

    capacity=None keeps the reference's behaviour (one host sync to size the intersection buffers exactly).
    capacity=N runs sync-free: buffers hold N intersections, the count stays on the device, nothing blocks the host, and
    the call can be captured in a CUDA graph; if a view ever needs more than N intersections the excess is dropped and
    `check_overflow()` reports it (results of that call are then incomplete — re-run with a larger capacity).  With
    zero intersections the sync-free path returns alpha = 0, not the reference's alpha = 1 quirk.

    finish=True (only where blend_finishes_view holds) returns the finished view instead, as render._FinishView makes it
    of out4 and alpha: (rgb [3,H,W], alpha [1,H,W] (no gradient), depth [1,H,W] / clamp(alpha, 0.05, 1), radii)."""
    if finish and not blend_finishes_view(means3d.size(0), capacity):
        raise ValueError("render_fused(finish=True) needs the sync-free bucket path with ranked records")
    if _bucket_path(means3d.size(0), capacity):
        return _RenderBuckets.apply(means3d, scales, quats, opacity, colors, viewmat, background, glob_scale, fx, fy,
                                    cx, cy, img_height, img_width, clip_thresh, capacity, colors_event, finish)
    if colors_event is not None:  # _RenderFused: the colours must be complete before its first kernel
        torch.cuda.current_stream(means3d.device).wait_event(colors_event)
    return _RenderFused.apply(means3d, scales, quats, opacity, colors, viewmat, background, glob_scale, fx, fy, cx, cy,
                              img_height, img_width, clip_thresh, capacity)
