"""Host-side mirror of the reference's splat render wrapper ca_code/utils/render_gsplat.py:13-108
(`render`) and of rgca.AutoEncoder.render's post-processing (ca_code/models/rgca.py:112-151).

`render(...)` keeps the reference signature and call sequence (project, rasterise rgb, rasterise depth as
colour) so that its results are comparable call-for-call; the kernels underneath are the sm_90a ones.
"""
from typing import Optional

import torch as th

from .gsplat import project_gaussians, rasterize_gaussians


def render(
    cam_img_w: int,
    cam_img_h: int,
    fx: float,
    fy: float,
    cx: float,
    cy: float,
    Rt: th.Tensor,
    primpos: th.Tensor,
    primqvec: th.Tensor,
    primscale: th.Tensor,
    opacity: th.Tensor,
    colors: th.Tensor,
    return_depth: bool = True,
    bg_color: Optional[th.Tensor] = None,
    block_width: int = 16,
    global_scale: float = 1.0,
    z_near: float = 0.1,
    fused: bool = True,
    capacity: Optional[int] = None,
):
    means3D = primpos.view(-1, 3).contiguous()
    scales = primscale.view(-1, 3).contiguous()
    rotations = primqvec.view(-1, 4).contiguous()
    opacity = opacity.view(-1, 1).contiguous()
    colors = colors.view(-1, 3).contiguous()
    if bg_color is None:
        bg_color = th.zeros(3, device=Rt.device)

    if fused and return_depth and block_width == 16:
        # one autograd node for project + bin/sort + pack + 4-channel blend (gsplat/fused.py): same kernels and
        # arithmetic as the branch below, minus the intermediate tensors and their autograd glue
        from .gsplat.fused import render_fused

        out4, alpha, radii = render_fused(means3D, scales, global_scale, rotations, Rt, fx, fy, cx, cy, cam_img_h,
                                          cam_img_w, opacity, colors, bg_color, z_near, capacity)
        return {"render": out4[..., :3].permute(2, 0, 1), "final_T": (1.0 - alpha)[None], "alpha": alpha[None],
                "radii": radii, "depth": out4[..., 3][None]}

    xys, depths, radii, conics, compensation, num_tiles_hit, cov3d = project_gaussians(
        means3D, scales, global_scale, rotations, Rt, fx, fy, cx, cy, cam_img_h, cam_img_w, block_width, z_near)

    if fused and return_depth:
        # SURVEY.md §8f-1: rgb and depth share the alphas, so one 4-channel pass gives the same pixels as the
        # reference's two 3-channel passes (render_gsplat.py:65-78 + :90-104) with half the blend work
        bg4 = th.cat([bg_color, bg_color[:1]])
        out4, alpha = rasterize_gaussians(
            xys, depths, radii, conics, num_tiles_hit, th.cat([colors, depths[:, None]], 1),
            opacity * compensation[:, None], cam_img_h, cam_img_w, block_width, bg4, return_alpha=True)
        return {"render": out4[..., :3].permute(2, 0, 1), "final_T": (1.0 - alpha)[None], "alpha": alpha[None],
                "radii": radii, "depth": out4[..., 3][None]}

    out_img, alpha = rasterize_gaussians(
        xys, depths, radii, conics, num_tiles_hit, colors, opacity * compensation[:, None], cam_img_h, cam_img_w,
        block_width, bg_color, return_alpha=True)
    assert alpha is not None
    out_color = out_img[..., :3]
    final_T = 1.0 - alpha
    out = {"render": out_color.permute(2, 0, 1), "final_T": final_T[None], "alpha": alpha[None], "radii": radii}

    if return_depth:
        out_depth = rasterize_gaussians(
            xys, depths, radii, conics, num_tiles_hit, depths[:, None].expand(-1, 3).contiguous(),
            opacity * compensation[:, None], cam_img_h, cam_img_w, block_width, bg_color, return_alpha=True)[0]
        out["depth"] = out_depth[..., 0][None]
    return out


_BLACK = {}
_VIEW_STREAMS = {}
MAX_VIEW_STREAMS = int(__import__("os").environ.get("GOLIATH_B200_VIEW_STREAMS", "4"))  # 0 / 1: views one after another


class _nullctx:
    def __enter__(self): return None
    def __exit__(self, *a): return False


def view_streams(dev, n_views):
    """Side streams for independent views of one frame (at most MAX_VIEW_STREAMS, created once per device); None when
    disabled.  The binning workspace is per (device, stream) (gsplat/utils.py), so concurrent views never share scratch."""
    n = min(int(n_views), MAX_VIEW_STREAMS)
    if n < 2:
        return None
    pool = _VIEW_STREAMS.setdefault(dev.index if dev.index is not None else th.cuda.current_device(), [])
    while len(pool) < n:
        pool.append(th.cuda.Stream(device=dev))
    return pool[:n]


def _black(dev):
    """the default background, allocated once per device"""
    t = _BLACK.get(dev)
    if t is None:
        t = _BLACK[dev] = th.zeros(3, device=dev)
    return t


class _FinishView(th.autograd.Function):
    """out4 [H,W,4] + alpha [H,W] -> (rgb [3,H,W], alpha [1,H,W], depth [1,H,W]) in one kernel (csrc/render_finish.cu)."""

    @staticmethod
    def forward(ctx, out4, alpha):
        from . import _lib
        out4, alpha = out4.contiguous(), alpha.contiguous()
        _lib.check_input(out4, "out4")
        H, W = out4.shape[0], out4.shape[1]
        dev = out4.device
        rgb = th.empty(3, H, W, device=dev)
        a_img, depth = th.empty(1, H, W, device=dev), th.empty(1, H, W, device=dev)
        with th.cuda.device(dev):
            _lib.check(_lib.lib().gb_render_finish_fwd(H, W, _lib.ptr(out4), _lib.ptr(alpha), _lib.ptr(rgb), _lib.ptr(a_img),
                                                       _lib.ptr(depth), _lib.stream_ptr(dev)), "render_finish_fwd")
        ctx.save_for_backward(alpha)
        ctx.hw = (H, W)
        ctx.mark_non_differentiable(a_img)
        ctx.set_materialize_grads(False)
        return rgb, a_img, depth

    @staticmethod
    def backward(ctx, g_rgb, _g_alpha, g_depth):
        from . import _lib
        (alpha,) = ctx.saved_tensors
        H, W = ctx.hw
        g_out4 = th.empty(H, W, 4, device=alpha.device)
        g_rgb = None if g_rgb is None else g_rgb.contiguous()
        g_depth = None if g_depth is None else g_depth.contiguous()
        with th.cuda.device(alpha.device):
            _lib.check(_lib.lib().gb_render_finish_bwd(H, W, _lib.ptr(alpha), _lib.ptr(g_rgb), _lib.ptr(g_depth),
                                                       _lib.ptr(g_out4), _lib.stream_ptr(alpha.device)), "render_finish_bwd")
        return g_out4, None


_SHADE_STREAMS = {}


def shade_stream(device):
    """The side stream a caller may run its shade on while render_views projects and bins (see `color_event` there)."""
    dev = th.device(device)
    st = _SHADE_STREAMS.get(dev)
    if st is None:
        # lowest priority: the shade fills the SMs the latency-bound binning kernels of a high-priority main stream
        # (render_stream) leave idle instead of taking their slots
        st = _SHADE_STREAMS[dev] = th.cuda.Stream(device=dev, priority=0)
    return st


_RENDER_STREAMS = {}


def render_stream(device):
    """A high-priority stream for the render itself (use it as the step's / the graph capture's stream when the shade
    runs on shade_stream)."""
    dev = th.device(device)
    st = _RENDER_STREAMS.get(dev)
    if st is None:
        st = _RENDER_STREAMS[dev] = th.cuda.Stream(device=dev, priority=-1)
    return st


def render_views(width: int, height: int, K: th.Tensor, Rt: th.Tensor, preds, intrinsics_host=None, fused=True,
                 capacity=None, color_event=None):
    """rgca.AutoEncoder.render (rgca.py:112-151): loop over the batch, stack, alpha from the DETACHED final_T,
    depth normalised by alpha.clamp(0.05, 1).  `intrinsics_host` (list of (fx,fy,cx,cy)) avoids the reference's
    four `.item()` device syncs per view when the caller already has them on the host.  `color_event`: preds["color"]
    is still being written on another stream (shade_stream) and this torch.cuda.Event was recorded after its last writer;
    the sync-free fused path then waits for it only where the colours are first read (the record gather at the end of the
    binning), so projection, depth ranks, tile buckets and the per-tile sort run beside the shade."""
    B = Rt.shape[0]
    if fused:
        # per view: one autograd node for project + bin/sort + pack + blend and one for the post-processing.  With several
        # views and the sync-free path the views are issued on a small pool of side streams (view_streams): independent
        # views overlap on the device — one view's blend tail (SMs idle while the last tiles finish) runs under the next
        # view's projection / binning — and become parallel branches when the step is captured in a CUDA graph.
        from .gsplat.fused import render_fused
        rgbs, alphas, depths = [], [], []
        pool = view_streams(Rt.device, B) if (capacity is not None and B > 1) else None
        main = th.cuda.current_stream(Rt.device) if pool else None
        # per-view slices as views whose backward is a plain view / stack: `x[b]` (select) would make autograd zero-fill a
        # full-batch tensor and copy into it for every field of every view (5 fills of up to 4.8 MB per view at B = 1)
        def per_view(x, last):
            return [x.reshape(-1, last)] if B == 1 else [t.reshape(-1, last) for t in th.unbind(x, 0)]
        pv = dict(primpos=per_view(preds["primpos"], 3), primscale=per_view(preds["primscale"], 3),
                  primqvec=per_view(preds["primqvec"], 4), opacity=per_view(preds["opacity"], 1),
                  color=per_view(preds["color"], 3))
        for b in range(B):
            if intrinsics_host is not None:
                fx, fy, cx, cy = intrinsics_host[b]
            else:
                fx, fy, cx, cy = K[b, 0, 0].item(), K[b, 1, 1].item(), K[b, 0, 2].item(), K[b, 1, 2].item()
            side = pool[b % len(pool)] if pool else None
            if side is not None and b < len(pool):
                side.wait_stream(main)
            with (th.cuda.stream(side) if side is not None else _nullctx()):
                out4, alpha, _ = render_fused(
                    pv["primpos"][b].contiguous(), pv["primscale"][b].contiguous(), 1.0, pv["primqvec"][b].contiguous(),
                    Rt[b], fx, fy, cx, cy, height, width, pv["opacity"][b].contiguous(), pv["color"][b].contiguous(),
                    _black(Rt.device), 0.1, capacity, colors_event=color_event)
                r, a, d = _FinishView.apply(out4, alpha)
            if side is not None:
                for t_ in (r, a, d):
                    t_.record_stream(main)
            rgbs.append(r); alphas.append(a); depths.append(d)
        if pool:
            for side in pool[:min(B, len(pool))]:
                main.wait_stream(side)
        if B == 1:
            return rgbs[0][None], alphas[0][None], depths[0][None]
        return th.stack(rgbs), th.stack(alphas), th.stack(depths)
    if color_event is not None:
        th.cuda.current_stream(Rt.device).wait_event(color_event)
    rgbs, Ts, depths = [], [], []
    for b in range(B):
        if intrinsics_host is not None:
            fx, fy, cx, cy = intrinsics_host[b]
        else:
            fx, fy, cx, cy = K[b, 0, 0].item(), K[b, 1, 1].item(), K[b, 0, 2].item(), K[b, 1, 2].item()
        o = render(width, height, fx, fy, cx, cy, Rt[b], preds["primpos"][b], preds["primqvec"][b],
                   preds["primscale"][b], preds["opacity"][b], preds["color"][b], return_depth=True, fused=fused, capacity=capacity)
        rgbs.append(o["render"])
        Ts.append(o["final_T"].detach())
        depths.append(o["depth"])
    rgb = th.stack(rgbs)
    depth = th.stack(depths)
    alpha = 1.0 - th.stack(Ts)
    depth = depth / alpha.clamp(0.05, 1.0)
    return rgb, alpha, depth
