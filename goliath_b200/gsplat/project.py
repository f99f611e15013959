"""project_gaussians — EWA projection (gsplat 0.1.11 `project_gaussians.py` API).

Call site in the reference: ca_code/utils/render_gsplat.py:49-63.
"""
from typing import Tuple

import torch
from torch import Tensor
from torch.autograd import Function

from .. import _lib


def project_gaussians(
    means3d: Tensor,
    scales: Tensor,
    glob_scale: float,
    quats: Tensor,
    viewmat: Tensor,
    fx: float,
    fy: float,
    cx: float,
    cy: float,
    img_height: int,
    img_width: int,
    block_width: int,
    clip_thresh: float = 0.01,
) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    """Returns (xys [G,2], depths [G], radii [G] i32, conics [G,3], compensation [G], num_tiles_hit [G] i32,
    cov3d [G,6]).  viewmat: row-major world->camera, first 12 floats are used ([3,4] or [4,4])."""
    assert block_width > 1 and block_width <= 16, "block_width must be between 2 and 16"
    assert (quats.norm(dim=-1) - 1 < 1e-6).all(), "quats must be normalized"
    outs = _ProjectGaussians.apply(
        means3d.contiguous(), scales.contiguous(), glob_scale, quats.contiguous(), viewmat.contiguous(),
        fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh,
    )
    # one token per call: rasterize_gaussians reuses a binning only for the tensors of the same projection (rasterize.py)
    token = object()
    for t in (outs[0], outs[1], outs[2], outs[5]):  # xys, depths, radii, num_tiles_hit
        t._gb_bin_token = token
    return outs


def _project_fwd(means3d, scales, quats, viewmat, glob_scale, fx, fy, cx, cy, img_height, img_width, block_width,
                 clip_thresh, grad_acc=None):
    """The projection kernel on the current stream.  Returns (xys [G,2], depths [G], radii [G] i32, conics [G,3],
    compensation [G], num_tiles_hit [G] i32, cov3d [G,6]).  `grad_acc` [10 G], if given, is zeroed by the same kernel
    for the fused render's blend backward (gb_project_gaussians_fwd_acc)."""
    G = means3d.size(0)
    dev = means3d.device
    f32 = dict(device=dev, dtype=torch.float32)
    i32 = dict(device=dev, dtype=torch.int32)
    cov3d, xys, depths = torch.empty(G, 6, **f32), torch.empty(G, 2, **f32), torch.empty(G, **f32)
    radii, conics, comp = torch.empty(G, **i32), torch.empty(G, 3, **f32), torch.empty(G, **f32)
    num_tiles_hit = torch.empty(G, **i32)
    L = _lib.kernels()
    args = (G, means3d, scales, float(glob_scale), quats, viewmat, float(fx), float(fy), float(cx), float(cy),
            int(img_height), int(img_width), int(block_width), float(clip_thresh), cov3d, xys, depths, radii, conics,
            comp, num_tiles_hit)
    if grad_acc is None:
        L.gb_project_gaussians_fwd(*args)
    else:
        L.gb_project_gaussians_fwd_acc(*args, grad_acc)
    return xys, depths, radii, conics, comp, num_tiles_hit, cov3d


def _project_bwd(means3d, scales, quats, viewmat, cov3d, radii, conics, comp, glob_scale, fx, fy, v_xy, v_depth, v_conic,
                 v_comp):
    """The projection backward on the current stream; a missing (None) gradient counts as zero.  Returns (v_means3d,
    v_scales, v_quats)."""
    G = means3d.size(0)
    dev = means3d.device
    f32 = dict(device=dev, dtype=torch.float32)

    def z(t, shape):
        return torch.zeros(shape, **f32) if t is None else t.contiguous()

    v_xy, v_depth, v_conic, v_comp = z(v_xy, (G, 2)), z(v_depth, (G,)), z(v_conic, (G, 3)), z(v_comp, (G,))
    g_cov2d, g_cov3d = torch.empty(G, 3, **f32), torch.empty(G, 6, **f32)
    g_mean, g_scale, g_quat = torch.empty(G, 3, **f32), torch.empty(G, 3, **f32), torch.empty(G, 4, **f32)
    _lib.kernels().gb_project_gaussians_bwd(
        G, means3d, scales, float(glob_scale), quats, viewmat, float(fx), float(fy), cov3d, radii, conics, comp,
        v_xy, v_depth, v_conic, v_comp, g_cov2d, g_cov3d, g_mean, g_scale, g_quat)
    return g_mean, g_scale, g_quat


class _ProjectGaussians(Function):
    @staticmethod
    def forward(ctx, means3d, scales, glob_scale, quats, viewmat, fx, fy, cx, cy, img_height, img_width,
                block_width, clip_thresh):
        for t, n in ((means3d, "means3d"), (scales, "scales"), (quats, "quats"), (viewmat, "viewmat")):
            _lib.check_input(t, n)
        if means3d.ndimension() != 2 or means3d.size(1) != 3:
            raise ValueError("means3d must have dimensions (N, 3)")
        if viewmat.numel() < 12:
            raise ValueError("viewmat must hold at least a 3x4 matrix")
        xys, depths, radii, conics, compensation, num_tiles_hit, cov3d = _project_fwd(
            means3d, scales, quats, viewmat, glob_scale, fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh)
        ctx.glob_scale, ctx.fx, ctx.fy = glob_scale, fx, fy
        ctx.save_for_backward(means3d, scales, quats, viewmat, cov3d, radii, conics, compensation)
        ctx.mark_non_differentiable(radii, num_tiles_hit)
        ctx.set_materialize_grads(False)
        return xys, depths, radii, conics, compensation, num_tiles_hit, cov3d

    @staticmethod
    def backward(ctx, v_xys, v_depths, v_radii, v_conics, v_compensation, v_num_tiles_hit, v_cov3d):
        means3d, scales, quats, viewmat, cov3d, radii, conics, compensation = ctx.saved_tensors
        g_mean3d, g_scale, g_quat = _project_bwd(means3d, scales, quats, viewmat, cov3d, radii, conics, compensation,
                                                 ctx.glob_scale, ctx.fx, ctx.fy, v_xys, v_depths, v_conics,
                                                 v_compensation)
        # v_cov3d (gradient of the returned cov3d) is ignored, as in gsplat 0.1.11
        v_viewmat = None
        if ctx.needs_input_grad[4]:
            # gsplat 0.1.11 camera-pose approximation: d f/d t = sum_g v_mean_cam, d f/d R_ij ~= v_mean_cam_i * mean_j
            v_viewmat = torch.zeros_like(viewmat)
            R = viewmat[..., :3, :3]
            v_mean_cam = torch.matmul(g_mean3d, R.transpose(-1, -2))
            v_viewmat[..., :3, 3] = v_mean_cam.sum(-2)
            for j in range(3):
                for l in range(3):
                    v_viewmat[..., j, l] = torch.dot(v_mean_cam[..., j], means3d[..., l])
        return (g_mean3d, g_scale, None, g_quat, v_viewmat, None, None, None, None, None, None, None, None)
