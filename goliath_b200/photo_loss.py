"""Post-render chain and photometric losses of the RGCA train step as four fused kernels (csrc/photo_loss.cu,
SURVEY.md section 8f-2):

  post_render(rgb, ...)          CalV5 colour calibration (ca_code/nn/color_cal.py:211-241) -> background composite
                                 (ca_code/models/rgca.py:226-230) -> LearnableBlur (ca_code/nn/dof_cal.py:44-56)
  photometric_loss(pred, ...)    loss = l1_weight * rgb_l1 + ssim_weight * rgb_ssim with the reference's definitions
                                 (ca_code/loss/__init__.py:391-410 and :479-494 over ca_code/utils/ssim.py)

Both are autograd Functions; the gradient that leaves `post_render` is dL/d(rendered rgb), i.e. the `v_out` of the blend
backward.  No host synchronisation anywhere (the sums stay on the device), so the whole train step stays capturable."""
from typing import Dict, Optional, Tuple

import torch
from torch.autograd import Function

from . import _lib


class _PostRender(Function):
    @staticmethod
    def forward(ctx, rgb, alpha, background, cal_w, cal_b, grey, blur_w):
        rgb = rgb.contiguous()
        _lib.check_input(rgb, "rgb")
        B, C, H, W = rgb.shape
        if C != 3:
            raise RuntimeError("post_render: rgb must be [B,3,H,W]")
        opt = {}
        for name, t, shape, dt in (("alpha", alpha, (B, 1, H, W), torch.float32), ("background", background, (B, 3, H, W), torch.float32),
                                   ("cal_w", cal_w, (B, 3), torch.float32), ("cal_b", cal_b, (B, 3), torch.float32),
                                   ("grey", grey, (B,), torch.int32), ("blur_w", blur_w, (B, 3), torch.float32)):
            if t is not None:
                t = t.contiguous()
                _lib.check_input(t, name, dt)
                if tuple(t.shape) != shape:
                    raise RuntimeError("post_render: %s must have shape %s" % (name, (shape,)))
            opt[name] = t
        if (opt["cal_w"] is None) != (opt["cal_b"] is None):
            raise RuntimeError("post_render: cal_w and cal_b go together")
        if opt["background"] is not None and opt["alpha"] is None:
            raise RuntimeError("post_render: the background composite needs alpha")
        pred = torch.empty_like(rgb)
        _lib.kernels().gb_post_render_fwd(
            B, H, W, rgb, opt["alpha"], opt["background"], opt["cal_w"], opt["cal_b"], opt["grey"], opt["blur_w"],
            pred)
        ctx.save_for_backward(rgb, *[opt[k] for k in ("alpha", "background", "cal_w", "cal_b", "grey", "blur_w")])
        return pred

    @staticmethod
    def backward(ctx, g_pred):
        rgb, alpha, background, cal_w, cal_b, grey, blur_w = ctx.saved_tensors
        B, _, H, W = rgb.shape
        g_pred = g_pred.contiguous()
        g_rgb = torch.empty_like(rgb)
        z = lambda t: None if t is None else torch.zeros_like(t)
        g_cw, g_cb, g_bw = z(cal_w), z(cal_b), z(blur_w)
        _lib.kernels().gb_post_render_bwd(
            B, H, W, rgb, alpha, background, cal_w, cal_b, grey, blur_w, g_pred, g_rgb, g_cw, g_cb, g_bw)
        return g_rgb, None, None, g_cw, g_cb, None, g_bw


def post_render(rgb: torch.Tensor, alpha: Optional[torch.Tensor] = None, background: Optional[torch.Tensor] = None,
                cal_w: Optional[torch.Tensor] = None, cal_b: Optional[torch.Tensor] = None,
                grey: Optional[torch.Tensor] = None, blur_weights: Optional[torch.Tensor] = None) -> torch.Tensor:
    """rgb [B,3,H,W] -> blur(cal(rgb) + (1 - alpha) * background).  cal_w / cal_b [B,3]: per-frame calibration rows
    (identity camera: w = 1, b = 0); grey [B] int32 marks grey cameras (out = sum_c img_c w_c + sum_c b_c on all three
    channels); background [B,3,H,W] with alpha [B,1,H,W] (detached upstream, rgca.py:137); blur_weights [B,3] = the
    softmax-ed LearnableBlur weights (identity, 3x3, 7x7).  Any stage whose tensors are None is skipped.
    Gradients: rgb, cal_w, cal_b, blur_weights."""
    return _PostRender.apply(rgb, alpha, background, cal_w, cal_b, grey, blur_weights)


class _SsimL1(Function):
    @staticmethod
    def forward(ctx, pred, target, mask, l1_weight, ssim_weight):
        pred, target, mask = pred.contiguous(), target.contiguous(), mask.contiguous()
        for t, n in ((pred, "pred"), (target, "target"), (mask, "mask")):
            _lib.check_input(t, n)
        B, C, H, W = pred.shape
        if C != 3 or target.shape != pred.shape or mask.shape != (B, 1, H, W):
            raise RuntimeError("photometric_loss: pred / target [B,3,H,W], mask [B,1,H,W]")
        dev = pred.device
        d_mu, d_pp, d_tp = torch.empty_like(pred), torch.empty_like(pred), torch.empty_like(pred)
        sums = torch.zeros(3, dtype=torch.float64, device=dev)
        _lib.kernels().gb_ssim_l1_fwd(B, H, W, pred, target, mask, d_mu, d_pp, d_tp, sums)
        l1 = (sums[0] / float(B * 3 * H * W)).float()
        ssim = (sums[1] / sums[2].clamp(min=1.0)).float()
        loss = l1_weight * l1 + ssim_weight * (1.0 - ssim)
        ctx.save_for_backward(pred, target, mask, d_mu, d_pp, d_tp, sums)
        ctx.w = (float(l1_weight), float(ssim_weight))
        ctx.mark_non_differentiable(l1, ssim)
        return loss, l1, ssim

    @staticmethod
    def backward(ctx, g_loss, _g_l1, _g_ssim):
        pred, target, mask, d_mu, d_pp, d_tp, sums = ctx.saved_tensors
        B, _, H, W = pred.shape
        g_pred = torch.empty_like(pred)
        g_loss = g_loss.contiguous().float()
        _lib.kernels().gb_ssim_l1_bwd(B, H, W, pred, target, mask, d_mu, d_pp, d_tp, sums, g_loss, ctx.w[0],
                                      ctx.w[1], g_pred)
        return g_pred, None, None, None, None


def photometric_loss(pred: torch.Tensor, target: torch.Tensor, mask: torch.Tensor, l1_weight: float = 10.0,
                     ssim_weight: float = 0.2) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """loss = l1_weight * rgb_l1 + ssim_weight * rgb_ssim (config/rgca_example.yml weights by default) with
    rgb_l1 = mean(|(pred - target) * mask|) and rgb_ssim = 1 - sum(ssim_map(target, pred) * mask) / clamp(sum(mask), 1)
    (mask [B,1,H,W] broadcast over the channels, 11x11 window).  Returns (loss, {"rgb_l1", "rgb_ssim"})."""
    loss, l1, ssim = _SsimL1.apply(pred, target, mask, l1_weight, ssim_weight)
    return loss, {"rgb_l1": l1, "rgb_ssim": 1.0 - ssim}


def _indices_to_device(rows, device: torch.device) -> torch.Tensor:
    """host int list -> int64 device tensor in one non-blocking copy from pinned memory (no host synchronisation)"""
    if device.type != "cuda":
        raise RuntimeError("the camera modules run on CUDA only (no CPU fallback): move them to the GPU first")
    return torch.tensor(rows, dtype=torch.int64).pin_memory().to(device, non_blocking=True)


class ParamHolder(torch.nn.Module):
    """ca_code/utils/torchutils.py:56-72: `params` [len(key_list), *param_shape] over the sorted key list"""

    def __init__(self, param_shape, key_list, init_value=None):
        super().__init__()
        if isinstance(param_shape, int):
            param_shape = (param_shape,)
        self.key_list = sorted(key_list)
        self.params = torch.nn.Parameter(torch.zeros(len(self.key_list), *param_shape))
        if init_value is not None:
            self.params.data[:] = init_value

    def to_idx(self, keys):
        """host indices of `keys` in the sorted key list (a ValueError names an unknown key)"""
        return [self.key_list.index(k) for k in keys]


class CalV5(torch.nn.Module):
    """ca_code/nn/color_cal.py:101-241 on post_render's calibration stage.  `holder.params` [n_cams, 6] = (w, b) per
    camera in sorted name order; cameras whose name starts with "41" are grey (out = sum_c img_c w_c + sum_c b_c on
    all three channels, initial w = (0.37, 0.52, 0.52)); the identity camera passes through and its row gets no
    gradient.  In training the parameter gradient is scaled per item by gs_lrscale (grey) / col_lrscale (colour), as
    the reference's scale_hook does.  `name_to_idx` maps names on the host and copies the indices without a sync."""

    def __init__(self, cameras, identity_camera, gs_lrscale: float = 1e0, col_lrscale: float = 1e-1):
        super().__init__()
        if identity_camera not in cameras:   # the reference's fallback (an id given as a YAML int lands here too)
            identity_camera = cameras[0]
        self.identity_camera = identity_camera
        self.cameras = cameras
        self.gs_lrscale, self.col_lrscale = gs_lrscale, col_lrscale
        self.holder = ParamHolder(3 + 3, cameras, init_value=torch.FloatTensor([1, 1, 1, 0, 0, 0]))
        self.identity_idx = self.holder.to_idx([identity_camera])[0]
        self.grey_idxs = [self.holder.to_idx([c])[0] for c in cameras if c.startswith("41")]
        self.holder.params.data[torch.LongTensor(self.grey_idxs), :3] = torch.FloatTensor([0.37, 0.52, 0.52])
        grey = torch.zeros(len(self.holder.key_list), dtype=torch.bool)
        grey[self.grey_idxs] = True
        self.register_buffer("grey_mask", grey, persistent=False)

    def name_to_idx(self, cam_names) -> torch.Tensor:
        return _indices_to_device(self.holder.to_idx(cam_names), self.holder.params.device)

    def rows(self, cam_idxs: torch.Tensor):
        """post_render's calibration arguments for the cameras `cam_idxs`: (cal_w, cal_b) [B,3] and grey [B] int32,
        with the training gradient scale hooked onto the gathered rows"""
        params = self.holder.params[cam_idxs]
        ident = cam_idxs == self.identity_idx
        grey = self.grey_mask[cam_idxs] & ~ident
        if self.training and params.requires_grad:
            scale = torch.where(grey, self.gs_lrscale, self.col_lrscale).masked_fill(ident, 1.0).to(params.dtype)
            params.register_hook(lambda g: g * scale[:, None])
        w = torch.where(ident[:, None], 1.0, params[:, :3])
        b = torch.where(ident[:, None], 0.0, params[:, 3:])
        return w, b, grey.to(torch.int32)

    def forward(self, image: torch.Tensor, cam_idxs: torch.Tensor) -> torch.Tensor:
        w, b, grey = self.rows(cam_idxs)
        return post_render(image, cal_w=w, cal_b=b, grey=grey)


class LearnableBlur(torch.nn.Module):
    """ca_code/nn/dof_cal.py:20-56 on post_render's blur stage: softmax(weights_raw[camera]) mixes the image with its
    3x3 and 7x7 Gaussian blurs.  Cameras index `weights_raw` in the list's order, as in the reference."""

    def __init__(self, cameras):
        super().__init__()
        self.cameras = cameras
        self.register_parameter("weights_raw", torch.nn.Parameter(torch.ones(len(cameras), 3, dtype=torch.float32)))

    def name_to_idx(self, cameras) -> torch.Tensor:
        return _indices_to_device([self.cameras.index(c) for c in cameras], self.weights_raw.device)

    def reg(self, cameras):
        return self.weights_raw[self.name_to_idx(cameras)]

    def weights(self, cameras) -> torch.Tensor:
        """post_render's blur weights [B,3] for `cameras`: softmax(weights_raw[camera])"""
        return torch.softmax(self.weights_raw[self.name_to_idx(cameras)], dim=-1)

    def forward(self, img: torch.Tensor, cameras) -> torch.Tensor:
        return post_render(img, blur_weights=self.weights(cameras))
