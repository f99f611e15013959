"""The relightable hand teacher's `OLATRGBDecoder` (ca_code/models/hand_teacher_mvp.py:159-554, DESIGN.md row R8″)
with the reference's constructor, `forward` / `forward_rgb` signatures, state-dict keys (`enc_layers.i.0.*`,
`dec_layers.i.0.*`) and `glorot(·, 0.2)` initialisation.

Per chunk of lights the reference expands a [B·L, K, TD, TH, TW, 4] template whose rgb is the constant 255, marches
it from every light with `with_shadow=True`, builds the U-Net input with ~30 eager ops, runs the U-Net and composes
the OLAT sum in torch.  Here:

  * light cameras (`light_cameras`): `build_cam_rot_mat` without its in-place write into the caller's lights, drtk's
    `transform` restated, and the focal fit of :315-334 with masked min / max over the valid primitives, so the
    forward has no host sync and can be captured in a CUDA graph;
  * deep shadow march (`gb_mvp_shadow_march`, csrc/mvp_raymarch.cu): bounds once per item, the alpha slab sampled in
    place, only the splat volume written;
  * U-Net input and `primshadow` in one pass (`gb_olat_features`, csrc/olat_teacher.cu);
  * U-Net on the stride-1 `Conv2dWNUB` kernels with the LeakyReLU fused; bilinear resizes and concatenations in
    torch, as in the reference;
  * OLAT compose forward / backward (`gb_olat_compose_fwd / _bwd`).

The features carry no gradient (the reference builds them under no_grad and marks them as leaves nobody reads), so
the first convolution computes no input gradient.

`AutoEncoder` (hand_teacher_mvp.py:49-156) is the teacher's whole frame: `hand_mvp.AutoEncoder` with a second pose
encoder and this decoder, rendered through the hand frame's gather, march and finish."""
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

from . import _lib, hand_mvp
from .envmap import compose_envmap
from .mvpraymarch import build_accel
from .nn import Conv2dWNUB, FusedLeakyReLU, glorot
from .utils import compute_raydirs


def build_cam_rot_mat(campos, objcenter=None):
    """hand_teacher_mvp.py:28-46: rows (x, y, z) of a camera at `campos` [N,3] looking at `objcenter` (or the origin)
    with y up.  A camera on the y axis is moved by 1e-2 along z for the rotation only; unlike the reference, the
    caller's tensor is not written."""
    on_axis = (campos[:, 0].abs() + campos[:, 2].abs()) < 1e-8
    campos = torch.stack([campos[:, 0], campos[:, 1], torch.where(on_axis, campos[:, 2] + 1e-2, campos[:, 2])], dim=1)
    z = F.normalize(-campos if objcenter is None else objcenter - campos, dim=1)
    up = torch.zeros_like(campos)
    up[:, 1] = 1
    x = F.normalize(torch.cross(z, up, dim=1), dim=1)
    y = F.normalize(torch.cross(z, x, dim=1), dim=1)
    return torch.stack([x, y, z], dim=1)


def transform(v, campos, camrot, focal, princpt):
    """drtk's `transform` as the teacher calls it: v [N,P,3] -> [N,P,3] = (focal (x/z, y/z) + princpt, z) with
    (x, y, z) = camrot (v - campos)."""
    vc = torch.einsum("nij,npj->npi", camrot, v - campos[:, None])
    z = vc[..., 2:3]
    pix = torch.einsum("nij,npj->npi", focal, vc[..., :2] / z) + princpt[:, None]
    return torch.cat([pix, z], dim=-1)


def light_cameras(primpos, valid_prims, light_pos, img_h, img_w):
    """hand_teacher_mvp.py:315-334: per light view (B·L of them) the camera position, rotation, focal [B·L,2] and
    principal point [B·L,2] that frame the valid primitives of its item in 90% of an img_h x img_w shadow image.
    The centre and the largest |pixel ratio| are reductions over the valid primitives, taken with masked min / max."""
    B, L = light_pos.shape[:2]
    v = valid_prims.reshape(1, -1, 1).bool()
    posc = (torch.where(v, primpos, float("-inf")).amax(1) + torch.where(v, primpos, float("inf")).amin(1)) / 2
    posc = posc[:, None].expand(B, L, 3).reshape(B * L, 3)
    lpos = light_pos.reshape(B * L, 3)
    lrot = build_cam_rot_mat(lpos, posc)
    dt, dev = primpos.dtype, primpos.device
    focal = torch.diag(torch.full((2,), 1000.0, dtype=dt, device=dev))[None].expand(B * L, -1, -1)
    # no host tensors: built with fills, so the forward can be captured in a CUDA graph
    princpt = torch.stack([torch.full((B * L,), img_w / 2, dtype=dt, device=dev),
                           torch.full((B * L,), img_h / 2, dtype=dt, device=dev)], dim=1)
    pts = primpos[:, None].expand(-1, L, -1, -1).reshape(B * L, -1, 3)
    v_pix = transform(pts, lpos, lrot, focal, princpt)
    half = torch.stack([torch.full((1,), 0.45 * img_w, dtype=dt, device=dev),
                        torch.full((1,), 0.45 * img_h, dtype=dt, device=dev)], dim=1)
    pix_ratio = (v_pix[..., :2] - princpt[:, None]) / half[None]
    m = torch.where(v, pix_ratio.abs(), 0.0).amax(1)
    return lpos.contiguous(), lrot.contiguous(), (torch.diagonal(focal, 0, 1, 2) / m).contiguous(), princpt.contiguous()


class _OLATCompose(Function):
    """rgb (+= into `prev`, which is then returned) and texolat of one chunk; gradient to tex (and prev)."""

    @staticmethod
    def forward(ctx, tex, intensity, shadow_feat, prev, Z, want_texolat):
        BL, _, U, _ = tex.shape
        B, L = intensity.shape[:2]
        rgb = prev if prev is not None else torch.empty(B, Z, 3, U, U, device=tex.device)
        texolat = torch.empty(B, L, Z, 3, U, U, device=tex.device) if want_texolat else None
        with torch.cuda.device(tex.device):
            _lib.check(_lib.lib().gb_olat_compose_fwd(
                B, L, Z, U, _lib.ptr(tex), _lib.ptr(intensity), _lib.ptr(shadow_feat), _lib.ptr(rgb),
                int(prev is not None), _lib.ptr(texolat), _lib.stream_ptr(tex.device)), "olat_compose_fwd")
        if prev is not None:
            ctx.mark_dirty(prev)
        ctx.save_for_backward(tex, intensity, shadow_feat)
        ctx.meta = (B, L, Z, U, prev is not None)
        ctx.set_materialize_grads(False)
        return rgb, texolat

    @staticmethod
    def backward(ctx, g_rgb, g_texolat):
        tex, intensity, shadow_feat = ctx.saved_tensors
        B, L, Z, U, has_prev = ctx.meta
        g_tex = None
        if g_rgb is not None or g_texolat is not None:
            g_rgb = torch.zeros(B, Z, 3, U, U, device=tex.device) if g_rgb is None else g_rgb.contiguous()
            g_texolat = None if g_texolat is None else g_texolat.contiguous()
            g_tex = torch.empty_like(tex)
            with torch.cuda.device(tex.device):
                _lib.check(_lib.lib().gb_olat_compose_bwd(
                    B, L, Z, U, _lib.ptr(tex), _lib.ptr(intensity), _lib.ptr(shadow_feat), _lib.ptr(g_rgb),
                    _lib.ptr(g_texolat), _lib.ptr(g_tex), _lib.stream_ptr(tex.device)), "olat_compose_bwd")
        return g_tex, None, None, g_rgb if has_prev else None, None, None


def olat_compose(tex, light_intensity, Z, shadow_feat=None, prev=None, want_texolat=False):
    """hand_teacher_mvp.py:468-479 for one chunk: tex [B·L,4Z,U,U] viewed [B,L,Z,4,U,U], light_intensity [B,L,3] ->
    (rgb [B,Z,3,U,U], texolat [B,L,Z,3,U,U] or None).  s = sigmoid(t0), or `shadow_feat` [B·L,Z,U,U] (training
    warm-up, no gradient).  With `prev` the chunk's sum is added into it in place (the reference's `rgb + tmp_rgb`)."""
    tex = tex.contiguous()
    intensity = light_intensity.to(torch.float32).contiguous()
    _lib.check_input(tex, "tex")
    _lib.check_input(intensity, "light_intensity")
    BL, C, U, U2 = tex.shape
    B, L = intensity.shape[:2]
    if C != 4 * Z or U != U2 or BL != B * L or intensity.shape != (B, L, 3):
        raise RuntimeError("tex must be [B*L, 4Z, U, U] and light_intensity [B, L, 3]")
    if shadow_feat is not None:
        shadow_feat = shadow_feat.detach().contiguous()
        _lib.check_input(shadow_feat, "shadow_feat")
        if shadow_feat.shape != (BL, Z, U, U):
            raise RuntimeError("shadow_feat must be [B*L, Z, U, U]")
    if prev is not None and (prev.shape != (B, Z, 3, U, U) or not prev.is_contiguous()):
        raise RuntimeError("prev must be a contiguous [B, Z, 3, U, U] tensor")
    return _OLATCompose.apply(tex, intensity, shadow_feat, prev, Z, bool(want_texolat))


def _colour_intensity(light_intensity):
    """[B,L,1] intensities (SingleLightCycleDecorator's) broadcast over the three colours, as the reference's product
    does (hand_teacher_mvp.py:407, 478); any other shape is passed on unchanged"""
    if light_intensity.dim() == 3 and light_intensity.shape[2] == 1:
        return light_intensity.expand(-1, -1, 3)
    return light_intensity


def _unet_layer(n_in, n_out, size):
    conv = Conv2dWNUB(n_in, n_out, size, size, 3, 1, 1)
    conv.fused_slope = 0.2
    return nn.Sequential(conv, FusedLeakyReLU())  # keys `.0.*`, as the reference's (Conv2dWNUB, LeakyReLU)


class OLATRGBDecoder(nn.Module):
    """hand_teacher_mvp.py:159-554.  `raymarcher` supplies the step size (`raymarcher.dt`) and, like the reference's
    `Raymarcher`, the radius primitive positions are divided by (`raymarcher.volume_radius`, else `volradius`)."""

    def __init__(self, uv_size, primsize, n_prim_x, n_prim_y, raymarcher, volradius, n_init_channels=64,
                 n_enc_dims=[64, 64, 64, 64, 64], shadow_img_size=1024):
        super().__init__()
        self.chunksize = 5
        self.uv_size = uv_size
        self.primsize = primsize
        self.n_prim_x = n_prim_x
        self.n_prim_y = n_prim_y
        self.uv_multiple = 1
        in_feats = 2 * 3 + 1  # light_dir, view_dir, shadow
        self.n_enc_dims = [(in_feats * primsize[2], n_enc_dims[0])] + [(n_enc_dims[i], n_enc_dims[i + 1])
                                                                       for i in range(4)]
        self.n_dec_dims = [(n_enc_dims[4] + n_init_channels, n_enc_dims[3]), (n_enc_dims[3] * 2, n_enc_dims[2]),
                           (n_enc_dims[2] * 2, n_enc_dims[1]), (n_enc_dims[1] * 2, n_enc_dims[0]),
                           (n_enc_dims[0] * 2, primsize[2] * 4)]
        self.sizes = [(primsize[0] * n_prim_x) // (2 ** i) for i in range(len(self.n_enc_dims))]
        self.enc_layers = nn.ModuleList(_unet_layer(*self.n_enc_dims[i], s) for i, s in enumerate(self.sizes))
        self.dec_layers = nn.ModuleList(_unet_layer(*self.n_dec_dims[i], self.sizes[-i - 1])
                                        for i in range(len(self.sizes)))
        self.volradius = volradius
        self.raymarcher = raymarcher
        # the reference's ray grid is stack([y, x]): the shadow image is transposed (hand_teacher_mvp.py:247-249)
        y, x = torch.meshgrid(torch.arange(shadow_img_size), torch.arange(shadow_img_size), indexing="ij")
        self.register_buffer("pixel_coords", torch.stack([y, x], dim=-1).float(), persistent=False)
        self.apply(lambda m: glorot(m, 0.2))

    # ------------------------------------------------------------------------------------------------ stages
    def _prims(self, primpos, primrot, primscale, primalpha, valid_prims):
        """Per-item inputs shared by every chunk: transforms, bounds, alpha slab and mask."""
        pp, pr, ps = (t.detach().to(torch.float32).contiguous() for t in (primpos, primrot, primscale))
        alpha = primalpha.detach().to(torch.float32).contiguous()
        valid = valid_prims.detach().to(device=pp.device, dtype=torch.float32).reshape(-1).contiguous()
        for t, n in ((pp, "primpos"), (pr, "primrot"), (ps, "primscale"), (alpha, "primalpha"), (valid, "valid_prims")):
            _lib.check_input(t, n)
        B, K = pp.shape[:2]
        TD, TH, TW = self.primsize[2], self.primsize[1], self.primsize[0]
        U = self.uv_size
        if (K != self.n_prim_x * self.n_prim_y or alpha.shape != (B, TD, 1, U, U) or valid.numel() != K
                or U != self.n_prim_x * TW or U != self.n_prim_y * TH):
            raise RuntimeError("primpos must be [B, n_prim_x*n_prim_y, 3], primalpha [B, primsize[2], 1, uv, uv] with "
                               "uv = n_prim_x*primsize[0] = n_prim_y*primsize[1], valid_prims [n_prims]")
        radius = float(getattr(self.raymarcher, "volume_radius", self.volradius))
        pp_n = (pp / radius).contiguous()
        nodeaabb = build_accel((pp_n, pr, ps), 0, fixedorder=True)[2]
        return pp, pr, ps, pp_n, nodeaabb, alpha, valid

    def shadow_march(self, prims, light_pos):
        """Un-normalised deep shadow volume [B·L,K,TD,TH,TW,2] of every light in `light_pos` [B,L,3]."""
        pp, pr, ps, pp_n, nodeaabb, alpha, valid = prims
        B, L = light_pos.shape[:2]
        K = pp.shape[1]
        S0, S1 = self.pixel_coords.shape[:2]
        lpos, lrot, focal, princpt = light_cameras(pp, valid, light_pos, S0, S1)
        pix = self.pixel_coords[None].expand(B * L, -1, -1, -1).contiguous()
        raypos, raydir, tminmax = compute_raydirs(lpos, lrot, focal, princpt, pix, self.volradius)
        TD, TH, TW = self.primsize[2], self.primsize[1], self.primsize[0]
        shadow = torch.zeros(B * L, K, TD, TH, TW, 2, device=pp.device)
        with torch.cuda.device(pp.device):
            _lib.check(_lib.lib().gb_mvp_shadow_march(
                B * L, L, S0, S1, K, _lib.ptr(raypos), _lib.ptr(raydir), float(self.raymarcher.dt), _lib.ptr(tminmax),
                _lib.ptr(nodeaabb), _lib.ptr(pp_n), _lib.ptr(pr), _lib.ptr(ps), TD, TH, TW, self.uv_size,
                _lib.ptr(alpha), _lib.ptr(valid), _lib.ptr(shadow), 8.0, 8.0, 8, 16, _lib.stream_ptr(pp.device)),
                "mvp_shadow_march")
        return shadow

    def features(self, prims, campos, light_pos, shadow, primshadow=None, want_shadow_feat=False):
        """U-Net input [B·L,7Z,U,U]; the chunk's light mean of the shadow written into (or, when given, added to)
        `primshadow` [B,Z,3,U,U]; the normalised shadow [B·L,Z,U,U] when asked for."""
        pp, pr, ps, _, _, _, valid = prims
        B, L = light_pos.shape[:2]
        K = pp.shape[1]
        TD, TH, TW, U = self.primsize[2], self.primsize[1], self.primsize[0], self.uv_size
        lp = light_pos.detach().to(torch.float32).contiguous()
        cp = campos.detach().to(torch.float32).contiguous()
        _lib.check_input(lp, "light_pos")
        _lib.check_input(cp, "campos")
        if cp.shape != (B, 3) or lp.shape != (B, L, 3) or shadow.shape != (B * L, K, TD, TH, TW, 2):
            raise RuntimeError("campos must be [B, 3], light_pos [B, L, 3], shadow [B*L, K, TD, TH, TW, 2]")
        feat = torch.empty(B * L, 7 * TD, U, U, device=pp.device)
        accumulate = primshadow is not None
        if primshadow is None:
            primshadow = torch.empty(B, TD, 3, U, U, device=pp.device)
        sf = torch.empty(B * L, TD, U, U, device=pp.device) if want_shadow_feat else None
        with torch.cuda.device(pp.device):
            _lib.check(_lib.lib().gb_olat_features(
                B, L, K, TD, TH, TW, U, float(self.volradius), _lib.ptr(pp), _lib.ptr(pr), _lib.ptr(ps), _lib.ptr(valid),
                _lib.ptr(lp), _lib.ptr(cp), _lib.ptr(shadow), _lib.ptr(feat), _lib.ptr(primshadow), int(accumulate),
                _lib.ptr(sf), _lib.stream_ptr(pp.device)), "olat_features")
        return feat, primshadow, sf

    def unet(self, x, joint_feat, L):
        """hand_teacher_mvp.py:441-467: [B·L,7Z,U,U] -> tex [B·L,4Z,U,U]; joint_feat [B,C,s,s] joins at the smallest
        level."""
        B = joint_feat.shape[0]
        joint_feat = joint_feat[:, None].expand(-1, L, -1, -1, -1).reshape(B * L, *joint_feat.shape[-3:])
        enc_acts = []
        for i, layer in enumerate(self.enc_layers):
            x = layer(x)
            enc_acts.append(x)
            if i < len(self.sizes) - 1:
                x = F.interpolate(x, scale_factor=0.5, mode="bilinear", recompute_scale_factor=True, align_corners=True)
        for i, layer in enumerate(self.dec_layers):
            if i == 0:
                x = torch.cat([x, joint_feat], dim=1)
            else:
                x_prev = enc_acts[-i - 1]
                x = F.interpolate(x, size=x_prev.shape[2:4], mode="bilinear", align_corners=True)
                x = torch.cat([x, x_prev], dim=1)
            x = layer(x)
        return x

    def _chunk(self, prims, campos, joint_feat, light_pos, light_intensity, iteration, rgb, primshadow, last):
        warm = self.training and iteration is not None and iteration < 1000
        shadow = self.shadow_march(prims, light_pos)
        x, primshadow, sf = self.features(prims, campos, light_pos, shadow, primshadow, want_shadow_feat=warm)
        del shadow
        tex = self.unet(x, joint_feat, light_pos.shape[1])
        rgb, texolat = olat_compose(tex, light_intensity, self.primsize[2], sf if warm else None, rgb,
                                    want_texolat=self.training and last)
        return rgb, primshadow, texolat

    # ------------------------------------------------------------------------------------------------ interface
    def forward_rgb(self, campos, K, Rt, primpos, primrot, primscale, primalpha, valid_prims, joint_feat, light_pos,
                    light_intensity, iteration: Optional[int] = None):
        """hand_teacher_mvp.py:253-493: one chunk of lights ([B,L,3] positions, [B,L,3] or [B,L,1] intensities).  K and
        Rt are unused, as in the reference."""
        light_intensity = _colour_intensity(light_intensity)
        prims = self._prims(primpos, primrot, primscale, primalpha, valid_prims)
        rgb, primshadow, texolat = self._chunk(prims, campos, joint_feat, light_pos, light_intensity, iteration, None,
                                               None, True)
        output = {"primrgb": rgb, "primshadow": primshadow}
        if self.training:
            output["texolat"] = texolat
        return output

    def forward(self, campos, K, Rt, primpos, primrot, primscale, primalpha, valid_prims, joint_feat, light_pos,
                light_intensity, iteration: Optional[int] = None):
        """hand_teacher_mvp.py:496-554: the lights in chunks of `chunksize`; `primrgb` is the sum over the chunks,
        `primshadow` the sum over the chunks of each chunk's light mean, `texolat` (training) the last chunk's."""
        light_intensity = _colour_intensity(light_intensity)
        prims = self._prims(primpos, primrot, primscale, primalpha, valid_prims)
        L = light_pos.shape[1]
        n_chunks = (L - 1) // self.chunksize + 1
        rgb = primshadow = texolat = None
        for i in range(n_chunks):
            sl = slice(i * self.chunksize, (i + 1) * self.chunksize)
            rgb, primshadow, texolat = self._chunk(prims, campos, joint_feat, light_pos[:, sl],
                                                   light_intensity[:, sl], iteration, rgb, primshadow,
                                                   i == n_chunks - 1)
        output = {"primrgb": rgb, "primshadow": primshadow}
        if self.training:
            output["texolat"] = texolat
        return output


# ------------------------------------------------------------------------------------------------ the frame
class AutoEncoder(hand_mvp.AutoEncoder):
    """hand_teacher_mvp.AutoEncoder (ca_code/models/hand_teacher_mvp.py:49-156): the hand frame with a second pose
    encoder and the OLAT decoder in place of the RGB slab decoder.  The constructor and the state-dict keys are the
    reference's: the hand frame's plus `poseencoder2.*` and `relightdecoder.{enc,dec}_layers.*`, so
    `AutoEncoder(**config.model, assets=assets)` builds from hand_teacher_mvp_example.yml, a teacher checkpoint loads
    with strict=True and a hand_mvp checkpoint with strict=False (missing exactly the two new modules).

    As in the reference, the constructor leaves `geomdecoder` in eval mode: until the next .train() / .eval() a fresh
    model marches its geometry without the training branch and relights in training mode.  The frame is the hand
    frame's: the relit `primrgb` (already activated) and `primalpha` make the template, the valid-primitive gather and
    the march run through `hand_mvp.AutoEncoder._march`, calibration and background through `hand_finish`.  With an
    `envbg` (EnvSpinDecorator) the environment is composited behind the render by `envmap.compose_envmap`.  The
    decorators' other keys are accepted and ignored.  CUDA only; forward and backward issue no host synchronisation
    after the first call."""

    def __init__(self, assets, image_height, image_width, cal=None, n_pose_dims: int = 54, n_embs: int = 64,
                 volradius: float = 2000.0, primsize=(16, 16, 8), learn_blur: bool = True):
        super().__init__(assets, image_height, image_width, cal, n_pose_dims, n_embs, volradius, primsize, learn_blur)
        self.poseencoder2 = hand_mvp.PoseEncoder(n_pose_dims, n_embs, self.n_prim_x)
        self.relightdecoder = OLATRGBDecoder(self.uv_size, self.primsize, self.n_prim_x, self.n_prim_y,
                                             self.raymarcher, self.volradius)
        self.geomdecoder.eval()

    def forward(self, pose, campos, K, Rt, light_intensity, light_pos, camera_id=None, frame_id=None, iteration=None,
                background=None, **kwargs):
        for t, n in ((pose, "pose"), (campos, "campos"), (K, "K"), (Rt, "Rt"), (light_intensity, "light_intensity"),
                     (light_pos, "light_pos")):
            if t is None or not t.is_cuda:
                raise RuntimeError("hand_teacher.AutoEncoder runs on CUDA only (no CPU fallback): %s is %s"
                                   % (n, "missing" if t is None else "on %s" % t.device))
        joint = self.poseencoder(pose)
        geo_preds = self.geomdecoder(pose, joint, iteration)
        joint2 = self.poseencoder2(pose)
        dec_preds = self.relightdecoder(campos, K, Rt, geo_preds["primpos"], geo_preds["primrot"],
                                        geo_preds["primscale"], geo_preds["primalpha"], self.valid_prims, joint2,
                                        light_pos, light_intensity, iteration)
        preds = {"primrgb": dec_preds["primrgb"], "valid_prims": self.valid_prims, **geo_preds, **dec_preds}
        preds["primrgba"] = hand_mvp.slabs_to_primrgba(preds["primrgb"], preds["primalpha"], self.primsize)
        rgb, alpha = self._finish(self._march(K, Rt, preds), camera_id, background)
        if "envbg" in kwargs:
            rgb = compose_envmap(rgb / 255.0, alpha, kwargs["envbg"], K, Rt)
        preds.update(rgb=rgb, alpha=alpha, ae=self)
        self._blur(preds, camera_id)
        return preds
