"""Host-side mirror of the hand-MVP decoders (SURVEY.md §8 row R8): `PoseEncoder`, `TransDecoder`,
`DeconvContentDecoder` (ca_code/models/hand_mvp.py:269-348) with the reference's module / parameter names so its
checkpoints load, plus the two glue stages between those decoders and the raymarcher as single kernels:

  * `prim_transforms`   — TransDecoder's head scaling + GeomDecoder's composition with the mesh-attached base frame
                          (hand_mvp.py:317-321, 410-425, 477-510), csrc/mvp_prims.cu
  * `slabs_to_primrgba` — output activations + cat/permute/reshape + valid-primitive gather
                          (hand_mvp.py:434,472,172-185; render_raymarcher.py:44-46), csrc/mvp_prims.cu

The mesh front end (DESIGN.md row R8') runs on kernels too: `GeomDecoder` poses the mesh with `lbs.LBSModule` and
builds each primitive's base frame with `prim_base_frames`; `view_cos_uv` gives the RGB decoder's view conditioning
(hand_mvp.py:230-236), both on csrc/mvp_prims.cu.

`AutoEncoder` (hand_mvp.py:71-266) runs the whole frame on these stages and the MVP raymarcher, with the valid-primitive
gather before the march and the render finish after it on csrc/hand_frame.cu."""
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.autograd import Function

from . import _lib
from .geom import vert_normals
from .nn import ConvBlock, ConvTranspose2dWNUB, Conv2dWNUB, FusedLeakyReLU, glorot, tile2d


class PoseEncoder(nn.Module):
    """hand_mvp.py:269-294: local pose -> [B, n_embs, in_size, in_size] joint feature map."""

    def __init__(self, n_pose_dims, n_embs, in_size):
        super().__init__()
        self.in_size = in_size
        self.local_pose_conv_block = ConvBlock(n_pose_dims, 16, in_size, kernel_size=1, padding=0)
        self.joint_conv_block = ConvBlock(16, n_embs, in_size)

    def forward(self, pose):
        pose_tile = tile2d(pose[:, 6:], self.in_size)
        return self.joint_conv_block(self.local_pose_conv_block(pose_tile))


def _seq_with_fused_act(layers, slope=0.2):
    """[conv, LeakyReLU, conv, LeakyReLU, ..., conv] with the activations executed inside the conv kernels; the
    placeholders keep the Sequential indices (= checkpoint keys dec0.0, dec0.2, ...) of the reference."""
    mods = []
    for i, layer in enumerate(layers):
        mods.append(layer)
        if i + 1 < len(layers):
            layer.fused_slope = slope
            mods.append(FusedLeakyReLU())
    return nn.Sequential(*mods)


class TransDecoder(nn.Module):
    """hand_mvp.py:297-321: five 3x3 Conv2dWNUB @64x64 -> per-primitive (dpos, drvec, dscale)."""

    def __init__(self, inch):
        super().__init__()
        self.dec0 = _seq_with_fused_act([
            Conv2dWNUB(inch, 64, 64, 64, 3, 1, 1),
            Conv2dWNUB(64, 128, 64, 64, 3, 1, 1),
            Conv2dWNUB(128, 64, 64, 64, 3, 1, 1),
            Conv2dWNUB(64, 64, 64, 64, 3, 1, 1),
            Conv2dWNUB(64, 9, 64, 64, 3, 1, 1),
        ])
        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.dec0[-1], 1.0)

    def raw(self, local_encoding):
        """dec0 output [B, 9, 64, 64] — the input of `prim_transforms`."""
        return self.dec0(local_encoding)

    def forward(self, local_encoding):
        out = self.dec0(local_encoding)
        out = out.view(local_encoding.size(0), 9, -1).permute(0, 2, 1).contiguous()
        return out[:, :, 0:3] * 1.0e-4, out[:, :, 3:6] * 0.01, torch.exp(0.01 * out[:, :, 6:9])


class DeconvContentDecoder(nn.Module):
    """hand_mvp.py:324-348: 64^2 -> 1024^2 in four stride-2 deconvs, primsize_z * outch output channels."""

    def __init__(self, primsize_z, inch, outch):
        super().__init__()
        self.primsize_z, self.outch = primsize_z, outch
        self.texbranch = _seq_with_fused_act([
            ConvTranspose2dWNUB(inch, 32, 128, 128, 4, 2, 1),
            ConvTranspose2dWNUB(32, 32, 256, 256, 4, 2, 1),
            ConvTranspose2dWNUB(32, 16, 512, 512, 4, 2, 1),
            ConvTranspose2dWNUB(16, primsize_z * outch, 1024, 1024, 4, 2, 1),
        ])
        self.apply(lambda m: glorot(m, 0.2))
        glorot(self.texbranch[-1], 1.0)

    def forward(self, local_enc):
        return self.texbranch(local_enc)


# ------------------------------------------------------------------------------------------------ glue kernels
class _PrimTransforms(Function):
    @staticmethod
    def forward(ctx, dec, posbase, rotbase, prim_scale, zero_delta):
        dec, posbase, rotbase = dec.contiguous(), posbase.contiguous(), rotbase.contiguous()
        for t, n in ((dec, "dec"), (posbase, "primposbase"), (rotbase, "primrotbase")):
            _lib.check_input(t, n)
        B = dec.shape[0]
        K = dec.numel() // (B * 9)
        if posbase.shape != (B, K, 3) or rotbase.shape != (B, K, 3, 3):
            raise RuntimeError("primposbase must be [B,K,3] and primrotbase [B,K,3,3] with K = dec.numel()/(9B)")
        dev = dec.device
        primpos = torch.empty(B, K, 3, device=dev)
        primrot = torch.empty(B, K, 3, 3, device=dev)
        primscale = torch.empty(B, K, 3, device=dev)
        _lib.kernels().gb_mvp_prim_transform_fwd(
            B, K, dec, posbase, rotbase, float(prim_scale), int(zero_delta), primpos, primrot, primscale)
        ctx.save_for_backward(dec, posbase, rotbase)
        ctx.meta = (B, K, float(prim_scale), int(zero_delta))
        ctx.set_materialize_grads(False)
        return primpos, primrot, primscale

    @staticmethod
    def backward(ctx, g_pos, g_rot, g_scale):
        dec, posbase, rotbase = ctx.saved_tensors
        B, K, prim_scale, zero_delta = ctx.meta
        g_pos, g_rot, g_scale = (None if g is None else g.contiguous() for g in (g_pos, g_rot, g_scale))
        g_dec = torch.empty_like(dec)
        _lib.kernels().gb_mvp_prim_transform_bwd(
            B, K, dec, posbase, rotbase, prim_scale, zero_delta, g_pos, g_rot, g_scale, g_dec)
        return g_dec, None, None, None, None


def prim_transforms(dec, primposbase, primrotbase, prim_scale=512.0, zero_delta=False):
    """dec [B,9,64,64] (TransDecoder.raw) + base frame -> (primpos [B,K,3], primrot [B,K,3,3], primscale [B,K,3]):
    `primposbase + primrotbase @ (1e-4 d[0:3])`, `primrotbase @ axisangle_to_matrix(0.01 d[3:6])`,
    `prim_scale * exp(0.01 d[6:9])`.  Gradients flow to `dec` only (the base frame is built under no_grad upstream)."""
    return _PrimTransforms.apply(dec, primposbase, primrotbase, prim_scale, zero_delta)


class _SlabsToPrims(Function):
    @staticmethod
    def forward(ctx, rgb, alpha, primsize, prim_slot, n_out, rgb_mul, rgb_add, relu):
        rgb, alpha = rgb.contiguous(), alpha.contiguous()
        _lib.check_input(rgb, "primrgb")
        _lib.check_input(alpha, "primalpha")
        B, PZ, three, U, U2 = rgb.shape
        if three != 3 or U != U2 or alpha.shape != (B, PZ, 1, U, U) or PZ != primsize[2]:
            raise RuntimeError("primrgb must be [B,PZ,3,U,U] and primalpha [B,PZ,1,U,U] with PZ = primsize[2]")
        PSX, PSY = int(primsize[0]), int(primsize[1])
        tpl = torch.empty(B, n_out, PZ, PSY, PSX, 4, device=rgb.device)
        _lib.kernels().gb_mvp_slab_to_prims_fwd(
            B, PZ, U, PSX, PSY, n_out, rgb, alpha, prim_slot, float(rgb_mul), float(rgb_add), int(relu), tpl)
        ctx.save_for_backward(rgb, alpha, prim_slot)
        ctx.meta = (B, PZ, U, PSX, PSY, n_out, float(rgb_mul), float(rgb_add), int(relu))
        return tpl

    @staticmethod
    def backward(ctx, g_tpl):
        rgb, alpha, prim_slot = ctx.saved_tensors
        B, PZ, U, PSX, PSY, n_out, rgb_mul, rgb_add, relu = ctx.meta
        g_tpl = g_tpl.contiguous()
        g_rgb, g_alpha = torch.empty_like(rgb), torch.empty_like(alpha)
        _lib.kernels().gb_mvp_slab_to_prims_bwd(
            B, PZ, U, PSX, PSY, n_out, rgb, alpha, prim_slot, rgb_mul, rgb_add, relu, g_tpl, g_rgb, g_alpha)
        return g_rgb, g_alpha, None, None, None, None, None, None


_SLOTS = {}


def slabs_to_primrgba(primrgb, primalpha, primsize: Tuple[int, int, int] = (16, 16, 8),
                      valid_prims: Optional[torch.Tensor] = None, raw: bool = False):
    """UV slabs -> raymarcher template [B, K, PZ, PSY, PSX, 4].

    raw=False: inputs are the activated `primrgb` / `primalpha` of the reference's preds; the result equals
    hand_mvp.py:172-185 (and, with `valid_prims` (bool [n_prims]), the `template[:, valid_prims].contiguous()` of
    render_raymarcher.py:44-46 on top).  raw=True: inputs are the decoders' raw outputs and relu(25*rgb+100),
    relu(alpha) (hand_mvp.py:472,434) are applied in the same pass."""
    n_prims = (primrgb.shape[-1] // primsize[0]) * (primrgb.shape[-2] // primsize[1])
    slot, n_out = None, n_prims
    if valid_prims is not None:
        # valid_prims is a fixed buffer of the model (hand_mvp.py:153-160): its slot table is built once.  The entry
        # holds the mask itself: a freed mask whose address is reused by another one must not hit
        key = (valid_prims.data_ptr(), valid_prims._version, primrgb.device.index)
        hit = _SLOTS.get(key)
        if hit is not None and hit[2] is not valid_prims:
            hit = None
        if hit is None:
            v = valid_prims.to(device=primrgb.device).reshape(-1).bool()
            if v.numel() != n_prims:
                raise RuntimeError("valid_prims must have one entry per primitive")
            ranks = torch.cumsum(v.to(torch.int32), 0, dtype=torch.int32) - 1
            hit = (torch.where(v, ranks, torch.full_like(ranks, -1)).contiguous(), int(v.sum().item()), valid_prims)
            if len(_SLOTS) > 16:
                _SLOTS.clear()
            _SLOTS[key] = hit
        slot, n_out = hit[0], hit[1]
    mul, add, relu = (25.0, 100.0, 1) if raw else (1.0, 0.0, 0)
    return _SlabsToPrims.apply(primrgb, primalpha, tuple(primsize), slot, n_out, mul, add, relu)


# ------------------------------------------------------------------------------------------------ mesh front end
def init_primitives(slab_size, n_prims, geo_fn):
    """hand_mvp.py:50-68: sample the UV index images at the centre texel of each primitive's slab cell.  `geo_fn` is
    the reference's GeometryModule or any holder with `vi`, `vti`, `vt` and `render_index_images(size, impaint=True)`.
    As in the reference, the face image is the un-inpainted one, and torch's indexing of `vi[face]` makes a -1 face
    index select the last face.  Returns (prim_vidx_img, prim_vtidx_img, prim_bary_img), each [S, S, 3]."""
    stride = slab_size // int(n_prims ** 0.5)
    _, face_index, bary_index = geo_fn.render_index_images(slab_size, impaint=True)
    bary_index = torch.as_tensor(bary_index, device=geo_fn.vt.device)
    cell = (slice(stride // 2, None, stride), slice(stride // 2, None, stride))
    face = face_index[cell]
    return geo_fn.vi[face], geo_fn.vti[face], bary_index[cell]


def _frame_inputs(geom, name):
    if torch.is_grad_enabled() and geom.requires_grad:
        raise RuntimeError("%s: the base frames carry no gradient (the reference builds them under no_grad)" % name)
    geom = geom.contiguous()
    _lib.check_input(geom, "geom")
    return geom


def _i32(t):
    return t.to(torch.int32).contiguous()


def prim_base_frames(geom_lbs, vt, prim_vidx_img, prim_vtidx_img, prim_bary_img):
    """make_postex + compute_tbn (geom.py:355-397,515-520) as GeomDecoder.forward uses them (hand_mvp.py:393-408), in
    one kernel: geom_lbs [B,V,3] posed vertices -> (primposbase [B,K,3], primrotbase [B,K,3,3] with columns T, B, N),
    K = S*S texels of the [S,S,3] index / barycentric images."""
    geom = _frame_inputs(geom_lbs, "prim_base_frames")
    vidx, vtidx = _i32(prim_vidx_img), _i32(prim_vtidx_img)
    bary, vt = prim_bary_img.to(torch.float32).contiguous(), vt.to(torch.float32).contiguous()
    for t, n in ((vidx, "prim_vidx_img"), (vtidx, "prim_vtidx_img")):
        _lib.check_input(t, n, torch.int32)
    _lib.check_input(bary, "prim_bary_img")
    _lib.check_input(vt, "vt")
    B, V = geom.shape[0], geom.shape[1]
    T = vidx.numel() // 3
    if vidx.shape[-1] != 3 or vtidx.shape != vidx.shape or bary.shape != vidx.shape or vt.shape[-1] != 2:
        raise RuntimeError("index / barycentric images must be [S,S,3] and vt [NT,2]")
    posbase = torch.empty(B, T, 3, device=geom.device)
    rotbase = torch.empty(B, T, 3, 3, device=geom.device)
    _lib.kernels().gb_mvp_prim_frames_fwd(
        B, V, vt.shape[0], T, geom, vidx, vtidx, bary, vt, None, None, posbase, rotbase, None)
    return posbase, rotbase


def view_cos_uv(geom_lbs, vi, campos, prim_vidx_img, prim_bary_img):
    """compute_view_cos + values_to_uv (geom.py:308-352) as hand_mvp.AutoEncoder.forward uses them (:230-236):
    geom_lbs [B,V,3], vi [F,3] faces, campos [B,3] -> [B,1,S,S], zero at texels with a -1 index.  The vertex normals
    come from `geom.vert_normals` (gb_vert_normals_fwd)."""
    geom = _frame_inputs(geom_lbs, "view_cos_uv")
    vidx = _i32(prim_vidx_img)
    bary = prim_bary_img.to(torch.float32).contiguous()
    campos = campos.to(torch.float32).contiguous()
    _lib.check_input(vidx, "prim_vidx_img", torch.int32)
    _lib.check_input(bary, "prim_bary_img")
    _lib.check_input(campos, "campos")
    B, V = geom.shape[0], geom.shape[1]
    S0, S1 = vidx.shape[0], vidx.shape[1]
    if vidx.shape != (S0, S1, 3) or bary.shape != vidx.shape or campos.shape != (B, 3):
        raise RuntimeError("prim_vidx_img / prim_bary_img must be [S,S,3] and campos [B,3]")
    vn = vert_normals(geom, vi)
    out = torch.empty(B, 1, S0, S1, device=geom.device)
    _lib.kernels().gb_mvp_prim_frames_fwd(
        B, V, 0, S0 * S1, geom, vidx, None, bary, None, vn, campos, None, None, out)
    return out


class GeomDecoder(nn.Module):
    """hand_mvp.py:351-444 with the reference's constructor, submodules (`lbs_fn`, `transdecoder`, `alphadecoder`)
    and non-persistent `prim_*_img` buffers.  The front end (pose, base frames) runs under no_grad on the kernels;
    `prim_transforms` composes it with TransDecoder's deltas, and the alpha slab's ReLU runs inside the last deconv."""

    def __init__(self, inch, primsize_z, uv_size, n_prims, lbs_fn, geo_fn, primposstart, prim_scale=512):
        super().__init__()
        self.lbs_fn = lbs_fn
        self.geo_fn = geo_fn
        self.primposstart = primposstart
        self.uv_size = uv_size
        self.n_prims = n_prims
        self.primsize_z = primsize_z
        self.prim_scale = prim_scale
        prim_vidx_img, prim_vtidx_img, prim_bary_img = init_primitives(uv_size, n_prims, geo_fn)
        self.register_buffer("prim_vidx_img", prim_vidx_img, persistent=False)
        self.register_buffer("prim_vtidx_img", prim_vtidx_img, persistent=False)
        self.register_buffer("prim_bary_img", prim_bary_img, persistent=False)
        self.transdecoder = TransDecoder(inch)
        self.alphadecoder = DeconvContentDecoder(primsize_z, inch, 1)

    def forward(self, pose, joint, iteration=-1):
        B = pose.shape[0]
        with torch.no_grad():
            geom_lbs = self.lbs_fn.pose(torch.zeros_like(self.lbs_fn.lbs_template_verts), pose)
            primposbase, primrotbase = prim_base_frames(geom_lbs, self.geo_fn.vt, self.prim_vidx_img,
                                                        self.prim_vtidx_img, self.prim_bary_img)
        zero_delta = bool(self.training and iteration < self.primposstart)
        primpos, primrot, primscale = prim_transforms(self.transdecoder.raw(joint), primposbase, primrotbase,
                                                      self.prim_scale, zero_delta)
        tex = self.alphadecoder.texbranch
        alpha = tex[-1](tex[:-1](joint), slope=0.0)  # LeakyReLU(0) = the reference's F.relu (:434)
        alpha = alpha.view(B, self.primsize_z, 1, self.uv_size, self.uv_size)
        return {"primalpha": alpha, "primpos": primpos, "primscale": primscale, "primrot": primrot,
                "geom_lbs": geom_lbs}


class RGBSlabDecoder(nn.Module):
    """hand_mvp.py:447-474: the bilinear AO resize and the concatenation in torch, the deconv tower on the kernels,
    then relu(25 x + 100)."""

    def __init__(self, inch, primsize_z, uv_size, geo_fn):
        super().__init__()
        self.geo_fn = geo_fn
        self.primsize_z = primsize_z
        self.uv_size = uv_size
        self.texdecoder = DeconvContentDecoder(primsize_z, inch, 3)

    def forward(self, view_cos_uv, joint, ambient_occlusion):
        B = joint.shape[0]
        ao_ds = F.interpolate(ambient_occlusion, (64, 64), mode="bilinear")
        rgb = self.texdecoder(torch.cat((joint, view_cos_uv, ao_ds), 1))
        rgb = rgb.view(B, self.primsize_z, 3, self.uv_size, self.uv_size)
        return F.relu(25.0 * rgb + 100.0)


# ------------------------------------------------------------------------------------------------ the frame
class _ValidGather(Function):
    """Raymarcher.forward's primpos / volradius and valid-primitive selection (render_raymarcher.py:36-47) in one
    launch of csrc/hand_frame.cu; the backward writes the full-size gradients once (zero at invalid primitives)."""

    @staticmethod
    def forward(ctx, template, primpos, primrot, primscale, slot, n_valid, volradius):
        template, primpos = template.contiguous(), primpos.contiguous()
        primrot, primscale = primrot.contiguous(), primscale.contiguous()
        for t, n in ((template, "primrgba"), (primpos, "primpos"), (primrot, "primrot"), (primscale, "primscale")):
            _lib.check_input(t, n)
        _lib.check_input(slot, "slot table", torch.int32)
        B, K = template.shape[:2]
        E = template[0, 0].numel()
        if (primpos.shape != (B, K, 3) or primrot.shape != (B, K, 3, 3) or primscale.shape != (B, K, 3)
                or slot.shape != (K,)):
            raise RuntimeError("valid gather: template [B,K,...], primpos / primscale [B,K,3], primrot [B,K,3,3] and "
                               "a slot table [K] (got K = %d, slot %s)" % (K, tuple(slot.shape)))
        # torch evaluates `primpos / volradius` as primpos * (1 / volradius) in fp32 (div by a CPU scalar)
        inv = float(torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(volradius), dtype=torch.float32))
        dev = template.device
        tpl = torch.empty((B, n_valid) + tuple(template.shape[2:]), device=dev)
        pos, scale = torch.empty(B, n_valid, 3, device=dev), torch.empty(B, n_valid, 3, device=dev)
        rot = torch.empty(B, n_valid, 3, 3, device=dev)
        _lib.kernels().gb_hand_valid_gather_fwd(
            B, K, n_valid, E, slot, template, primpos, primrot, primscale, inv, tpl, pos, rot, scale)
        ctx.save_for_backward(slot)
        ctx.meta = (tuple(template.shape), n_valid, inv)
        return tpl, pos, rot, scale

    @staticmethod
    def backward(ctx, g_tpl, g_pos, g_rot, g_scale):
        (slot,) = ctx.saved_tensors
        shape, n_valid, inv = ctx.meta
        B, K = shape[:2]
        g_tpl, g_pos, g_rot, g_scale = (g.contiguous() for g in (g_tpl, g_pos, g_rot, g_scale))
        dev = g_tpl.device
        gt = torch.empty(shape, device=dev)
        gp, gr, gs = torch.empty(B, K, 3, device=dev), torch.empty(B, K, 3, 3, device=dev), torch.empty(B, K, 3,
                                                                                                      device=dev)
        _lib.kernels().gb_hand_valid_gather_bwd(
            B, K, n_valid, gt[0, 0].numel(), slot, g_tpl, g_pos, g_rot, g_scale, inv, gt, gp, gr, gs)
        return gt, gp, gr, gs, None, None, None


def valid_gather(template, primpos, primrot, primscale, slot, n_valid, volradius):
    """(template [B,K,TD,TH,TW,4], primpos, primrot, primscale) -> the same tensors at the n_valid primitives with
    slot[k] >= 0, in slot order, and primpos divided by volradius: the march inputs render_raymarcher.py:36-47 builds.
    `slot` [K] int32 (rank among the valid primitives, -1 for the others) and n_valid come from the host, so the
    call issues no host synchronisation."""
    return _ValidGather.apply(template, primpos, primrot, primscale, slot, int(n_valid), float(volradius))


def slot_table(valid_prims):
    """bool [K] -> (slot [K] int32: rank among the valid entries, -1 elsewhere; the number of valid entries), on
    valid_prims' device"""
    v = valid_prims.reshape(-1).to(torch.bool)
    ranks = torch.cumsum(v.to(torch.int32), 0, dtype=torch.int32) - 1
    return torch.where(v, ranks, torch.full_like(ranks, -1)), int(v.sum())


class _HandFinish(Function):
    """rayrgba [B,H,W,4] -> calibrated rgb (+ training background) [B,3,H,W], alpha [B,1,H,W] on csrc/hand_frame.cu"""

    @staticmethod
    def forward(ctx, rayrgba, cal_w, cal_b, grey, bg):
        rayrgba = rayrgba.contiguous()
        _lib.check_input(rayrgba, "rayrgba")
        B, H, W, four = rayrgba.shape
        if four != 4:
            raise RuntimeError("hand_finish: rayrgba must be [B,H,W,4]")
        opt = {}
        for name, t, shape, dt in (("cal_w", cal_w, (B, 3), torch.float32), ("cal_b", cal_b, (B, 3), torch.float32),
                                   ("grey", grey, (B,), torch.int32), ("background", bg, (B, 3, H, W), torch.float32)):
            if t is not None:
                t = t.contiguous()
                _lib.check_input(t, name, dt)
                if tuple(t.shape) != shape:
                    raise RuntimeError("hand_finish: %s must have shape %s (got %s)" % (name, shape, tuple(t.shape)))
            opt[name] = t
        if (opt["cal_w"] is None) != (opt["cal_b"] is None):
            raise RuntimeError("hand_finish: cal_w and cal_b go together")
        dev = rayrgba.device
        rgb, alpha = torch.empty(B, 3, H, W, device=dev), torch.empty(B, 1, H, W, device=dev)
        _lib.kernels().gb_hand_finish_fwd(
            B, H, W, rayrgba, opt["cal_w"], opt["cal_b"], opt["grey"], opt["background"], rgb, alpha)
        ctx.save_for_backward(rayrgba, opt["cal_w"], opt["grey"], opt["background"])
        ctx.set_materialize_grads(False)
        return rgb, alpha

    @staticmethod
    def backward(ctx, g_rgb, g_alpha):
        rayrgba, cal_w, grey, bg = ctx.saved_tensors
        B, H, W, _ = rayrgba.shape
        dev = rayrgba.device
        if g_rgb is None:
            g_rgb = torch.zeros(B, 3, H, W, device=dev)
        g_rgb = g_rgb.contiguous()
        g_alpha = None if g_alpha is None else g_alpha.contiguous()
        g_ray = torch.empty_like(rayrgba)
        g_cw = g_cb = ws = None
        L = _lib.kernels()
        if cal_w is not None:
            g_cw, g_cb = torch.empty(B, 3, device=dev), torch.empty(B, 3, device=dev)
            ws = torch.empty(L.gb_hand_finish_workspace_bytes(B, H, W) // 4, device=dev)
        L.gb_hand_finish_bwd(B, H, W, rayrgba, cal_w, grey, bg, g_rgb, g_alpha, g_ray, g_cw, g_cb, ws)
        return g_ray, g_cw, g_cb, None, None


def hand_finish(rayrgba, cal_w=None, cal_b=None, grey=None, background=None):
    """The raymarcher's channels-last rayrgba [B,H,W,4] -> (rgb [B,3,H,W], alpha [B,1,H,W]) with, in the reference's
    order (hand_mvp.py:249-255), the calibration rows of `CalV5.rows` (cal_w / cal_b [B,3], grey [B] int32) and the
    training background [B,3,H,W]: rgb = cal(rayrgb) + (1 - alpha) * background.  Any stage whose tensors are None is
    skipped.  Gradients: rayrgba (its alpha channel also through the background term), cal_w, cal_b."""
    return _HandFinish.apply(rayrgba, cal_w, cal_b, grey, background)


class Raymarcher(nn.Module):
    """render_raymarcher.py:17-24: the volume radius and the step size dt / volume_radius (no parameters)"""

    def __init__(self, volradius, dt: float = 1.0):
        super().__init__()
        self.volume_radius = volradius
        self.dt = dt / self.volume_radius


class _ImageSize(nn.Module):
    """the state of pytorch3d's RenderLayer (render_pytorch3d.py:30-31): its persistent `image_size` [2] int32.  The
    frame never rasterises the mesh, so this holds the checkpoint key only."""

    def __init__(self, h, w):
        super().__init__()
        self.register_buffer("image_size", torch.as_tensor([h, w], dtype=torch.int32))


class _InpaintedIndexImages:
    """what `init_primitives` reads of a geometry module: vi, vti, vt and render_index_images(size, impaint=True),
    whose face and barycentric images come from the assets"""

    def __init__(self, geo_fn, face_index, bary):
        self.vi, self.vti, self.vt = geo_fn.vi.to(torch.int64), geo_fn.vti.to(torch.int64), geo_fn.vt
        self.face_index, self.bary = face_index, bary

    def render_index_images(self, uv_size, flip_uv=False, impaint=False):
        if uv_size != self.face_index.shape[0]:
            raise ValueError("the assets' inpainted index images are %d x %d, not %d"
                             % (self.face_index.shape[0], self.face_index.shape[1], uv_size))
        return None, self.face_index, self.bary


HAND_UV_IMAGES = ("face_index_image_impaint", "bary_image_impaint")


class AutoEncoder(nn.Module):
    """hand_mvp.AutoEncoder (ca_code/models/hand_mvp.py:71-266): the hand avatar's frame with the reference's
    constructor, submodules and state-dict keys (`geomdecoder.{lbs_fn,geo_fn}.*` and `rgbdecoder.geo_fn.*` repeat the
    shared modules), so `AutoEncoder(**config.model, assets=assets)` builds from hand_mvp_example.yml and a reference
    checkpoint loads with strict=True.

    `assets` (attributes or dict keys) carries the reference's assets and, because this project does not rasterise UV
    layouts, the four `geo_fn` images (`mesh_vae._uv_geometry`) plus what `render_index_images(1024, impaint=True)`
    returns for `init_primitives`: face_index_image_impaint [1024,1024] and bary_image_impaint [1024,1024,3].
    `renderer` holds only the mesh renderer's `image_size` key: the frame never rasterises the mesh.

    `valid_prims`, its slot table and its count are built once on the host at construction, so forward() (CUDA only)
    and its backward issue no host synchronisation after the first call.  preds["primrgba"] is the full
    [B, n_prims, 8, 16, 16, 4] template, as in the reference; the raymarcher receives its valid primitives only."""

    def __init__(self, assets, image_height, image_width, cal=None, n_pose_dims: int = 54, n_embs: int = 64,
                 volradius: float = 2000.0, primsize: Tuple[int, int, int] = (16, 16, 8), learn_blur: bool = True):
        super().__init__()
        import numpy as np

        from .lbs import LBSModule
        from .mesh_vae import UV_IMAGES, _get, _uv_geometry
        from .photo_loss import CalV5, LearnableBlur

        missing = [k for k in UV_IMAGES + HAND_UV_IMAGES if _get(assets, k) is None]
        if missing:
            raise ValueError("hand_mvp.AutoEncoder: assets must carry the UV images %s at 1024 x 1024; missing: %s"
                             % (", ".join(UV_IMAGES + HAND_UV_IMAGES), ", ".join(missing)))
        self.uv_size = 1024
        self.primsize = tuple(primsize)
        self.n_prim_x = self.uv_size // self.primsize[0]
        self.n_prim_y = self.uv_size // self.primsize[1]
        self.n_prims = self.n_prim_x * self.n_prim_y
        self.height, self.width = image_height, image_width
        self.volradius = volradius
        template = torch.as_tensor(np.asarray(_get(assets, "template_mesh_unscaled")), dtype=torch.float32)
        self.lbs_fn = LBSModule(_get(assets, "lbs_model_json"), _get(assets, "lbs_config_dict"), template[None],
                                _get(assets, "skeleton_scales"), global_scaling=[10.0, 10.0, 10.0])
        self.geo_fn, _ = _uv_geometry(assets)
        imgs = {k: torch.as_tensor(np.asarray(_get(assets, k))) for k in HAND_UV_IMAGES}
        if tuple(imgs["face_index_image_impaint"].shape) != (1024, 1024) or \
                tuple(imgs["bary_image_impaint"].shape) != (1024, 1024, 3):
            raise ValueError("hand_mvp.AutoEncoder: face_index_image_impaint must be [1024,1024] and "
                             "bary_image_impaint [1024,1024,3]")

        self.poseencoder = PoseEncoder(n_pose_dims, n_embs, self.n_prim_x)
        index_images = _InpaintedIndexImages(self.geo_fn, imgs["face_index_image_impaint"].to(torch.int64),
                                             imgs["bary_image_impaint"].to(torch.float32))
        self.geomdecoder = GeomDecoder(n_embs, self.primsize[2], self.uv_size, self.n_prims, self.lbs_fn,
                                       index_images, primposstart=1000)
        self.geomdecoder.geo_fn = self.geo_fn
        self.rgbdecoder = RGBSlabDecoder(n_embs + 2, self.primsize[2], self.uv_size, self.geo_fn)
        self.raymarcher = Raymarcher(volradius=self.volradius, dt=1.0)
        self.renderer = _ImageSize(image_height, image_width)
        cameras = _get(assets, "camera_ids")
        self.learn_blur_enabled = bool(learn_blur)
        if self.learn_blur_enabled:
            self.learn_blur = LearnableBlur(cameras)
        self.cal_enabled = cal is not None
        if self.cal_enabled:
            self.cal = CalV5(**cal, cameras=cameras)

        # hand_mvp.py:153-160, once on the host, with the gather's slot table and count
        valid_mask = F.interpolate(self.geo_fn.valid_mask.float()[None].permute(0, 3, 1, 2),
                                   (self.n_prim_x, self.n_prim_y), mode="area")
        valid_prims = (valid_mask != 0).reshape(-1)
        self.register_buffer("valid_prims", valid_prims, persistent=False)
        slot, self.n_valid = slot_table(valid_prims)
        self.register_buffer("valid_slot", slot, persistent=False)

    def forward(self, pose, campos, ambient_occlusion=None, K=None, Rt=None, camera_id=None, frame_id=None,
                embs=None, encode=True, iteration=None, background=None, **kwargs):
        for t, n in ((pose, "pose"), (campos, "campos"), (K, "K"), (Rt, "Rt")):
            if t is None or not t.is_cuda:
                raise RuntimeError("hand_mvp.AutoEncoder runs on CUDA only (no CPU fallback): %s is %s"
                                   % (n, "missing" if t is None else "on %s" % t.device))
        B = pose.shape[0]
        joint = self.poseencoder(pose)
        geo_preds = self.geomdecoder(pose, joint, iteration)
        gd = self.geomdecoder
        with torch.no_grad():
            vc = view_cos_uv(geo_preds["geom_lbs"], self.geo_fn.vi, campos, gd.prim_vidx_img, gd.prim_bary_img)
        # RGBSlabDecoder.forward (hand_mvp.py:457-474) with the deconv tower's raw output kept: the template takes it
        # with the activation applied in the slab kernel, so the template's gradient skips the torch activation
        ao_ds = F.interpolate(ambient_occlusion, (64, 64), mode="bilinear")
        rd = self.rgbdecoder
        raw = rd.texdecoder(torch.cat((joint, vc, ao_ds), 1)).view(B, rd.primsize_z, 3, rd.uv_size, rd.uv_size)
        primrgb = F.relu(25.0 * raw + 100.0)
        primrgba = slabs_to_primrgba(raw, geo_preds["primalpha"], self.primsize, raw=True)
        preds = {"primrgb": primrgb, "valid_prims": self.valid_prims, **geo_preds, "primrgba": primrgba}
        rgb, alpha = self._finish(self._march(K, Rt, preds), camera_id, background)
        preds.update(rgb=rgb, alpha=alpha)
        self._blur(preds, camera_id)
        return preds

    def _march(self, K, Rt, preds):
        """AutoEncoder.render (hand_mvp.py:187-203) and Raymarcher.forward (render_raymarcher.py:36-70): the camera
        of K / Rt, its rays, the valid primitives of preds["primrgba"] and the primitive transforms, and the march ->
        channels-last rayrgba [B,H,W,4]"""
        from .mvpraymarch import mvpraymarch  # looked up per call, so a test can wrap the march
        from .utils import compute_raydirs

        for t, n in ((K, "K"), (Rt, "Rt"), (preds["primrgba"], "primrgba")):
            if t is None or not t.is_cuda:
                raise RuntimeError("hand_mvp.AutoEncoder runs on CUDA only (no CPU fallback): %s is %s"
                                   % (n, "missing" if t is None else "on %s" % t.device))
        focal = torch.diagonal(K[:, :2, :2], dim1=1, dim2=2).contiguous()
        princpt = K[:, :2, 2].contiguous()
        camrot = Rt[:, :3, :3].contiguous()
        ray_campos = -(camrot.transpose(-2, -1) @ Rt[:, :3, 3:4])[..., 0]
        raypos, raydir, tminmax = compute_raydirs(ray_campos.contiguous(), camrot, focal, princpt,
                                                  (self.width, self.height), self.raymarcher.volume_radius)
        tpl, pos, rot, scale = valid_gather(preds["primrgba"], preds["primpos"], preds["primrot"], preds["primscale"],
                                            self.valid_slot, self.n_valid, self.raymarcher.volume_radius)
        return mvpraymarch(raypos, raydir, self.raymarcher.dt, tminmax, (pos, rot, scale), template=tpl, warp=None)

    def _finish(self, rayrgba, camera_id, background):
        """the march's rgb / alpha [B,·,H,W], calibrated and, in training, over the background (hand_mvp.py:249-255)"""
        cal_w = cal_b = grey = None
        if self.cal_enabled:
            cal_w, cal_b, grey = self.cal.rows(self.cal.name_to_idx(camera_id))
        bg = background[:, :3] if self.training and background is not None else None
        return hand_finish(rayrgba, cal_w, cal_b, grey, bg)

    def _blur(self, preds, camera_id):
        if self.learn_blur_enabled:
            preds["rgb"] = self.learn_blur(preds["rgb"], camera_id)
            preds["learn_blur_weights"] = self.learn_blur.reg(camera_id)

    def render(self, K, Rt, preds, with_shadow: bool = False):
        """hand_mvp.py:162-205: the template of preds["primrgb"] (activated) and preds["primalpha"], stored as
        preds["primrgba"] [B, n_prims, 8, 16, 16, 4], marched from the cameras K / Rt -> (rgb [B,3,H,W],
        alpha [B,1,H,W], None), uncalibrated.  HandMVPSummary draws the teacher's shadow image with it.  No frame
        marches with `with_shadow=True`, so it raises."""
        if with_shadow:
            raise NotImplementedError("hand_mvp.AutoEncoder.render: with_shadow=True is not supported")
        preds["primrgba"] = slabs_to_primrgba(preds["primrgb"], preds["primalpha"], self.primsize)
        rgb, alpha = hand_finish(self._march(K, Rt, preds))
        return rgb, alpha, None
