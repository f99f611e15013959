"""Host-side mirror of the hand-MVP decoders (SURVEY.md §8 row R8): `PoseEncoder`, `TransDecoder`,
`DeconvContentDecoder` (ca_code/models/hand_mvp.py:269-348) with the reference's module / parameter names so its
checkpoints load, plus the two glue stages between those decoders and the raymarcher as single kernels:

  * `prim_transforms`   — TransDecoder's head scaling + GeomDecoder's composition with the mesh-attached base frame
                          (hand_mvp.py:317-321, 410-425, 477-510), csrc/mvp_prims.cu
  * `slabs_to_primrgba` — output activations + cat/permute/reshape + valid-primitive gather
                          (hand_mvp.py:434,472,172-185; render_raymarcher.py:44-46), csrc/mvp_prims.cu

The mesh front end (DESIGN.md row R8') runs on kernels too: `GeomDecoder` poses the mesh with `lbs.LBSModule` and
builds each primitive's base frame with `prim_base_frames`; `view_cos_uv` gives the RGB decoder's view conditioning
(hand_mvp.py:230-236), both on csrc/mvp_prims.cu."""
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
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gb_mvp_prim_transform_fwd(
                B, K, _lib.ptr(dec), _lib.ptr(posbase), _lib.ptr(rotbase), float(prim_scale), int(zero_delta),
                _lib.ptr(primpos), _lib.ptr(primrot), _lib.ptr(primscale), _lib.stream_ptr(dev)), "mvp_prim_transform_fwd")
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
        with torch.cuda.device(dec.device):
            _lib.check(_lib.lib().gb_mvp_prim_transform_bwd(
                B, K, _lib.ptr(dec), _lib.ptr(posbase), _lib.ptr(rotbase), prim_scale, zero_delta, _lib.ptr(g_pos),
                _lib.ptr(g_rot), _lib.ptr(g_scale), _lib.ptr(g_dec), _lib.stream_ptr(dec.device)), "mvp_prim_transform_bwd")
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
        with torch.cuda.device(rgb.device):
            _lib.check(_lib.lib().gb_mvp_slab_to_prims_fwd(
                B, PZ, U, PSX, PSY, n_out, _lib.ptr(rgb), _lib.ptr(alpha), _lib.ptr(prim_slot), float(rgb_mul),
                float(rgb_add), int(relu), _lib.ptr(tpl), _lib.stream_ptr(rgb.device)), "mvp_slab_to_prims_fwd")
        ctx.save_for_backward(rgb, alpha, prim_slot)
        ctx.meta = (B, PZ, U, PSX, PSY, n_out, float(rgb_mul), float(rgb_add), int(relu))
        return tpl

    @staticmethod
    def backward(ctx, g_tpl):
        rgb, alpha, prim_slot = ctx.saved_tensors
        B, PZ, U, PSX, PSY, n_out, rgb_mul, rgb_add, relu = ctx.meta
        g_tpl = g_tpl.contiguous()
        g_rgb, g_alpha = torch.empty_like(rgb), torch.empty_like(alpha)
        with torch.cuda.device(rgb.device):
            _lib.check(_lib.lib().gb_mvp_slab_to_prims_bwd(
                B, PZ, U, PSX, PSY, n_out, _lib.ptr(rgb), _lib.ptr(alpha), _lib.ptr(prim_slot), rgb_mul, rgb_add, relu,
                _lib.ptr(g_tpl), _lib.ptr(g_rgb), _lib.ptr(g_alpha), _lib.stream_ptr(rgb.device)), "mvp_slab_to_prims_bwd")
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
    with torch.cuda.device(geom.device):
        _lib.check(_lib.lib().gb_mvp_prim_frames_fwd(
            B, V, vt.shape[0], T, _lib.ptr(geom), _lib.ptr(vidx), _lib.ptr(vtidx), _lib.ptr(bary), _lib.ptr(vt), None,
            None, _lib.ptr(posbase), _lib.ptr(rotbase), None, _lib.stream_ptr(geom.device)), "mvp_prim_frames_fwd")
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
    with torch.cuda.device(geom.device):
        _lib.check(_lib.lib().gb_mvp_prim_frames_fwd(
            B, V, 0, S0 * S1, _lib.ptr(geom), _lib.ptr(vidx), None, _lib.ptr(bary), None, _lib.ptr(vn),
            _lib.ptr(campos), None, None, _lib.ptr(out), _lib.stream_ptr(geom.device)), "mvp_prim_frames_fwd")
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
