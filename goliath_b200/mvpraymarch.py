"""Host-side mirror of the reference wrapper extensions/mvpraymarch/mvpraymarch.py: `build_accel` (:21-84),
`MVPRaymarch` (:87-311) and `mvpraymarch` (:314-418) with the same names, keyword arguments (ca_code/utils/
render_raymarcher.py:59 introspects `mvpraymarch.__code__.co_varnames`), asserts and gradient wiring, calling the
sm_90a kernels through `mvpraymarchlib`.

Differences that do not change results: the fixed-order heap topology (a function of N, K only) is cached per
device instead of being rebuilt with torch ops on every call; bounds scratch is a cached workspace."""
import torch
from torch.autograd import Function

from . import mvpraymarchlib

_TOPOLOGY = {}


def _fixedorder_topology(N, K, dev):
    """sortedobjid [N,K] = k; implicit heap over 2K-1 nodes: children (2i+1, 2i+2) for internal i < K-1 (the values
    stored for leaves are never read), parent floor((i-1)/2), root -1 (mvpraymarch.py:44-73)."""
    key = (N, K, dev.index)
    hit = _TOPOLOGY.get(key)
    if hit is None:
        sortedobjid = (torch.arange(N * K, dtype=torch.int32, device=dev) % K).view(N, K)
        nodechildren = (
            torch.cat([
                torch.arange(1, (K - 1) * 2 + 1, dtype=torch.int32, device=dev),
                torch.div(torch.arange(-2, -(K * 2 + 1) - 1, -1, dtype=torch.int32, device=dev), 2, rounding_mode="floor"),
            ], dim=0).view(1, K + K - 1, 2).repeat(N, 1, 1))
        nodeparent = (torch.div(torch.arange(-1, K * 2 - 2, dtype=torch.int32, device=dev), 2, rounding_mode="floor")
                      .view(1, -1).repeat(N, 1))
        hit = (sortedobjid.contiguous(), nodechildren.contiguous(), nodeparent.contiguous())
        if len(_TOPOLOGY) > 16:
            _TOPOLOGY.clear()
        _TOPOLOGY[key] = hit
    return hit


def build_accel(primtransfin, algo, fixedorder=False):
    """Bounds of the acceleration structure for the primitives (mvpraymarch.py:21-84).  Only the fixed-order heap is
    a functional path of the reference (SURVEY.md §0.9)."""
    primpos, primrot, primscale = primtransfin
    N, K = primpos.size(0), primpos.size(1)
    dev = primpos.device
    if not fixedorder:
        raise NotImplementedError("usebvh=True builds a tree the reference traversal never reads; use 'fixedorder'")
    sortedobjid, nodechildren, nodeparent = _fixedorder_topology(N, K, dev)
    nodeaabb = torch.empty((N, K + K - 1, 2, 3), dtype=torch.float32, device=dev)
    mvpraymarchlib.compute_aabb(*primtransfin, sortedobjid, nodechildren, nodeparent, nodeaabb, algo)
    return sortedobjid, nodechildren, nodeaabb


def _block(opt):
    return opt if isinstance(opt, tuple) else (opt, 1)


def _check_march_inputs(raypos, raydir, tminmax, primpos, primrot, primscale, template, warp, chlast):
    for name, t, last in (("raypos", raypos, 3), ("raydir", raydir, 3), ("tminmax", tminmax, 2)):
        assert t.is_contiguous() and t.size(3) == last, "%s must be contiguous [N,H,W,%d]" % (name, last)
    for name, t in (("primpos", primpos), ("primrot", primrot), ("primscale", primscale)):
        assert t is None or (t.is_contiguous() and t.size(2) == 3), name
    assert template.is_contiguous() and template.dim() == 6
    ch = -1 if chlast else 2
    assert template.size(ch) == 4
    assert warp is None or (warp.is_contiguous() and warp.size(ch) == 3)


class MVPRaymarch(Function):
    """autograd node around mvpraymarchlib.raymarch_forward / raymarch_backward (mvpraymarch.py:87-311 upstream)."""

    @staticmethod
    def forward(self, raypos, raydir, stepsize, tminmax, primpos, primrot, primscale, template, warp, rayterm, gradmode,
                options):
        o = options
        _check_march_inputs(raypos, raydir, tminmax, primpos, primrot, primscale, template, warp, o["chlast"])
        transf = (primpos, primrot, primscale)
        tree = (None, None, None)
        if o["usebvh"] is not False:
            tree = build_accel(transf, o["algo"], fixedorder=o["usebvh"] == "fixedorder")
        sortedobjid, nodechildren, nodeaabb = tree

        N, H, W = raypos.shape[:3]
        dev = raypos.device
        rayrgba = torch.empty((N, H, W, 4), device=dev)
        # written for every ray by the kernel, so no fill(-1) pass (the reference pre-fills it, mvpraymarch.py:150)
        raysat = torch.empty((N, H, W, 3), device=dev) if gradmode else None
        shadow = None
        if o["with_shadow"]:
            vol = template.shape[:-1] + (2,) if o["chlast"] else template.shape[:2] + (2,) + template.shape[3:]
            shadow = torch.zeros(vol, device=template.device, dtype=torch.float32)

        bx, by = _block(o["blocksize"])
        mvpraymarchlib.raymarch_forward(
            raypos, raydir, stepsize, tminmax, sortedobjid, nodechildren, nodeaabb, *transf, template, warp, rayrgba,
            raysat, None, shadow, o["algo"], o["sortprims"], o["maxhitboxes"], o["synchitboxes"], o["chlast"],
            o["fadescale"], o["fadeexp"], o["accum"], o["termthresh"], o["griddim"], bx, by)

        self.save_for_backward(raypos, raydir, tminmax, sortedobjid, nodechildren, nodeaabb, primpos, primrot, primscale,
                               template, warp, rayrgba, raysat)
        self.options, self.stepsize = o, stepsize
        return rayrgba, shadow

    @staticmethod
    def backward(self, grad_rayrgba, grad_shadow):
        (raypos, raydir, tminmax, sortedobjid, nodechildren, nodeaabb, primpos, primrot, primscale, template, warp, rayrgba,
         raysat) = self.saved_tensors
        o = self.options
        # accumulated into by the kernel (REDs), hence zero-filled
        g_pos, g_rot, g_scale = (torch.zeros_like(t) for t in (primpos, primrot, primscale))
        g_template = torch.zeros_like(template)
        g_warp = None if warp is None else torch.zeros_like(warp)
        bx, by = _block(o["bwdblocksize"])
        mvpraymarchlib.raymarch_backward(
            raypos, raydir, self.stepsize, tminmax, sortedobjid, nodechildren, nodeaabb, primpos, g_pos, primrot, g_rot,
            primscale, g_scale, template, g_template, warp, g_warp, rayrgba, grad_rayrgba.contiguous(), raysat, None,
            o["algo"], o["sortprims"], o["maxhitboxes"], o["synchitboxes"], o["chlast"], o["fadescale"], o["fadeexp"],
            o["accum"], o["termthresh"], o["griddim"], bx, by)
        return (None, None, None, None, g_pos, g_rot, g_scale, g_template, g_warp, None, None, None)


def mvpraymarch(
    raypos,
    raydir,
    stepsize,
    tminmax,
    primtransf,
    template,
    warp,
    rayterm=None,
    algo=0,
    usebvh="fixedorder",
    sortprims=False,
    randomorder=False,
    maxhitboxes=512,
    synchitboxes=True,
    chlast=True,
    fadescale=8.0,
    fadeexp=8.0,
    accum=2,
    termthresh=0.99,
    griddim=3,
    blocksize=(8, 16),
    bwdblocksize=(8, 16),
    with_shadow=False,
):
    """Main entry point for raymarching MVP (argument meaning: extensions/mvpraymarch/mvpraymarch.py:341-378).

    raypos, raydir [N,H,W,3]; tminmax [N,H,W,2]; primtransf = (primpos [N,K,3], primrot [N,K,3,3], primscale [N,K,3])
    or a packed [N,K,5,3] tensor; template [N,K,TD,TH,TW,4] (chlast); warp [N,K,WD,WH,WW,3] or None.
    algo 0 = no warp field, 1 = warp field.  Returns rayrgba [N,H,W,4] (and the shadow volume when with_shadow)."""
    if isinstance(primtransf, tuple):
        primpos, primrot, primscale = primtransf
    else:
        primpos, primrot, primscale = (primtransf[:, :, 0, :].contiguous(), primtransf[:, :, 1:4, :].contiguous(),
                                       primtransf[:, :, 4, :].contiguous())
    primtransfin = (primpos, primrot, primscale)
    out, shadow = MVPRaymarch.apply(
        raypos, raydir, stepsize, tminmax, *primtransfin, template, warp, rayterm, torch.is_grad_enabled(),
        {"algo": algo, "usebvh": usebvh, "sortprims": sortprims, "randomorder": randomorder, "maxhitboxes": maxhitboxes,
         "synchitboxes": synchitboxes, "chlast": chlast, "fadescale": fadescale, "fadeexp": fadeexp, "accum": accum,
         "termthresh": termthresh, "griddim": griddim, "blocksize": blocksize, "bwdblocksize": bwdblocksize,
         "with_shadow": with_shadow})
    if with_shadow:
        assert shadow is not None
        if chlast:
            shadow = shadow[..., 0:1] / (shadow[..., 1:] + 1e-5)
        else:
            shadow = shadow[:, :, 0:1] / (shadow[:, :, 1:] + 1e-5)
        return out, shadow
    return out
