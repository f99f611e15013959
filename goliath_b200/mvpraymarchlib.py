"""Drop-in for the reference's pybind module `mvpraymarchlib` (extensions/mvpraymarch/mvpraymarch.cpp:402-409):
same function names and PURELY POSITIONAL argument lists (28 / 33 arguments, mvpraymarch.py:171-198,266-295), same
in-place output convention.  Kernels: csrc/mvp_raymarch.cu, on the caller's current stream and device.

Arguments the reference kernels accept and ignore (SURVEY.md §0.9: sortboxes, maxhitboxes, synchitboxes, chlast,
accum, termthresh, griddim, rayterm) are accepted and ignored here too; `chlast` must be True, the only layout the
reference kernels implement."""
import torch

from . import _lib

_WS = {}


def _workspace(dev, nbytes):
    key = dev.index
    buf = _WS.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes), 1 << 16), dtype=torch.uint8, device=dev)
        _WS[key] = buf
    return buf


def _chk(t, name, dtype=torch.float32):
    if t is not None:
        _lib.check_input(t, name, dtype)


def compute_morton(primpos, code, algorithm):
    """mvpraymarch.cpp compute_morton -> bvh.cu:42-57.  Only reachable with usebvh=True, a path on which the reference
    traversal reads neither the codes nor the tree (SURVEY.md §0.9); provided for API parity."""
    _chk(primpos, "primpos")
    _chk(code, "code", torch.int32)
    x = (primpos.clamp(0, 1) * 1023).to(torch.int64)

    def expand(v):
        v = (v * 0x00010001) & 0xFF0000FF
        v = (v * 0x00000101) & 0x0F00F00F
        v = (v * 0x00000011) & 0xC30C30C3
        v = (v * 0x00000005) & 0x49249249
        return v

    code.copy_((expand(x[..., 0]) * 4 + expand(x[..., 1]) * 2 + expand(x[..., 2])).to(torch.int32))
    return []


def build_tree(sortedcode, nodechildren, nodeparent):
    raise NotImplementedError(
        "usebvh=True is not a functional path of the reference (its traversal assumes the implicit fixed-order heap, "
        "extensions/mvpraymarch/utils.h:1018); use usebvh='fixedorder'")


def compute_aabb(primpos, primrot, primscale, sortedobjid, nodechildren, nodeparent, nodeaabb, algorithm):
    """mvpraymarch.cpp compute_aabb -> bvh.cu:157-201,249-294.  nodeaabb [N, 2K-1, 2, 3] written in place."""
    for t, n in ((primpos, "primpos"), (primrot, "primrot"), (primscale, "primscale"), (nodeaabb, "nodeaabb")):
        _chk(t, n)
    for t, n in ((sortedobjid, "sortedobjid"), (nodechildren, "nodechildren"), (nodeparent, "nodeparent")):
        _chk(t, n, torch.int32)
    N, K = primpos.size(0), primpos.size(1)
    dev = primpos.device
    L = _lib.kernels()
    ws = _workspace(dev, L.gb_mvp_aabb_workspace_bytes(N, K))
    L.gb_mvp_compute_aabb(N, K, primpos, primrot, primscale, sortedobjid, nodechildren, nodeparent, nodeaabb, ws)
    return []


def _dims(rayposim, primposim, tplateim, warpim, chlast):
    if not chlast:
        raise RuntimeError("only channels-last templates are implemented (as in the reference kernels)")
    N, H, W = rayposim.size(0), rayposim.size(1), rayposim.size(2)
    K = primposim.size(1)
    TD, TH, TW = tplateim.size(2), tplateim.size(3), tplateim.size(4)
    WD, WH, WW = (warpim.size(2), warpim.size(3), warpim.size(4)) if warpim is not None else (0, 0, 0)
    return N, H, W, K, TD, TH, TW, WD, WH, WW


def raymarch_forward(rayposim, raydirim, stepsize, tminmaxim, sortedobjid, nodechildren, nodeaabb, primposim, primrotim,
                     primscaleim, tplateim, warpim, rayrgbaim, raysatim, raytermim, shadow, algorithm, sortboxes,
                     maxhitboxes, synchitboxes, chlast, fadescale, fadeexp, accum, termthresh, griddim, blocksizex,
                     blocksizey):
    """mvpraymarch.cpp:179-283."""
    for t, n in ((rayposim, "rayposim"), (raydirim, "raydirim"), (tminmaxim, "tminmaxim"), (nodeaabb, "nodeaabb"),
                 (primposim, "primposim"), (primrotim, "primrotim"), (primscaleim, "primscaleim"), (tplateim, "tplateim"),
                 (warpim, "warpim"), (rayrgbaim, "rayrgbaim"), (raysatim, "raysatim"), (shadow, "shadow")):
        _chk(t, n)
    if nodeaabb is None or primrotim is None or primscaleim is None:
        raise RuntimeError("usebvh=False / missing primitive transform is not a functional path of the reference")
    N, H, W, K, TD, TH, TW, WD, WH, WW = _dims(rayposim, primposim, tplateim, warpim, chlast)
    algo = int(algorithm)
    _lib.kernels().gb_mvp_raymarch_fwd(
        N, H, W, K, rayposim, raydirim, float(stepsize), tminmaxim, nodeaabb, primposim, primrotim, primscaleim, TD,
        TH, TW, tplateim, WD, WH, WW, warpim if algo == 1 else None, rayrgbaim, raysatim, shadow, algo,
        float(fadescale), float(fadeexp), int(blocksizex), int(blocksizey))
    return []


def raymarch_backward(rayposim, raydirim, stepsize, tminmaxim, sortedobjid, nodechildren, nodeaabb, primposim,
                      grad_primposim, primrotim, grad_primrotim, primscaleim, grad_primscaleim, tplateim, grad_tplateim,
                      warpim, grad_warpim, rayrgbaim, grad_rayrgba, raysatim, raytermim, algorithm, sortboxes, maxhitboxes,
                      synchitboxes, chlast, fadescale, fadeexp, accum, termthresh, griddim, blocksizex, blocksizey):
    """mvpraymarch.cpp:285-399."""
    for t, n in ((rayposim, "rayposim"), (raydirim, "raydirim"), (tminmaxim, "tminmaxim"), (nodeaabb, "nodeaabb"),
                 (primposim, "primposim"), (grad_primposim, "grad_primposim"), (primrotim, "primrotim"),
                 (grad_primrotim, "grad_primrotim"), (primscaleim, "primscaleim"), (grad_primscaleim, "grad_primscaleim"),
                 (tplateim, "tplateim"), (grad_tplateim, "grad_tplateim"), (warpim, "warpim"), (grad_warpim, "grad_warpim"),
                 (rayrgbaim, "rayrgbaim"), (grad_rayrgba, "grad_rayrgba"), (raysatim, "raysatim")):
        _chk(t, n)
    N, H, W, K, TD, TH, TW, WD, WH, WW = _dims(rayposim, primposim, tplateim, warpim, chlast)
    algo = int(algorithm)
    _lib.kernels().gb_mvp_raymarch_bwd(
        N, H, W, K, rayposim, raydirim, float(stepsize), tminmaxim, nodeaabb, primposim, primrotim, primscaleim, TD,
        TH, TW, tplateim, WD, WH, WW, warpim if algo == 1 else None, raysatim, grad_rayrgba, grad_primposim,
        grad_primrotim, grad_primscaleim, grad_tplateim, grad_warpim if algo == 1 else None, algo, float(fadescale),
        float(fadeexp), int(blocksizex), int(blocksizey))
    return []
