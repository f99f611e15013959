"""Mesh front end of the decoders (SURVEY.md section 8f-4): `vert_normals` and `values_to_uv` of ca_code/utils/geom.py:308-346
as sm_90a kernels (csrc/geom_uv.cu) behind the reference's function names, and a `GeometryModule`-shaped holder with
the `vn` / `to_uv` methods `rgca.PrimDecoder` calls on its `geo_fn` (ca_code/models/rgca.py:478-491).  The index /
barycentric images the reference rasterises once at start-up (geom.py:31-265) are built from the UV layout by
csrc/uv_layout.cu: `make_uv_face_index`, `make_uv_vert_index`, `make_uv_barys`, `index_image_impaint`,
`GeometryModule.from_topology` / `render_index_images`, and `uv_assets` for the frames' constructors."""
import functools
import math

import numpy as np
import torch
from torch.autograd import Function

from . import _lib

EPS = 1.0e-5  # geom.py:327,336


class _VertNormals(Function):
    @staticmethod
    def forward(ctx, v, vi, eps):
        v = v.contiguous()
        _lib.check_input(v, "verts")
        vi = vi.to(torch.int32).contiguous()
        _lib.check_input(vi, "vi", torch.int32)
        B, V, _ = v.shape
        F = vi.shape[0]
        acc = torch.zeros_like(v)
        vn = torch.empty_like(v)
        _lib.kernels().gb_vert_normals_fwd(B, V, F, v, vi, float(eps), acc, vn)
        ctx.save_for_backward(v, vi, acc)
        ctx.eps = float(eps)
        return vn

    @staticmethod
    def backward(ctx, g_vn):
        v, vi, acc = ctx.saved_tensors
        B, V, _ = v.shape
        g_acc = torch.empty_like(v)
        g_v = torch.zeros_like(v)
        _lib.kernels().gb_vert_normals_bwd(B, V, vi.shape[0], v, vi, ctx.eps, acc, g_vn.contiguous(), g_acc, g_v)
        return g_v, None, None


def vert_normals(v: torch.Tensor, vi: torch.Tensor, eps: float = EPS) -> torch.Tensor:
    """geom.py:336-346: v [B,V,3], vi [F,3] -> unit vertex normals [B,V,3] (area-unweighted mean of the unit face normals)."""
    return _VertNormals.apply(v, vi, eps)


class _ValuesToUV(Function):
    @staticmethod
    def forward(ctx, values, index_img, bary_img):
        values = values.contiguous()
        _lib.check_input(values, "values")
        index = index_img.to(torch.int32).contiguous()
        bary = bary_img.to(torch.float32).contiguous()
        _lib.check_input(index, "index_img", torch.int32)
        _lib.check_input(bary, "bary_img")
        B, V, C = values.shape
        U0, U1 = index.shape[0], index.shape[1]
        if index.shape[-1] != 3 or bary.shape != index.shape:
            raise RuntimeError("values_to_uv: index_img / bary_img must be [U,U,3]")
        out = torch.empty(B, C, U0, U1, device=values.device, dtype=torch.float32)
        _lib.kernels().gb_values_to_uv_fwd(B, V, C, U0 * U1, values, index, bary, out)
        ctx.save_for_backward(index, bary)
        ctx.shape = (B, V, C, U0 * U1)
        return out

    @staticmethod
    def backward(ctx, g_out):
        index, bary = ctx.saved_tensors
        B, V, C, T = ctx.shape
        g_values = torch.zeros(B, V, C, device=g_out.device, dtype=torch.float32)
        _lib.kernels().gb_values_to_uv_bwd(B, V, C, T, index, bary, g_out.contiguous(), g_values)
        return g_values, None, None


def values_to_uv(values: torch.Tensor, index_img: torch.Tensor, bary_img: torch.Tensor) -> torch.Tensor:
    """geom.py:308-324: values [B,V,C] -> [B,C,U,U] by barycentric interpolation of the three vertices of each texel; zero
    where a texel is not covered (any index == -1)."""
    return _ValuesToUV.apply(values, index_img, bary_img)


def sample_uv_table(uv_coords: torch.Tensor, v2uv, H: int, W: int):
    """the gather table of sample_uv (geom.py:281-304): bilinear at vt with align_corners=True and zeros padding, then
    the mean over the v2uv columns (a padded row repeats its first entry, which the mean then weights more, as in the
    reference).  One row per vertex (per UV coordinate without v2uv), 4 n_max entries."""
    from .seams import GatherTable, _corners

    vt = uv_coords.to(torch.float64).reshape(-1, 2)
    cols, ws = _corners(vt[:, 0] * (W - 1), vt[:, 1] * (H - 1), H, W)
    if v2uv is None:
        return GatherTable(cols, ws, H * W)
    idx = v2uv.to(torch.int64)
    n_max = idx.shape[1]
    return GatherTable(cols[idx].reshape(idx.shape[0], 4 * n_max), (ws[idx] / n_max).reshape(idx.shape[0], 4 * n_max),
                       H * W)


def sample_uv(values_uv: torch.Tensor, uv_coords: torch.Tensor, v2uv=None) -> torch.Tensor:
    """geom.py:281-304 (mode bilinear, align_corners=True, flip_uvs=False): values_uv [B,C,H,W], uv_coords [N,2] ->
    [B,N,C], or [B,V,C] averaged over the columns of v2uv [V,n_max].  Builds its table per call (no host sync); use
    GeometryModule.from_uv to build it once."""
    from .seams import gather

    _lib.check_input(values_uv, "values_uv")
    return gather(values_uv, sample_uv_table(uv_coords, v2uv, values_uv.shape[2], values_uv.shape[3]), rows_last=True)


class GeometryModule(torch.nn.Module):
    """The part of the reference's GeometryModule (geom.py:186-278) the decoders use: `vn(verts)`, `to_uv(values)` and,
    given vt [N_uv,2] (and optionally v2uv [V,n_max]), `from_uv(values_uv)`.  vi [F,3]; index_image / bary_image
    [U,U,3] are the reference's precomputed assets.  vt, v2uv, vti [F,3], face_index_image [U,U] and valid_mask
    [U,U,1] are each registered only when given, so a full module holds the reference's eight buffers (seven for the
    head, which has no v2uv), a checkpoint's `geo_fn.*` keys load strictly, and the smaller holders keep their keys."""

    def __init__(self, vi: torch.Tensor, index_image: torch.Tensor, bary_image: torch.Tensor, vt=None, v2uv=None,
                 vti=None, face_index_image=None, valid_mask=None):
        super().__init__()
        self.register_buffer("vi", torch.as_tensor(vi).to(torch.int32))
        self.register_buffer("index_image", torch.as_tensor(index_image).to(torch.int32))
        self.register_buffer("bary_image", torch.as_tensor(bary_image).to(torch.float32))
        if vt is not None:
            self.register_buffer("vt", torch.as_tensor(vt).to(torch.float32))
        if v2uv is not None:
            self.register_buffer("v2uv", torch.as_tensor(v2uv).to(torch.int32))
        if vti is not None:
            self.register_buffer("vti", torch.as_tensor(vti).to(torch.int32))
        if face_index_image is not None:
            self.register_buffer("face_index_image", torch.as_tensor(face_index_image).to(torch.int32))
        if valid_mask is not None:
            self.register_buffer("valid_mask", torch.as_tensor(valid_mask).to(torch.bool))
        self._uv_table, self._uv_key = None, None

    @classmethod
    def from_topology(cls, vi, vt, vti, v2uv, uv_size, flip_uv=False, impaint=False, impaint_threshold=100.0):
        """the reference's GeometryModule.__init__ (geom.py:197-249), same argument order: the index, barycentric and
        face images of the UV layout, `valid_mask` taken before the impaint, and with `impaint` all three images
        impainted from one source table.  The buffers are on vi's device, like the topology."""
        U = _uv_size(uv_size)
        face, index, bary, valid = _index_images(vt, vti, vi, U, flip_uv, face=True, vert=True, bary=True, valid=True)
        if impaint:
            src = _impaint_sources(index, impaint_threshold)
            index, bary, face = _impaint_gather(src, index, bary, face)
        dev = torch.as_tensor(vi).device
        return cls(vi, index.to(dev), bary.to(dev), vt=vt, v2uv=v2uv, vti=vti, face_index_image=face.to(dev),
                   valid_mask=valid[..., None].to(dev))

    @torch.no_grad()
    def render_index_images(self, uv_size, flip_uv=False, impaint=False):
        """geom.py:251-265: (index [U,U,3] int64, face [U,U] int64, bary [U,U,3] fp32) on vt's device.  With
        `impaint` only the index and barycentric images are impainted (threshold 100): the face image is returned
        as rasterised, which `hand_mvp.init_primitives` relies on."""
        U = _uv_size(uv_size)
        face, index, bary, _ = _index_images(self.vt, self.vti, self.vi, U, flip_uv, face=True, vert=True, bary=True)
        if impaint:
            index, bary = _impaint_gather(_impaint_sources(index, 100.0), index, bary)
        dev = self.vt.device
        return index.to(dev), face.to(dev), bary.to(dev)

    def from_uv(self, values_uv):
        """geom.py:273-275: sample_uv(values_uv, vt, v2uv) with the gather table built once per (buffers, map size);
        one row per UV coordinate when the module has no v2uv"""
        from .seams import gather

        _lib.check_input(values_uv, "values_uv")
        H, W = values_uv.shape[2], values_uv.shape[3]
        v2uv = getattr(self, "v2uv", None)
        key = (self.vt.device, self.vt.data_ptr(), self.vt._version, None if v2uv is None else v2uv.data_ptr(),
               None if v2uv is None else v2uv._version, H, W)
        if self._uv_key != key:
            self._uv_table, self._uv_key = sample_uv_table(self.vt, v2uv, H, W), key
        return gather(values_uv, self._uv_table, rows_last=True)

    def vn(self, verts):
        return vert_normals(verts, self.vi)

    def to_uv(self, values):
        return values_to_uv(values, self.index_image, self.bary_image)


def depth_discontuity_mask(depth: torch.Tensor, threshold: float = 40.0, kscale: float = 4.0,
                           pool_ksize: int = 3) -> torch.Tensor:
    """geom.py:768-794 (the reference's name) on one kernel (csrc/body_frame.cu): depth [B,1,H,W] -> torch.bool
    [B,1,H,W], true where a pixel within the 3x3 neighbourhood inside the image has a Sobel gradient norm (zero
    padding) above `threshold`.  `kscale` is unused, as in the reference; only pool_ksize 3 is implemented.  No
    gradient (the reference runs it under no_grad)."""
    if pool_ksize != 3:
        raise ValueError("depth_discontuity_mask: only pool_ksize = 3 is implemented (got %d)" % pool_ksize)
    depth = depth.detach().contiguous()
    _lib.check_input(depth, "depth")
    if depth.dim() != 4 or depth.shape[1] != 1:
        raise RuntimeError("depth_discontuity_mask: depth must be [B,1,H,W] (got %s)" % (tuple(depth.shape),))
    B, _, H, W = depth.shape
    mask = torch.empty(B, 1, H, W, device=depth.device, dtype=torch.bool)
    _lib.kernels().gb_depth_disc_mask(B, H, W, depth, float(threshold), mask)
    return mask


# ------------------------------------------------------------------------------------ UV layout images (uv_layout.cu)
def _uv_size(uv_shape) -> int:
    """an int or a square (H, W): pytorch3d's non-square NDC is a different convention, so it is refused"""
    if isinstance(uv_shape, (int, np.integer)):
        return int(uv_shape)
    h, w = (int(x) for x in uv_shape)
    if h != w:
        raise ValueError("uv_shape must be square (got %d x %d)" % (h, w))
    return h


def _device():
    return torch.device("cuda", torch.cuda.current_device())


def _index_images(vt, vti, vi, U, flip_uv, face=True, vert=False, bary=False, valid=False):
    """(face [U,U] int64, vert_index [U,U,3] int64, bary [U,U,3] fp32, valid [U,U] bool) on the current CUDA device,
    None for what is not asked for.  vt is rounded to fp32 first (a float64 vt included)."""
    dev = _device()
    vt = torch.as_tensor(vt).detach().to(dev, torch.float32).contiguous()
    vti = torch.as_tensor(vti).detach().to(dev, torch.int32).contiguous()
    if vt.dim() != 2 or vt.shape[1] != 2 or vti.dim() != 2 or vti.shape[1] != 3:
        raise ValueError("vt must be [N,2] and vti [F,3] (got %s, %s)" % (tuple(vt.shape), tuple(vti.shape)))
    F = vti.shape[0]
    vi = torch.as_tensor(vi).detach().to(dev, torch.int32).contiguous() if vert else None
    empty = lambda *shape, dtype: torch.empty(*shape, device=dev, dtype=dtype)
    out_face = empty(U, U, dtype=torch.int64) if face else None
    out_vert = empty(U, U, 3, dtype=torch.int64) if vert else None
    out_bary = empty(U, U, 3, dtype=torch.float32) if bary else None
    out_valid = empty(U, U, dtype=torch.bool) if valid else None
    grid = (torch.linspace(0.5, U - 0.5, U) / U).to(dev) if bary else None  # geom.py:133-136, evaluated by torch
    ws = empty(_lib.lib().gb_uv_raster_workspace_bytes(F, U), dtype=torch.uint8)
    _lib.kernels().gb_uv_index_images(F, U, int(bool(flip_uv)), vt, vti, vi, grid, ws, out_face, out_vert, out_bary,
                                      out_valid)
    return out_face, out_vert, out_bary, out_valid


def _max_d2(threshold, H, W) -> int:
    """the largest squared texel distance d2 with sqrt(d2) < threshold in double (the KDTree distance test), at most
    the image's diagonal; -1 when there is none"""
    cap = (H - 1) ** 2 + (W - 1) ** 2
    t = float(threshold)
    if not t > 0:
        return -1
    n = cap if t * t > cap + 1 else int(t * t)
    while n >= 0 and not math.sqrt(n) < t:
        n -= 1
    while n < cap and math.sqrt(n + 1) < t:
        n += 1
    return n


@functools.lru_cache(maxsize=16)
def _offset_table(d2max, H, W, device):
    """the offsets (di, dj) with di^2 + dj^2 <= d2max inside an H x W image, sorted by (di^2 + dj^2, di, dj), and the
    first offset of each squared length (d2max + 2 entries): for one squared distance the first in-image valid
    candidate is the equidistant valid texel with the smallest row-major index"""
    r = math.isqrt(d2max)
    di, dj = np.meshgrid(np.arange(-min(r, H - 1), min(r, H - 1) + 1), np.arange(-min(r, W - 1), min(r, W - 1) + 1),
                         indexing="ij")
    di, dj = di.ravel().astype(np.int64), dj.ravel().astype(np.int64)
    d2 = di * di + dj * dj
    keep = d2 <= d2max
    di, dj, d2 = di[keep], dj[keep], d2[keep]
    order = np.lexsort((dj, di, d2))
    offsets = np.stack([di[order], dj[order]], axis=1).astype(np.int32)
    start = np.concatenate([[0], np.cumsum(np.bincount(d2, minlength=d2max + 1))]).astype(np.int32)
    return torch.from_numpy(offsets).to(device), torch.from_numpy(start).to(device)


def _impaint_sources(index_image, threshold, return_d2=False):
    """the impaint's source table [H,W] int32 on the current CUDA device: the row-major index of the nearest valid
    texel (smallest row-major index among equidistant ones) for every invalid texel at a distance below `threshold`,
    -1 elsewhere.  Raises ValueError when no texel is valid."""
    index = torch.as_tensor(index_image).detach()
    if index.dim() == 2:
        index = index[..., None]
    elif index.dim() != 3:
        raise ValueError("`index_image` should be a [H,W] or [H,W,C] image")
    if not bool((index != -1).any()):  # one host read, on the image's own device
        raise ValueError("index_image_impaint: the image has no valid texel")
    dev = _device()
    index = index.to(dev, torch.int64).contiguous()
    H, W, C = index.shape
    d2max = _max_d2(threshold, H, W)
    offsets, start = _offset_table(d2max, H, W, dev) if d2max >= 0 else (None, None)
    ws = torch.empty(_lib.lib().gb_uv_impaint_workspace_bytes(H, W), device=dev, dtype=torch.uint8)
    d2 = torch.empty(H, W, device=dev, dtype=torch.int32)
    src = torch.empty(H, W, device=dev, dtype=torch.int32)
    _lib.kernels().gb_uv_impaint_sources(H, W, C, index, d2max, offsets, start, ws, d2, src)
    return (src, d2) if return_d2 else src


def _impaint_gather(src, *images):
    """each image [H,W,...] with its texels moved along the source table, as new tensors on src's device"""
    dev = src.device
    ins, outs = [], []
    for im in images:
        im = torch.as_tensor(im).detach().to(dev).contiguous()
        if (im[0, 0].numel() * im.element_size()) % 4:
            raise ValueError("impaint: a texel must be a whole number of 32-bit words")
        ins.append(im)
        outs.append(torch.empty_like(im))
    args = []
    for k in range(3):
        if k < len(ins):
            args += [ins[k], outs[k], ins[k][0, 0].numel() * ins[k].element_size() // 4]
        else:
            args += [None, None, 0]
    _lib.kernels().gb_uv_impaint_gather(src.numel(), src, *args)
    return tuple(outs)


@torch.no_grad()
def make_uv_face_index(vt, vti, uv_shape, flip_uv=True, device=None):
    """geom.py:31-66: the face under each texel [U,U] int64, -1 where none (this project's rasteriser conventions,
    DESIGN.md R12), on the current CUDA device.  vt is rounded to fp32."""
    if device is not None and torch.device(device).type != "cuda":
        raise ValueError("make_uv_face_index: device must be a CUDA device")
    return _index_images(vt, vti, None, _uv_size(uv_shape), flip_uv)[0]


@torch.no_grad()
def make_uv_vert_index(vt, vi, vti, uv_shape, flip_uv=True):
    """geom.py:69-83: vi[face] [U,U,3] int64, -1 in all three channels where no face covers the texel, on vi's
    device"""
    dev = torch.as_tensor(vi).device
    return _index_images(vt, vti, vi, _uv_size(uv_shape), flip_uv, face=False, vert=True)[1].to(dev)


@torch.no_grad()
def make_uv_barys(vt, vti, uv_shape, flip_uv=True):
    """geom.py:109-142: (face [U,U] int64, bary [U,U,3]) on vt's device; bary_coords of the texel centre in its UV
    triangle, zero where no face covers it.  The barycentrics are evaluated in fp32 (a float64 vt is rounded to fp32
    first) and returned in vt's float dtype."""
    vt_t = torch.as_tensor(vt)
    face, _, bary, _ = _index_images(vt_t, vti, None, _uv_size(uv_shape), flip_uv, bary=True)
    dtype = vt_t.dtype if vt_t.is_floating_point() else torch.float32
    return face.to(vt_t.device), bary.to(vt_t.device, dtype)


@torch.no_grad()
def index_image_impaint(index_image, bary_image=None, distance_threshold=100.0):
    """geom.py:145-194: every invalid texel (all channels -1 for [H,W,C], -1 for [H,W]) whose Euclidean distance to
    the nearest valid texel is below `distance_threshold` takes that texel's values; among equidistant valid texels
    the one with the smallest row-major index.  Returns new image(s) on index_image's device; ValueError when no
    texel is valid."""
    index_image = torch.as_tensor(index_image)
    src = _impaint_sources(index_image, distance_threshold)
    if bary_image is None:
        return _impaint_gather(src, index_image)[0].to(index_image.device)
    bary_image = torch.as_tensor(bary_image)
    idx, bary = _impaint_gather(src, index_image, bary_image)
    return idx.to(index_image.device), bary.to(bary_image.device)


# the flags each reference model passes to its GeometryModule (rgca.py:71-79, mesh_vae.py:91-98,
# mesh_vae_drivable.py:92-99, hand_mvp.py:102-110; hand_teacher_mvp's AutoEncoder is hand_mvp's): flip_uv, impaint,
# v2uv, and whether the frame also reads render_index_images(uv_size, impaint=True) (hand_mvp.init_primitives)
UV_ASSET_FLAGS = {
    "rgca": (True, False, False, False),
    "mesh_vae": (False, True, True, False),
    "mesh_vae_drivable": (False, True, True, False),
    "hand_mvp": (False, False, True, True),
    "hand_teacher_mvp": (False, False, True, True),
}


def uv_assets(topology, model, uv_size=1024):
    """the UV images a frame's constructor reads from its assets, built from the topology (vi, vt, vti and v2uv, as
    attributes or dict keys) with the flags the reference model passes: index_image, bary_image, face_index_image
    and valid_mask, plus face_index_image_impaint and bary_image_impaint for the hand frames.  CPU tensors, so
    `assets.update(uv_assets(assets.topology, "hand_mvp"))` and the frame builds as from the reference's assets."""
    if model not in UV_ASSET_FLAGS:
        raise ValueError("uv_assets: unknown model %r (one of %s)" % (model, ", ".join(sorted(UV_ASSET_FLAGS))))
    flip_uv, impaint, with_v2uv, hand = UV_ASSET_FLAGS[model]
    get = (lambda k: topology.get(k)) if isinstance(topology, dict) else (lambda k: getattr(topology, k, None))
    geo = GeometryModule.from_topology(get("vi"), get("vt"), get("vti"), get("v2uv") if with_v2uv else None, uv_size,
                                       flip_uv=flip_uv, impaint=impaint)
    cpu = lambda t: t.detach().cpu()
    out = {"index_image": cpu(geo.index_image).long(), "bary_image": cpu(geo.bary_image),
           "face_index_image": cpu(geo.face_index_image).long(), "valid_mask": cpu(geo.valid_mask)}
    if hand:
        _, face, bary = geo.render_index_images(uv_size, impaint=True)
        out["face_index_image_impaint"], out["bary_image_impaint"] = cpu(face), cpu(bary)
    return out
