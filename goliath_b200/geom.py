"""Mesh front end of the decoders (SURVEY.md section 8f-4): `vert_normals` and `values_to_uv` of ca_code/utils/geom.py:308-346
as sm_90a kernels (csrc/geom_uv.cu) behind the reference's function names, and a `GeometryModule`-shaped holder with
the `vn` / `to_uv` methods `rgca.PrimDecoder` calls on its `geo_fn` (ca_code/models/rgca.py:478-491).  The index /
barycentric images are assets the reference rasterises once at start-up (geom.py:218-247); they are taken as given."""
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
