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
        with torch.cuda.device(v.device):
            _lib.check(_lib.lib().gb_vert_normals_fwd(B, V, F, _lib.ptr(v), _lib.ptr(vi), float(eps), _lib.ptr(acc), _lib.ptr(vn),
                                                      _lib.stream_ptr(v.device)), "vert_normals_fwd")
        ctx.save_for_backward(v, vi, acc)
        ctx.eps = float(eps)
        return vn

    @staticmethod
    def backward(ctx, g_vn):
        v, vi, acc = ctx.saved_tensors
        B, V, _ = v.shape
        g_acc = torch.empty_like(v)
        g_v = torch.zeros_like(v)
        with torch.cuda.device(v.device):
            _lib.check(_lib.lib().gb_vert_normals_bwd(B, V, vi.shape[0], _lib.ptr(v), _lib.ptr(vi), ctx.eps, _lib.ptr(acc),
                                                      _lib.ptr(g_vn.contiguous()), _lib.ptr(g_acc), _lib.ptr(g_v),
                                                      _lib.stream_ptr(v.device)), "vert_normals_bwd")
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
        with torch.cuda.device(values.device):
            _lib.check(_lib.lib().gb_values_to_uv_fwd(B, V, C, U0 * U1, _lib.ptr(values), _lib.ptr(index), _lib.ptr(bary),
                                                      _lib.ptr(out), _lib.stream_ptr(values.device)), "values_to_uv_fwd")
        ctx.save_for_backward(index, bary)
        ctx.shape = (B, V, C, U0 * U1)
        return out

    @staticmethod
    def backward(ctx, g_out):
        index, bary = ctx.saved_tensors
        B, V, C, T = ctx.shape
        g_values = torch.zeros(B, V, C, device=g_out.device, dtype=torch.float32)
        with torch.cuda.device(g_out.device):
            _lib.check(_lib.lib().gb_values_to_uv_bwd(B, V, C, T, _lib.ptr(index), _lib.ptr(bary), _lib.ptr(g_out.contiguous()),
                                                      _lib.ptr(g_values), _lib.stream_ptr(g_out.device)), "values_to_uv_bwd")
        return g_values, None, None


def values_to_uv(values: torch.Tensor, index_img: torch.Tensor, bary_img: torch.Tensor) -> torch.Tensor:
    """geom.py:308-324: values [B,V,C] -> [B,C,U,U] by barycentric interpolation of the three vertices of each texel; zero
    where a texel is not covered (any index == -1)."""
    return _ValuesToUV.apply(values, index_img, bary_img)


class GeometryModule(torch.nn.Module):
    """The part of the reference's GeometryModule (geom.py:186-278) the decoders use: `vn(verts)` and `to_uv(values)`.
    vi [F,3]; index_image / bary_image [U,U,3] are the reference's precomputed assets."""

    def __init__(self, vi: torch.Tensor, index_image: torch.Tensor, bary_image: torch.Tensor):
        super().__init__()
        self.register_buffer("vi", vi.to(torch.int32))
        self.register_buffer("index_image", index_image.to(torch.int32))
        self.register_buffer("bary_image", bary_image.to(torch.float32))

    def vn(self, verts):
        return vert_normals(verts, self.vi)

    def to_uv(self, values):
        return values_to_uv(values, self.index_image, self.bary_image)
