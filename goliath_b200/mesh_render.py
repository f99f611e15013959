"""Body avatar render on the GPU: the reference's drtk `RenderLayer` (ca_code/utils/render_drtk.py:14-82) on
csrc/mesh_raster.cu.

`RenderLayer.forward` projects the posed mesh with `transform` (torch ops, so K and Rt keep their gradients),
rasterises it, interpolates the UVs, samples the texture (grid_sample's bilinear, align_corners=False, zero padding)
and multiplies by the coverage mask, in one autograd node over (v_pix, tex).  The backward includes the project's
edge-gradient estimator when `edge_grad` is set (DESIGN.md R9'') and gives bitwise-repeatable gradients.  drtk is
outside the reference tree, so its rasteriser conventions are restated, not pinned (PARITY UNPINNED).

Differences from the reference (INTEGRATION.md): only `render` carries a gradient (`depth_img`, `bary_img` and
`vt_img` are returned without one), and `flip_uvs=True` flips a copy of `vt` instead of the caller's tensor."""
from typing import List

import torch
import torch.nn as nn
from torch.autograd import Function

from . import _lib


def transform(v: torch.Tensor, K: torch.Tensor, Rt: torch.Tensor) -> torch.Tensor:
    """v [B,V,3] world -> v_pix [B,V,3]: v_cam = R v + t, then (K v_cam) x and y divided by z, z kept."""
    v_cam = torch.einsum("bij,bvj->bvi", Rt[:, :3, :3], v) + Rt[:, None, :3, 3]
    z = v_cam[..., 2:3]
    p = torch.einsum("bij,bvj->bvi", K[:, :3, :3], v_cam)
    return torch.cat([p[..., :2] / z, z], dim=-1)


class _Incidence:
    """per-vertex list of (face, corner) entries 3 f + k, ascending within a vertex, as CSR int32 device arrays"""

    def __init__(self, vi: torch.Tensor):
        flat = vi.reshape(-1).to(torch.int64)
        self.n_verts = int(flat.max().item()) + 1 if flat.numel() else 0
        order = torch.sort(flat, stable=True).indices
        self.inc = order.to(torch.int32).contiguous()
        counts = torch.zeros(self.n_verts + 1, device=vi.device, dtype=torch.int64).index_add_(
            0, flat + 1, torch.ones_like(flat))
        self.ptr = torch.cumsum(counts, 0).to(torch.int32).contiguous()


class _MeshRender(Function):
    @staticmethod
    def forward(ctx, v_pix, tex, layer, edge_grad):
        v_pix, tex = v_pix.contiguous(), tex.contiguous()
        _lib.check_input(v_pix, "v_pix")
        _lib.check_input(tex, "tex")
        vi, vti, vt, inc = layer._device_tables(v_pix.device)
        B, V = v_pix.shape[:2]
        if v_pix.shape[2] != 3 or tex.dim() != 4 or tex.shape[0] != B:
            raise RuntimeError("RenderLayer: v_pix must be [B,V,3] and tex [B,C,Ht,Wt] (got %s, %s)"
                               % (tuple(v_pix.shape), tuple(tex.shape)))
        if inc.n_verts > V:
            raise RuntimeError("RenderLayer: vi indexes %d vertices, verts has %d" % (inc.n_verts, V))
        F = vi.shape[0]
        C, Ht, Wt = tex.shape[1:]
        H, W = layer.h, layer.w
        dev = v_pix.device
        L = _lib.kernels()
        index_img = torch.empty(B, H, W, device=dev, dtype=torch.int32)
        depth = torch.empty(B, H, W, device=dev)
        bary = torch.empty(B, 3, H, W, device=dev)
        vt_img = torch.empty(B, 2, H, W, device=dev)
        mask = torch.empty(B, 1, H, W, device=dev)
        render = torch.empty(B, C, H, W, device=dev)
        ws = torch.empty(L.gb_mesh_raster_workspace_bytes(B, F, H, W), device=dev, dtype=torch.uint8)
        L.gb_mesh_raster(B, V, F, H, W, v_pix, vi, index_img, ws)
        L.gb_mesh_render_fwd(B, V, F, H, W, C, Ht, Wt, v_pix, vi, vti, vt, tex, index_img, depth, bary, vt_img,
                             mask, render)
        ctx.mark_non_differentiable(depth, bary, vt_img, index_img, mask)
        ctx.save_for_backward(v_pix, tex, index_img, vt_img, render)
        ctx.tables, ctx.edge_grad = (vi, vti, vt, inc), bool(edge_grad)
        return render, depth, bary, vt_img, index_img, mask

    @staticmethod
    def backward(ctx, g_render, *unused):
        v_pix, tex, index_img, vt_img, render = ctx.saved_tensors
        vi, vti, vt, inc = ctx.tables
        B, V = v_pix.shape[:2]
        F = vi.shape[0]
        C, Ht, Wt = tex.shape[1:]
        H, W = index_img.shape[1:]
        dev = v_pix.device
        g_render = g_render.contiguous()
        g_v = torch.empty_like(v_pix)
        g_tex = torch.empty_like(tex)
        L = _lib.kernels()
        ws = torch.empty(L.gb_mesh_render_bwd_workspace_bytes(B, F, H, W, Ht, Wt), device=dev, dtype=torch.uint8)
        inc_ptr = inc.ptr
        if inc_ptr.numel() < V + 1:  # vertices no face uses: empty lists
            inc_ptr = torch.cat([inc_ptr, inc_ptr[-1:].expand(V + 1 - inc_ptr.numel())]).contiguous()
        L.gb_mesh_render_bwd(
            B, V, F, H, W, C, Ht, Wt, v_pix, vi, vti, vt, tex, index_img, vt_img, render, g_render,
            int(ctx.edge_grad), inc_ptr, inc.inc, g_v, g_tex, ws)
        return g_v, g_tex, None, None


class RenderLayer(nn.Module):
    """render_drtk.RenderLayer with its buffers: vi, vt and vti non-persistent, image_size [h, w] int32 persistent
    (a mesh_vae checkpoint's `renderer.image_size` loads strictly)."""

    def __init__(self, h, w, vi, vt, vti, flip_uvs=False):
        super().__init__()
        self.h = h
        self.w = w
        vt = torch.as_tensor(vt)
        if flip_uvs:  # the reference writes into the caller's tensor; this flips a copy
            vt = vt.clone()
            vt[:, 1] = 1 - vt[:, 1]
        self.register_buffer("vi", torch.as_tensor(vi), persistent=False)
        self.register_buffer("vt", vt, persistent=False)
        self.register_buffer("vti", torch.as_tensor(vti), persistent=False)
        self.flip_uvs = flip_uvs
        self.register_buffer("image_size", torch.as_tensor([h, w], dtype=torch.int32))
        self._tables, self._key = None, None

    def _device_tables(self, device):
        """int32 / fp32 contiguous copies of vi, vti, vt on `device` and the vertex incidence lists, rebuilt when a
        buffer is replaced or modified"""
        key = (device,) + tuple((b.device, b.data_ptr(), b._version, tuple(b.shape))
                                for b in (self.vi, self.vti, self.vt))
        if self._key != key:
            vi = self.vi.to(device, torch.int32).contiguous()
            vti = self.vti.to(device, torch.int32).contiguous()
            vt = self.vt.to(device, torch.float32).contiguous()
            if vi.dim() != 2 or vi.shape[1] != 3 or vti.shape != vi.shape or vt.dim() != 2 or vt.shape[1] != 2:
                raise RuntimeError("RenderLayer: vi and vti must be [F,3] and vt [Vt,2]")
            if vi.numel() and int(vi.min().item()) < 0:
                raise RuntimeError("RenderLayer: negative vertex index in vi")
            if vti.numel() and (int(vti.min().item()) < 0 or int(vti.max().item()) >= vt.shape[0]):
                raise RuntimeError("RenderLayer: vti indexes outside vt")
            self._tables = (vi, vti, vt, _Incidence(vi))
            self._key = key
        return self._tables

    def forward(self, verts: torch.Tensor, tex: torch.Tensor, K: torch.Tensor, Rt: torch.Tensor,
                background: torch.Tensor = None, output_filters: List[str] = None, edge_grad: bool = True):
        if output_filters is not None:
            raise ValueError("RenderLayer: output_filters is not supported (the reference asserts it is None)")
        if background is not None:
            raise ValueError("RenderLayer: background is not supported (the reference asserts it is None)")
        for t, n in ((verts, "verts"), (tex, "tex"), (K, "K"), (Rt, "Rt")):
            if not t.is_cuda:
                raise RuntimeError("RenderLayer runs on CUDA only: %s is on %s" % (n, t.device))
        v_pix = transform(verts, K, Rt)
        render, depth, bary, vt_img, index_img, mask = _MeshRender.apply(v_pix.float(), tex.float(), self, edge_grad)
        return {
            "render": render,
            "depth_img": depth,
            "v_pix": v_pix,
            "vt_img": vt_img,
            "index_img": index_img,
            "bary_img": bary,
            "mask": mask,
        }
