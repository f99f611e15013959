"""Seam sampler of the body decoder (ca_code/utils/seams.py:14-41) and the sparse gather it shares with
`geom.sample_uv` / `GeometryModule.from_uv`.

Each of these maps is linear in the texture and fixed by constant buffers, so it is stored once as a table of rows
(output texel or vertex -> a few (input texel, coefficient) entries) together with its transpose, and both directions
run as the same fixed-order gather (`gb_sparse_rows_apply`, csrc/upconv_wnub.cu): no atomics, so two backward calls
give bitwise-equal gradients.  The tables are built on the buffers' device with fixed-size torch ops (a stable sort and
a count), once per set of buffers; `SeamSampler` rebuilds them when `load_state_dict` (or anything else) replaces or
modifies its buffers."""
import torch
import torch.nn as nn
from torch.autograd import Function

from . import _lib


class GatherTable:
    """rows [n_rows] x width entries (col into n_cols, coef) and the transposed table, as int32 / fp32 device arrays"""

    def __init__(self, col: torch.Tensor, coef: torch.Tensor, n_cols: int):
        n_rows, width = col.shape
        dev = col.device
        self.n_rows, self.n_cols = n_rows, n_cols
        col = col.reshape(-1).to(torch.int64)
        self.ptr = (torch.arange(n_rows + 1, device=dev, dtype=torch.int64) * width).to(torch.int32)
        self.col = col.to(torch.int32).contiguous()
        self.coef = coef.reshape(-1).to(torch.float32).contiguous()
        # transpose: entries grouped by input index, in row order within a group (stable sort)
        order = torch.sort(col, stable=True).indices
        self.t_col = torch.div(order, width, rounding_mode="floor").to(torch.int32).contiguous()
        self.t_coef = self.coef[order].contiguous()
        counts = torch.zeros(n_cols + 1, device=dev, dtype=torch.int64).index_add_(
            0, col + 1, torch.ones_like(col))
        self.t_ptr = torch.cumsum(counts, 0).to(torch.int32).contiguous()


def _apply(B, C, n_rows, ptr, col, coef, src, in_strides, out, out_strides):
    _lib.kernels().gb_sparse_rows_apply(B, C, n_rows, ptr, col, coef, src, *in_strides, out, *out_strides)


class _Gather(Function):
    """map [B,C,H,W] -> map [B,C,H,W] (rows = texels) or, with rows_last, [B,n_rows,C] (rows = vertices)"""

    @staticmethod
    def forward(ctx, x, table, rows_last):
        x = x.contiguous()
        _lib.check_input(x, "texture")
        B, C, H, W = x.shape
        if H * W != table.n_cols:
            raise RuntimeError("gather table was built for %d texels, the map has %dx%d" % (table.n_cols, H, W))
        N = table.n_rows
        if rows_last:
            out = torch.empty(B, N, C, device=x.device)
            ost = (N * C, 1, C)
        else:
            out = torch.empty(B, C, H, W, device=x.device)
            ost = (C * N, N, 1)
        _apply(B, C, N, table.ptr, table.col, table.coef, x, (C * H * W, H * W, 1), out, ost)
        ctx.table, ctx.rows_last, ctx.shape = table, rows_last, (B, C, H, W)
        return out

    @staticmethod
    def backward(ctx, g):
        t, (B, C, H, W) = ctx.table, ctx.shape
        g = g.contiguous()
        N = t.n_rows
        gst = (N * C, 1, C) if ctx.rows_last else (C * N, N, 1)
        gx = torch.empty(B, C, H, W, device=g.device)
        _apply(B, C, H * W, t.t_ptr, t.t_col, t.t_coef, g, gst, gx, (C * H * W, H * W, 1))
        return gx, None, None


def gather(x: torch.Tensor, table: GatherTable, rows_last: bool = False) -> torch.Tensor:
    return _Gather.apply(x, table, rows_last)


def _corners(ix, iy, H, W):
    """the four bilinear corners of (ix, iy) in texel units: flat indices [N,4] (clamped) and weights [N,4] (zero for a
    corner outside the map)"""
    x0, y0 = torch.floor(ix), torch.floor(iy)
    tx, ty = ix - x0, iy - y0
    cols, ws = [], []
    for dy, wy in ((0, 1 - ty), (1, ty)):
        for dx, wx in ((0, 1 - tx), (1, tx)):
            xx, yy = x0 + dx, y0 + dy
            inside = (xx >= 0) & (xx <= W - 1) & (yy >= 0) & (yy <= H - 1)
            cols.append((yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).to(torch.int64))
            ws.append(torch.where(inside, wy * wx, torch.zeros_like(wx)))
    return torch.stack(cols, 1), torch.stack(ws, 1)


def resample_entries(uvs: torch.Tensor, weights: torch.Tensor):
    """resample_tex (seams.py:21-25): (1 - w) tex + w grid_sample(tex, 2 (uv - 0.5)), align_corners=False, border
    padding.  Returns col / coef [H*W, 5]: the texel itself, then the four corners."""
    H, W = uvs.shape[0], uvs.shape[1]
    uv = uvs.to(torch.float64).reshape(-1, 2)
    w = weights.to(torch.float64).reshape(-1)
    if w.numel() != H * W:
        raise RuntimeError("seam weights must have one entry per texel")
    ix = (uv[:, 0] * W - 0.5).clamp(0, W - 1)         # unnormalised align_corners=False, then border clipping
    iy = (uv[:, 1] * H - 0.5).clamp(0, H - 1)
    cols, ws = _corners(ix, iy, H, W)
    self_col = torch.arange(H * W, device=uvs.device, dtype=torch.int64)[:, None]
    return torch.cat([self_col, cols], 1), torch.cat([(1 - w)[:, None], w[:, None] * ws], 1)


class SeamSampler(nn.Module):
    """seams.py:28-56 with the reference's four persistent buffers (dst_ij [P,2], src_ij [P,2], uvs [H,W,2], weights),
    so `seam_sampler.*` checkpoint keys load strictly.  `impaint`, `resample` and `forward` (= impaint then resample,
    one gather) take a CUDA [B,C,H,W] map and return a new one.  Duplicate dst texels are refused (the reference's
    index_put leaves them undefined)."""

    def __init__(self, seamless_data):
        super().__init__()
        for k in ("dst_ij", "src_ij", "uvs", "weights"):
            self.register_buffer(k, torch.as_tensor(seamless_data[k]))
        self._tables, self._key = None, None

    def _buffers_key(self):
        return tuple((b.device, b.data_ptr(), b._version, tuple(b.shape))
                     for b in (self.dst_ij, self.src_ij, self.uvs, self.weights))

    def tables(self):
        key = self._buffers_key()
        if self._key != key:
            if self.uvs.device.type != "cuda":
                raise RuntimeError("SeamSampler runs on CUDA only: move it to the GPU first")
            H, W = self.uvs.shape[0], self.uvs.shape[1]
            dst = (self.dst_ij[:, 0].long() * W + self.dst_ij[:, 1].long())
            src = (self.src_ij[:, 0].long() * W + self.src_ij[:, 1].long())
            if torch.unique(dst).numel() != dst.numel():
                raise RuntimeError("SeamSampler: duplicate dst_ij entries (undefined in the reference's index_put)")
            src_of = torch.arange(H * W, device=dst.device, dtype=torch.int64)
            src_of[dst] = src                              # impaint reads the values before the copy
            col, coef = resample_entries(self.uvs, self.weights)
            self._tables = {
                "impaint": GatherTable(src_of[:, None], torch.ones(H * W, 1, device=dst.device), H * W),
                "resample": GatherTable(col, coef, H * W),
                "impaint_resample": GatherTable(src_of[col], coef, H * W),
            }
            self._key = key
        return self._tables

    def impaint(self, value):
        return gather(value, self.tables()["impaint"])

    def resample(self, tex):
        return gather(tex, self.tables()["resample"])

    def resample_border_only(self, tex):
        return self.resample(tex)

    def forward(self, tex):
        return gather(tex, self.tables()["impaint_resample"])
