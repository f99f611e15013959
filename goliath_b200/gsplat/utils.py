"""Binning utilities with the gsplat 0.1.11 `gsplat.utils` names: cumulative intersects, intersection keys,
stable radix sort, tile bin edges.  Integer/byte work with a bit-exact contract (SURVEY.md Appendix A)."""
from typing import Tuple

import torch
from torch import Tensor

from .. import _lib

_WS = {}
_WS_RETIRED = {}  # outgrown buffers stay allocated: a captured CUDA graph may still hold their addresses


def _workspace(dev, nbytes: int) -> Tensor:
    """Grow-only scratch buffer per (device, stream) — the C ABI never allocates.  Renders issued on different streams
    get different buffers (a shared one would race); work on one stream is ordered, so sharing inside a stream is safe.
    A buffer that is outgrown is retired, not freed — kernels already captured in a CUDA graph keep pointing into it
    (sizes grow by at least 25 % per step, so the retired buffers together stay below four times the live one)."""
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    key = (dev.type, idx, torch.cuda.current_stream(idx).cuda_stream)
    buf = _WS.get(key)
    if buf is None or buf.numel() < nbytes:
        if buf is not None:
            _WS_RETIRED.setdefault(key, []).append(buf)
        buf = torch.empty(max(int(nbytes * 1.25), 1 << 20), dtype=torch.uint8, device=dev)
        _WS[key] = buf
    return buf


def _tile_bounds(img_height, img_width, block_width):
    return ((img_width + block_width - 1) // block_width, (img_height + block_width - 1) // block_width, 1)


def key_bits(num_tiles: int) -> int:
    return 32 + max(1, (max(num_tiles, 1) - 1).bit_length())


def compute_cumulative_intersects(num_tiles_hit: Tensor) -> Tuple[int, Tensor]:
    _lib.check_input(num_tiles_hit, "num_tiles_hit", torch.int32)
    n = num_tiles_hit.numel()
    cum = torch.empty_like(num_tiles_hit)
    if n == 0:
        return 0, cum
    dev = num_tiles_hit.device
    ws = _workspace(dev, _lib.kernels().gb_cumsum_workspace_bytes(n))
    _lib.kernels().gb_cumsum_i32(n, num_tiles_hit, cum, ws)
    num_intersects = int(cum[-1].item())  # same host sync as the reference (gsplat utils: cum_tiles_hit[-1].item())
    return num_intersects, cum


def map_gaussian_to_intersects(num_points: int, num_intersects: int, xys: Tensor, depths: Tensor, radii: Tensor,
                               cum_tiles_hit: Tensor, tile_bounds, block_width: int) -> Tuple[Tensor, Tensor]:
    dev = xys.device
    isect_ids = torch.empty(num_intersects, dtype=torch.int64, device=dev)
    gaussian_ids = torch.empty(num_intersects, dtype=torch.int32, device=dev)
    img_w, img_h = tile_bounds[0] * block_width, tile_bounds[1] * block_width
    _lib.kernels().gb_map_gaussian_to_intersects(
        num_points, xys.contiguous(), depths.contiguous(), radii.contiguous(), cum_tiles_hit.contiguous(), img_h,
        img_w, block_width, isect_ids, gaussian_ids)
    return isect_ids, gaussian_ids


def sort_intersects(isect_ids: Tensor, gaussian_ids: Tensor, num_tiles: int) -> Tuple[Tensor, Tensor]:
    n = isect_ids.numel()
    dev = isect_ids.device
    isect_sorted = torch.empty_like(isect_ids)
    gids_sorted = torch.empty_like(gaussian_ids)
    if n == 0:
        return isect_sorted, gids_sorted
    ws = _workspace(dev, _lib.kernels().gb_sort_workspace_bytes(n))
    _lib.kernels().gb_sort_intersects(n, isect_ids, gaussian_ids, isect_sorted, gids_sorted, key_bits(num_tiles),
                                      ws)
    return isect_sorted, gids_sorted


def get_tile_bin_edges(num_intersects: int, isect_ids_sorted: Tensor, tile_bounds) -> Tensor:
    dev = isect_ids_sorted.device
    tile_bins = torch.zeros(tile_bounds[0] * tile_bounds[1], 2, dtype=torch.int32, device=dev)
    _lib.kernels().gb_get_tile_bin_edges(num_intersects, isect_ids_sorted, tile_bins)
    return tile_bins


def bin_and_sort_gaussians(num_points: int, num_intersects: int, xys: Tensor, depths: Tensor, radii: Tensor,
                           cum_tiles_hit: Tensor, tile_bounds, block_width: int):
    isect_ids, gaussian_ids = map_gaussian_to_intersects(
        num_points, num_intersects, xys, depths, radii, cum_tiles_hit, tile_bounds, block_width)
    isect_ids_sorted, gaussian_ids_sorted = sort_intersects(isect_ids, gaussian_ids, tile_bounds[0] * tile_bounds[1])
    tile_bins = get_tile_bin_edges(num_intersects, isect_ids_sorted, tile_bounds)
    return isect_ids, gaussian_ids, isect_ids_sorted, gaussian_ids_sorted, tile_bins
