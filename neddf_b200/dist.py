"""Multi-GPU rendering: rays shard over ranks, one all-gather of image tiles, nothing else.

The reference is single-process (SURVEY 2: no torch.distributed anywhere); this is the H100
design of BASELINE.json north_star / SURVEY 8(e): one process per GPU, weights replicated
(each rank loads the same 2.6 MB state_dict), the row-major pixel list of every frame is cut
into ``world_size`` contiguous slices, each rank renders its slice with the single-GPU
kernels, and the only communication is ONE all-gather per frame of the packed
[pixels/rank, C] fp32 tile (NCCL over NVLink; gloo on CPU for the host-logic tests).
"""
import warnings
from typing import Dict, Iterable, List, Tuple

import torch
import torch.distributed as dist

from .network import EngineRangeError


def shard_range(n_items: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous slice [first, first+count) of ``n_items`` for ``rank``; slices differ by at most
    one item and tile the range exactly."""
    base, rem = divmod(n_items, world_size)
    first = rank * base + min(rank, rem)
    return first, base + (1 if rank < rem else 0)


def tile_capacity(n_items: int, world_size: int) -> int:
    """Per-rank tile length used for the gather (the largest slice)."""
    return (n_items + world_size - 1) // world_size


def gather_tiles(tile: torch.Tensor, n_items: int, group=None) -> torch.Tensor:
    """All-gather per-rank tiles [count_r, C] into the full [n_items, C] tensor (every rank gets
    it).  Exactly one collective; ragged last tiles are padded to a common length."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    cap = tile_capacity(n_items, world)
    C = tile.shape[1]
    first, count = shard_range(n_items, world, rank)
    assert tile.shape[0] == count, (tile.shape, count)
    if count != cap:
        pad = torch.zeros(cap, C, dtype=tile.dtype, device=tile.device)
        pad[:count] = tile
        tile = pad
    out = torch.empty(world * cap, C, dtype=tile.dtype, device=tile.device)
    dist.all_gather_into_tensor(out, tile.contiguous(), group=group)
    if n_items % world == 0:
        return out
    parts: List[torch.Tensor] = []
    for r in range(world):
        _, c = shard_range(n_items, world, r)
        parts.append(out[r * cap:r * cap + c])
    return torch.cat(parts, 0)


def render_image_sharded(render, width: int, height: int, camera, target_types: Iterable[str],
                         downsampling: int = 1, uniforms=None, group=None) -> Dict[str, torch.Tensor]:
    """NeRFRender.render_image across the ranks of ``group``: every rank returns the full images.

    ``uniforms`` (optional) are the full-image uniforms ([P,S_c+1], [P,S_f+1]); each rank consumes
    its own slice, so the result equals the single-GPU render with the same uniforms.
    """
    target_types = list(target_types)
    w, h = width // downsampling, height // downsampling
    n_pix = w * h
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    first, count = shard_range(n_pix, world, rank)
    u = None
    if uniforms is not None:
        u = (uniforms[0][first:first + count], uniforms[1][first:first + count])
    flat = render.render_pixels(width, height, camera, target_types, downsampling, first, count, u)
    if getattr(render, "check_nan", False):
        try:
            render.check_status()  # NaN weights raise, a failed resampling is reported - like render_image
        except EngineRangeError as e:  # engine "auto" left fp16 range on this rank: its shard again on the fp32 engine
            warnings.warn(str(e), RuntimeWarning)
            flat = render.render_pixels(width, height, camera, target_types, downsampling, first, count, u)
            render.check_status()
    widths = [flat[k].shape[1] for k in target_types]
    packed = torch.cat([flat[k] for k in target_types], 1) if len(target_types) > 1 else flat[target_types[0]]
    full = gather_tiles(packed, n_pix, group)
    out: Dict[str, torch.Tensor] = {}
    c0 = 0
    for k, cw in zip(target_types, widths):
        out[k] = full[:, c0:c0 + cw].reshape(h, w, cw)
        c0 += cw
    return out
