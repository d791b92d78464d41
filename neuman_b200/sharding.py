"""Ray sharding across the GPUs of one box (SURVEY.md §8e): every ray is independent, so the frame's pixels are dealt
to the ranks as interleaved 16x16 tiles (human-hit rays cluster spatially and cost more: contiguous row blocks would
leave some ranks with all of them), each rank renders its pixel list into one contiguous shard, ONE all_gather of
equal-sized shards moves them, and one un-permute kernel (nm_assemble_frame) writes the row-major frame.  No other
collective is on the path."""
import ctypes as C

import numpy as np
import torch

TILE = 16


def shard_range(n_pixels, rank, world):
    """Contiguous, balanced split: returns (first_pixel, count) of `rank` (kept for callers that shard by rows)."""
    base, rem = divmod(int(n_pixels), int(world))
    cnt = base + (1 if rank < rem else 0)
    p0 = rank * base + min(rank, rem)
    return p0, cnt


def tile_pixels(H, W, rank, world, tile=TILE):
    """Row-major pixel indices (int32 numpy) of the tiles t = rank, rank + world, ... of the H x W frame; tiles are numbered
    row-major over the tile grid, pixels inside a tile row-major, edge tiles are clipped."""
    ty, tx = (H + tile - 1) // tile, (W + tile - 1) // tile
    ids = np.arange(rank, ty * tx, world)
    if ids.size == 0:
        return np.zeros(0, np.int32)
    y0, x0 = (ids // tx) * tile, (ids % tx) * tile
    dy, dx = np.meshgrid(np.arange(tile), np.arange(tile), indexing="ij")
    ys = y0[:, None, None] + dy[None]
    xs = x0[:, None, None] + dx[None]
    ok = (ys < H) & (xs < W)
    return (ys * W + xs)[ok].astype(np.int32)


class TilePartition:
    """This rank's share of an H x W frame and the buffers of the one-gather reassembly.

        part = TilePartition(H, W, rank, world, device)
        rgb, depth, acc = part.buffers()          # views into this rank's shard: pass as `out=` with pixels=part.pixels
        frame = part.gather()                     # [H*W, planes] on every rank (world == 1: no collective, no copy pass)
    """

    def __init__(self, H, W, rank, world, device, group=None, tile=TILE):
        self.H, self.W, self.rank, self.world, self.group = int(H), int(W), int(rank), int(world), group
        self.device = torch.device(device)
        lists = [tile_pixels(H, W, r, world, tile) for r in range(world)]
        self.counts = [int(x.size) for x in lists]
        self.per = max(self.counts) if self.counts else 0
        self.n = self.counts[rank]
        self.pixels = torch.from_numpy(lists[rank]).to(self.device)
        allp = -np.ones((world, self.per), np.int32)
        for r, x in enumerate(lists):
            allp[r, :x.size] = x
        self.pixels_all = torch.from_numpy(allp.reshape(-1)).to(self.device)
        self._shard = None
        self._gathered = None
        self._frame = None
        self._planes = 5

    def _alloc(self, planes):
        if self._shard is None or self._planes != planes:
            self._planes = planes
            self._shard = torch.zeros(planes * self.per, device=self.device)
            self._gathered = torch.empty(self.world * planes * self.per, device=self.device) if self.world > 1 else None
            n_pix = self.H * self.W
            self._frame = (torch.empty(n_pix, 3, device=self.device), torch.empty(n_pix, device=self.device),
                           torch.empty(n_pix, device=self.device) if planes == 5 else None)

    def buffers(self, with_acc=True):
        """(rgb [n,3], depth [n], acc [n] | None): contiguous views into this rank's shard."""
        self._alloc(5 if with_acc else 4)
        per, n, s = self.per, self.n, self._shard
        return (s[:3 * per][:3 * n].view(n, 3), s[3 * per:4 * per][:n], s[4 * per:5 * per][:n] if with_acc else None)

    def gather(self):
        """One all_gather of the equal-sized shards + the un-permute kernel.  Returns the row-major frame planes
        (rgb [HW,3], depth [HW], acc [HW] | None) on every rank; the tensors are reused by the next call."""
        from . import ops
        ctx = ops._device_ctx(self.device)
        planes = self._planes
        if self.world > 1:
            import torch.distributed as dist
            dist.all_gather_into_tensor(self._gathered, self._shard, group=self.group)
            src = self._gathered
        else:
            src = self._shard
        rgb, depth, acc = self._frame
        ctx.check(ctx.lib.nm_assemble_frame(ctx.h, ops._p(src), self.world, self.per, planes, ops._p(self.pixels_all), ops._p(rgb),
                                            ops._p(depth), ops._p(acc), ctx.stream()))
        return rgb, depth, acc


def gather_frame(local, n_pixels, rank, world, group=None):
    """Row-block variant (contiguous shard_range shards): local [count_r, C] -> full [n_pixels, C] on every rank with one
    all_gather of equal-sized, padded shards.  Works with gloo (CPU) and nccl."""
    import torch.distributed as dist
    if world == 1:
        return local
    Cn = local.shape[1]
    per = (n_pixels + world - 1) // world
    pad = torch.zeros(per, Cn, dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    out = torch.empty(world * per, Cn, dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    parts = []
    for r in range(world):
        _, cnt = shard_range(n_pixels, r, world)
        parts.append(out[r * per:r * per + cnt])
    return torch.cat(parts, 0)
