"""Multi-GPU MultiExp: one process per GPU (torch.distributed, NCCL over NVLink), points/scalars
sharded contiguously, ONE tiny exchange at the end.

MSM is a sum over independent (P_i, s_i) terms; the reference exploits this with its recursive
halving joined by one AddAssign (ecc/bn254/multiexp.go:128-140).  Here rank r owns indices
[r*n/G, (r+1)*n/G), runs the full bucket pass on its slice and produces W per-window partial sums
(extended Jacobian, 128 B each for bn254 G1).  Elliptic-curve addition is not an NCCL reduction
operator, so the "allreduce of one partial point per window" is an all-gather of the W partials
(2 KiB per rank) followed by a local per-window add + Horner (gmsm_ctx_finalize_device) on every rank.
"""
from __future__ import annotations


def shard_range(n: int, rank: int, world: int):
    """contiguous shard [lo, hi) of n items for `rank` of `world`"""
    if not (0 <= rank < world):
        raise ValueError("rank %d out of range for world size %d" % (rank, world))
    return n * rank // world, n * (rank + 1) // world


def gather_partials(local, world: int, group=None):
    """all-gather equal-sized 1-D tensors -> concatenation ordered by rank (works for NCCL and gloo)"""
    import torch
    import torch.distributed as dist

    if world == 1:
        return local
    out = torch.empty(world * local.numel(), dtype=local.dtype, device=local.device)
    if dist.get_backend(group) == "gloo":
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local, group=group)
        return torch.cat(parts)
    dist.all_gather_into_tensor(out, local, group=group)
    return out


def window_bits_for_total(curve: str, n_total: int, world: int = 1) -> int:
    """the window width every rank of a sharded MSM must use: derived ONCE from (total size, world) -- the width model
    (gmsm_choose_window_bits) prices the work of one device, so it is asked for the LARGEST shard, ceil(n_total / world) -- and
    never from a rank's own shard: uneven shards would otherwise pick different plans and their partials could not be added"""
    from . import _native
    from .multiexp import CURVES

    world = max(1, int(world))
    return int(_native.lib().gmsm_choose_window_bits(CURVES[curve], (int(n_total) + world - 1) // world))


class ShardedMultiExp:
    """engine + process group.  msm() returns the Jacobian triple (device tensor) on every rank.  All ranks must run the same
    window plan: the constructor all-gathers (c, W) and refuses a mismatch (create the engines with
    c = window_bits_for_total(curve, n_total, world))."""

    def __init__(self, engine, group=None):
        import torch
        import torch.distributed as dist

        self.engine = engine
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if self.world > 1:
            dev = torch.device("cuda", engine.device) if dist.get_backend(group) != "gloo" else torch.device("cpu")
            mine = torch.tensor([engine.c, engine.nwin], dtype=torch.int64, device=dev)
            plans = gather_partials(mine, self.world, group).cpu().view(self.world, 2)
            if not bool((plans == plans[0]).all()):
                raise ValueError("ranks run different window plans (c, W): %s -- create every engine with "
                                 "c = window_bits_for_total(curve, n_total, world)" % plans.tolist())

    def msm_from_host(self, h_points, h_scalars, n_local: int, d_points_buf, d_scalars_buf, chunks: int = 4):
        """End-to-end sharded MSM from pinned host shards: the shard is cut into `chunks` batches; batch k+1
        crosses PCIe on a copy stream while batch k runs the bucket pass (each batch yields W window
        partials); all ranks all-gather their chunks x W partials and finalize over world x chunks groups."""
        torch = self.engine.torch
        if not hasattr(self, "_copy_stream"):
            self._copy_stream = torch.cuda.Stream(device=self.engine.device)
        main = torch.cuda.current_stream(self.engine.device)
        self._copy_stream.wait_stream(main)
        wa = 2 * self.engine.w          # int64 words per affine point
        ws = self.engine.sw             # int64 words per scalar
        pw = self.engine.partials_bytes // 8
        chunks = max(1, min(chunks, n_local))
        partials = torch.empty(chunks * pw, dtype=torch.int64, device=d_points_buf.device)
        for k in range(chunks):
            lo, hi = n_local * k // chunks, n_local * (k + 1) // chunks
            with torch.cuda.stream(self._copy_stream):
                d_scalars_buf[lo * ws : hi * ws].copy_(h_scalars[lo * ws : hi * ws], non_blocking=True)
                d_points_buf[lo * wa : hi * wa].copy_(h_points[lo * wa : hi * wa], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self._copy_stream)
            main.wait_event(ev)
            self.engine.window_sums(d_points_buf[lo * wa :], d_scalars_buf[lo * ws :], hi - lo, out=partials[k * pw : (k + 1) * pw])
        allp = gather_partials(partials, self.world, self.group)
        return self.engine.finalize(allp, self.world * chunks)

    def msm_from_host_pipelined(self, h_points_np, h_scalars_np):
        """End-to-end sharded MSM through the C ABI's pipelined host entry point (geometric batches into one shared
        bucket array, H2D under compute): every rank gets its W window partials back, the ranks all-gather them
        over NCCL and finalize.  h_points_np / h_scalars_np: this rank's (pinned) numpy shards, Go layout."""
        import numpy as np

        from . import _native
        from .multiexp import _check

        torch = self.engine.torch
        eng = self.engine
        n_local = h_scalars_np.size // eng.sw
        part = np.empty(eng.partials_bytes // 8, dtype=np.uint64)
        _check(_native.lib().gmsm_multiexp_window_sums(eng.cid, h_points_np.ctypes.data, h_scalars_np.ctypes.data, n_local, eng.c,
                                                       eng.device, part.ctypes.data))
        local = torch.from_numpy(part.view(np.int64)).to(torch.device("cuda", eng.device))
        allp = gather_partials(local, self.world, self.group)
        return eng.finalize(allp, self.world)

    def msm(self, d_points_shard, d_scalars_shard, n_local: int):
        partials = self.engine.window_sums(d_points_shard, d_scalars_shard, n_local)
        allp = gather_partials(partials, self.world, self.group)
        return self.engine.finalize(allp, self.world)
