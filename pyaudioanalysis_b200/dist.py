"""Clip sharding across the GPUs of one box (one process per GPU, torch.distributed).

Clips are independent (no state crosses feature_extraction calls), so the path shards with no data-path collective;
the only exchange is the final gather of the per-rank [clips, F, T] blocks on one rank (SURVEY 8e).  Two forms:

* ``gather="p2p"`` (GPUs): the root owns one [n_clips, F, T] buffer, every other rank maps it over NVLink
  (``b200aa_peer_buffer_*``, CUDA IPC) and pushes its finished block into its slice with the copy engines
  (``b200aa_peer_copy``): no collective kernel, no SMs taken on either side, and in a loop the push of batch i rides
  under the kernels of batch i + 1;
* ``gather="p2p_store"``: the feature kernel writes its slice of the mapped buffer directly (gather fused into the tile
  store); its 32-byte remote stores from many GPUs converge on one root, so it is not the default;
* ``gather="nccl"`` / gloo: ``torch.distributed.gather`` of padded blocks (the baseline, and what the CPU tests run).
"""
import ctypes

import torch
import torch.distributed as dist


def shard_bounds(n_clips, rank, world):
    """Contiguous block of clips owned by ``rank``: sizes differ by at most one."""
    base, rem = divmod(int(n_clips), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_blocks(local, n_clips, dst=0, group=None):
    """Gather per-rank blocks [n_local, ...] into [n_clips, ...] on ``dst`` (None elsewhere).

    Blocks may differ by one clip; they are padded to the largest block for the collective and
    trimmed afterwards.
    """
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_bounds(n_clips, r, world) for r in range(world)]
    big = max(hi - lo for lo, hi in sizes)
    pad = local
    if local.shape[0] < big:
        pad = torch.zeros((big,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        pad[:local.shape[0]] = local
    bufs = [torch.empty_like(pad) for _ in range(world)] if rank == dst else None
    dist.gather(pad.contiguous(), bufs, dst=dst, group=group)
    if rank != dst:
        return None
    return torch.cat([b[:hi - lo] for b, (lo, hi) in zip(bufs, sizes)], dim=0)


class _DevicePtr:
    """Minimal __cuda_array_interface__ carrier so torch can view raw (possibly peer-mapped) device memory."""

    def __init__(self, ptr, shape, typestr="<f4"):
        self.__cuda_array_interface__ = {"shape": tuple(int(s) for s in shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2, "strides": None}


class PeerGather:
    """One float32 [n_clips, F, T] buffer in the HBM of rank ``dst``, mapped into every rank of the group.

    ``view(lo, hi)`` is this rank's window onto clips lo..hi-1 (local memory on the root, NVLink peer memory
    elsewhere): pass it as ``out=`` of ``feature_extraction_batch``.  ``finish()`` makes the writes of all ranks
    visible to the root (stream synchronise + barrier) and returns the full tensor there (None elsewhere).
    """

    def __init__(self, n_clips, n_feats, n_frames, dst=0, group=None):
        from ._lib import lib, check
        self.group, self.dst = group, dst
        self.rank = dist.get_rank(group)
        self.shape = (int(n_clips), int(n_feats), int(n_frames))
        self.owner = self.rank == dst
        nbytes = 4 * self.shape[0] * self.shape[1] * self.shape[2]
        L = lib()
        p = ctypes.c_void_p()
        handle = (ctypes.c_ubyte * 64)()
        box = [None]
        if self.owner:
            check(L.b200aa_peer_buffer_create(nbytes, ctypes.byref(p), handle))
            box[0] = bytes(handle)
        dist.broadcast_object_list(box, src=dist.get_global_rank(group, dst) if group is not None else dst, group=group)
        if not self.owner:
            h = (ctypes.c_ubyte * 64).from_buffer_copy(box[0])
            check(L.b200aa_peer_buffer_open(h, ctypes.byref(p)))
        self.ptr = p.value
        self._L = L
        self.device = torch.device("cuda", torch.cuda.current_device())

    def view(self, lo, hi):
        n, F, T = self.shape
        if not (0 <= lo <= hi <= n):
            raise ValueError("clip range outside the gather buffer")
        if hi == lo:
            return torch.empty((0, F, T), dtype=torch.float32, device=self.device)
        if not self.owner:       # peer memory: only its address is needed (torch would attribute it to the owner's device)
            from .batch import DeviceBuffer
            return DeviceBuffer(self.ptr + 4 * lo * F * T, (hi - lo, F, T))
        return torch.as_tensor(_DevicePtr(self.ptr + 4 * lo * F * T, (hi - lo, F, T)), device=self.device)

    def push(self, local, lo, stream=None):
        """Copy this rank's finished block ``local`` ([n, F, T] float32 CUDA tensor) into clips lo.. of the buffer with the
        copy engines, asynchronously on ``stream`` (default: the current stream)."""
        n, F, T = self.shape
        if local.dtype != torch.float32 or not local.is_contiguous() or tuple(local.shape[1:]) != (F, T) or lo + local.shape[0] > n:
            raise ValueError("block does not fit the gather buffer")
        st = torch.cuda.current_stream() if stream is None else stream
        from ._lib import check
        check(self._L.b200aa_peer_copy(ctypes.c_void_p(self.ptr + 4 * lo * F * T), ctypes.c_void_p(local.data_ptr()),
                                       4 * local.numel(), ctypes.c_void_p(st.cuda_stream)))

    def finish(self):
        torch.cuda.current_stream().synchronize()      # this rank's kernels (and their remote stores) are complete
        dist.barrier(group=self.group)
        return self.view(0, self.shape[0]) if self.owner else None

    def close(self):
        if getattr(self, "ptr", None):
            self._L.b200aa_peer_buffer_close(ctypes.c_void_p(self.ptr), 1 if self.owner else 0)
            self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def feature_extraction_sharded(all_clips_fn, n_clips, sampling_rate, window, step, deltas=True, gather_to=0,
                               compute=None, group=None, gather="nccl"):
    """Each rank extracts features for its block of clips; optionally gather on ``gather_to``.

    ``all_clips_fn(lo, hi)`` returns this rank's clips [hi-lo, N] on its device; ``compute`` defaults to the GPU path
    (``feature_extraction_batch``) and is injectable so the sharding logic can be tested on CPU with gloo.
    ``gather="p2p"`` / ``"p2p_store"``: through the root's peer-mapped buffer (GPUs of one box only), see the module text.
    """
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    lo, hi = shard_bounds(n_clips, rank, world)
    clips = all_clips_fn(lo, hi)
    if gather in ("p2p", "p2p_store") and gather_to is not None and compute is None:
        from .batch import feature_extraction_batch
        from ._lib import lib
        T = lib().b200aa_num_frames(int(clips.shape[-1]), int(window), int(step))
        if T <= 0:
            raise ValueError("need at least one array to concatenate")
        pg = PeerGather(n_clips, 68 if deltas else 34, T, dst=gather_to, group=group)
        if hi > lo:
            if gather == "p2p_store" or pg.owner:
                feature_extraction_batch(clips, sampling_rate, window, step, deltas=deltas, out=pg.view(lo, hi))
            else:
                pg.push(feature_extraction_batch(clips, sampling_rate, window, step, deltas=deltas), lo)
        res = pg.finish()
        if res is not None:
            res = res.clone()
        dist.barrier(group=group)        # the root has copied: mappings may go
        pg.close()
        return res
    if compute is None:
        from .batch import feature_extraction_batch
        compute = lambda x: feature_extraction_batch(x, sampling_rate, window, step, deltas=deltas)   # noqa: E731
    local = compute(clips)
    if gather_to is None:
        return local
    return gather_blocks(local, n_clips, dst=gather_to, group=group)
