"""Gathering per-tile detections across ranks: the replacement of collect_results_gpu
(mmdet/apis/test.py:117-147: pickle -> uint8 tensor -> all_gather(shape) -> all_gather(padded bytes) ->
unpickle) by ONE all_gather_into_tensor of a fixed-layout buffer.

Layout per tile: float32 [max_per_img + 1, 28]: rows = reppoints(18) | box(8) | score | label, zero padded; the last
row carries the tile's detection count.  Rank r holds tiles r, r+world, r+2*world, ... (DistributedSampler(shuffle=False) takes
indices[rank::world], mmdet/datasets/loader/sampler.py:26-32); `interleave` restores dataset order exactly as
`zip(*part_list)` + truncation does at apis/test.py:143-147.
"""
import torch
import torch.distributed as dist


def pack(dets, labels, counts):
    """padded (dets [T,cap,27], labels [T,cap], counts [T]) -> (buf [T,cap+1,28], counts): rows 0..cap-1 are the detections,
    row `cap` carries the tile's count in column 0 (exact in fp32 up to 2^24), so payload and counts travel in ONE collective"""
    t, cap = dets.shape[0], dets.shape[1]
    if dets.is_cuda and dets.dtype == torch.float32:
        # one kernel of the library instead of a fill and three strided copies
        from . import _lib
        buf = torch.empty((t, cap + 1, 28), dtype=torch.float32, device=dets.device)
        d, l, c = dets.contiguous(), labels.to(torch.int64).contiguous(), counts.to(torch.int32).contiguous()
        with torch.cuda.device(dets.device):
            _lib.check(_lib.lib().orp_pack_detections(_lib.ptr(d), _lib.ptr(l), _lib.ptr(c), t, cap, _lib.ptr(buf),
                                                      _lib.current_stream_ptr()), "orp_pack_detections")
        return buf, c
    buf = torch.zeros((t, cap + 1, 28), dtype=dets.dtype, device=dets.device)
    buf[:, :cap, :27] = dets
    buf[:, :cap, 27] = labels.to(dets.dtype)
    buf[:, cap, 0] = counts.to(dets.dtype)
    return buf, counts.to(torch.int32).contiguous()


class _Gathered:
    """result of all_gather_detections(async_op=True): wait() -> (all_buf [world,T,cap,28], all_counts [world,T]), or the
    whole [world,T,cap+1,28] buffer when the gather was asked for it (packed=True)"""

    def __init__(self, all_buf, work, packed=False):
        self._all_buf, self._work, self._packed = all_buf, work, packed

    def wait(self):
        if self._work is not None:
            self._work.wait()            # NCCL: the current stream waits for the collective; gloo: the host does
            self._work = None
        if self._packed:
            return self._all_buf
        cap = self._all_buf.shape[2] - 1
        return self._all_buf[:, :, :cap], self._all_buf[:, :, cap, 0].to(torch.int32)


def all_gather_detections(buf, counts=None, group=None, async_op=False, packed=False):
    """buf from pack() -> (all_buf [world,T,cap,28], all_counts [world,T]) with ONE all_gather_into_tensor.
    packed=True returns the gathered buffer as it is instead, [world,T,cap+1,28] with every tile's count row still in
    place: the input of dota.result_merge.merge_packed (with dataset_slots), which must not be given the split pair's
    all_buf - without the count row a tile's last detection row would be read as its count.
    async_op=True returns a handle whose wait() gives the same pair: the collective then overlaps whatever the caller
    launches next (ranks are not forced into lockstep every step)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        h = _Gathered(buf.unsqueeze(0), None, packed)
        return h if async_op else h.wait()
    if buf.is_cuda:
        all_buf = torch.empty((world,) + tuple(buf.shape), dtype=buf.dtype, device=buf.device)
        work = dist.all_gather_into_tensor(all_buf, buf.contiguous(), group=group, async_op=True)
        h = _Gathered(all_buf, work, packed)
    else:   # gloo (CPU tests)
        lb = [torch.empty_like(buf) for _ in range(world)]
        work = dist.all_gather(lb, buf, group=group, async_op=True)
        work.wait()
        h = _Gathered(torch.stack(lb), None, packed)
    return h if async_op else h.wait()


def interleave(all_buf, all_counts, dataset_len):
    """[world,T,...] -> per-tile list in dataset order (tile i lives on rank i % world, slot i // world)"""
    world, t = all_counts.shape
    out = []
    for i in range(min(dataset_len, world * t)):
        r, s = i % world, i // world
        k = int(all_counts[r, s])
        rows = all_buf[r, s, :k]
        out.append((rows[:, :27], rows[:, 27].long()))
    return out


def dataset_slots(world, t, dataset_len):
    """int32 [min(dataset_len, world * t)]: for dataset tile i, its slot in the all-gather's buffer flattened to
    [world * t, cap + 1, 28] - rank i % world, slot i // world, as `interleave` reads it; the sampler's padding tiles
    (indices >= dataset_len) are left out.  This is the `tile_slot` of dota.result_merge.merge_packed."""
    i = torch.arange(min(int(dataset_len), int(world) * int(t)), dtype=torch.int32)
    return (i % world) * t + torch.div(i, world, rounding_mode='floor')
