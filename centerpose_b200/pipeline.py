"""Double-buffered image -> pose stream on top of `ObjectPoseDetector.run_batch` (not in the reference, whose
`demo.py` loop is one synchronous frame at a time: base_detector.py:390-772).

A serving loop has three transfers per batch: frames host -> device, the network + decode on the device, pose records
device -> host.  Run back to back they serialise (a 32-frame batch uploads 25 MB of frames); here
the upload of batch i+1 runs on a copy stream while batch i computes, and the records of batch i are read back into a
pinned buffer that the caller collects one submit later:

    pipe = BatchPipeline(det, batch=32, height=512, width=512, camera_matrix=K)
    for frames in loader:                       # uint8 [B,H,W,3], ideally pinned
        pipe.submit(frames)
        if pipe.in_flight == pipe.depth:
            poses, n_valid = pipe.collect()     # the OLDEST submitted batch
    while pipe.in_flight:
        poses, n_valid = pipe.collect()

Every batch still pays its own upload and its own download; only their latency is hidden.  Under `torchrun` the
per-rank records are all-gathered (one NCCL call per batch, `dist.PoseBuffer`) before the download.
"""
import collections

import numpy as np
import torch

from .dist import PoseBuffer


class _Slot(object):
    def __init__(self, batch, height, width, K, device, world):
        self.u8 = torch.empty((batch, height, width, 3), dtype=torch.uint8, device=device)
        self.staging = torch.empty((batch, height, width, 3), dtype=torch.uint8).pin_memory()
        self.pbuf = PoseBuffer(batch, K, device, world=world)
        self.h2d_done = torch.cuda.Event()
        self.compute_done = torch.cuda.Event()           # the pre-process kernel has consumed `u8`
        self.side_done = torch.cuda.Event()              # all-gather + download of this slot finished
        self.used = False


class BatchPipeline(object):
    def __init__(self, det, batch, height, width, camera_matrix, world=1, depth=2, to_host=True, group=None):
        self.det, self.cam, self.depth, self.to_host, self.group = det, camera_matrix, int(depth), to_host, group
        self.device = torch.device(det.opt.device)
        if self.device.type != "cuda":
            raise RuntimeError("BatchPipeline needs a CUDA device (the hot path has no CPU fallback)")
        self.batch, self.height, self.width = int(batch), int(height), int(width)
        with torch.cuda.device(self.device):
            self.copy_stream = torch.cuda.Stream()
            self.side_stream = torch.cuda.Stream()
            self.slots = [_Slot(batch, height, width, det.opt.K, self.device, world) for _ in range(self.depth)]
        self._queue = collections.deque()
        self._next = 0

    @property
    def in_flight(self):
        return len(self._queue)

    def submit(self, frames):
        """frames: uint8 [B,H,W,3] numpy array or CPU tensor (pinned memory makes the upload asynchronous)."""
        if len(self._queue) >= self.depth:
            raise RuntimeError("BatchPipeline: collect() the oldest batch before submitting batch %d" % (self.depth + 1))
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        if tuple(frames.shape) != tuple(self.slots[0].u8.shape) or frames.dtype != torch.uint8:
            raise ValueError("BatchPipeline: expected uint8 frames of shape %s, got %s %s"
                             % (tuple(self.slots[0].u8.shape), frames.dtype, tuple(frames.shape)))
        slot = self.slots[self._next]
        self._next = (self._next + 1) % self.depth
        compute = torch.cuda.current_stream(self.device)
        if not frames.is_pinned():                       # pageable source: stage it, so the upload below is asynchronous
            if slot.used:
                slot.h2d_done.synchronize()              # the slot's previous upload has left the staging buffer
            slot.staging.copy_(frames)
            frames = slot.staging
        with torch.cuda.stream(self.copy_stream):
            if slot.used:
                self.copy_stream.wait_event(slot.compute_done)      # do not overwrite frames a queued batch still reads
            slot.u8.copy_(frames, non_blocking=True)
            slot.h2d_done.record(self.copy_stream)
        compute.wait_event(slot.h2d_done)
        if slot.used:
            compute.wait_event(slot.side_done)           # the slot's previous gather / download have read its records
        self.det.run_batch(slot.u8, self.cam, to_host=False, out=(slot.pbuf.poses, slot.pbuf.n_valid))
        slot.compute_done.record(compute)
        slot.used = True
        # the all-gather and the download run on a side stream: the next batch's kernels neither queue behind the copy nor
        # wait for a slower peer rank (the collective couples the ranks once per batch, not once per kernel queue)
        with torch.cuda.stream(self.side_stream):
            self.side_stream.wait_event(slot.compute_done)
            slot.pbuf.all_gather(self.group)
            if self.to_host:
                slot.pbuf.to_host(sync=False)
            slot.side_done.record(self.side_stream)
        self._queue.append(slot)

    def collect(self):
        """(poses [world*B, K, 192], n_valid [world*B]) of the oldest submitted batch: numpy views of the pinned buffer when
        `to_host` (valid until the slot is submitted again), else the device tensors."""
        slot = self._queue.popleft()
        if self.to_host:
            slot.pbuf._evt.synchronize()
            return slot.pbuf.host_views()
        torch.cuda.current_stream(self.device).wait_event(slot.side_done)
        return slot.pbuf.views(slot.pbuf.gathered)
