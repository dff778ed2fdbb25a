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

`TrackPipeline` is the same loop for tracking: every submit is the next frame of S independent video slots
(`run_batch(list, track=True)`: frames of mixed sizes, None for an idle slot, `new_video` to start a video in a slot):

    pipe = TrackPipeline(det, slots=8, camera_matrix=K)
    for frames, starts in videos:               # per slot: uint8 [H_i,W_i,3] or None; per slot: bool
        pipe.submit(frames, new_video=starts)
        if pipe.in_flight == pipe.depth:
            tracks, n_tracks = pipe.collect()   # [S,T,320], [S] of the OLDEST submitted frame

Both take `pixel_format="nv12"` or `"i420"` for YUV 4:2:0 frames as video decoders give them (uint8 [3H/2,W] per
frame, H and W even): they are uploaded as they are, half the bytes of BGR, and converted inside the pre-process
kernel; the results equal those of the same frames converted by cv2.cvtColor and submitted as BGR.  The camera and
sensor formats of engine.check_pixel_format work the same way; a Bayer mosaic or "gray" frame is uint8 [H,W], a third
of the bytes of BGR, and a phone format ("nv21", "yv12", "nv12_full", "nv21_full", "i420_full", "yv12_full") is 4:2:0
like "nv12".

Both take `distortion=` (lens.LensDistortion, one for every camera or one per frame / slot) for cameras with lens
distortion: the frames are undistorted inside the pre-process exactly as run_batch(distortion=) does.
"""
import collections

import numpy as np
import torch

from . import _lib
from .dist import PoseBuffer, shard_range, slot_layout
from .engine import check_pixel_format, frame_shape
from .lens import slot_distortions


class _Slot(object):
    def __init__(self, batch, shape, K, device, world):
        self.u8 = torch.empty((batch,) + shape, dtype=torch.uint8, device=device)
        self.staging = torch.empty((batch,) + shape, dtype=torch.uint8).pin_memory()
        self.pbuf = PoseBuffer(batch, K, device, world=world)
        self.h2d_done = torch.cuda.Event()
        self.compute_done = torch.cuda.Event()           # the pre-process kernel has consumed `u8`
        self.side_done = torch.cuda.Event()              # all-gather + download of this slot finished
        self.used = False


class BatchPipeline(object):
    """height, width: the image size of every frame; pixel_format "bgr" (frames uint8 [B,H,W,3]), "nv12" or "i420"
    (uint8 [B,3H/2,W]); distortion: one LensDistortion for every frame, or a list of one per frame of a batch."""

    def __init__(self, det, batch, height, width, camera_matrix, world=1, depth=2, to_host=True, group=None,
                 pixel_format="bgr", distortion=None):
        self.pixel_format = check_pixel_format(pixel_format)
        self.distortion = slot_distortions(distortion, int(batch), "BatchPipeline")
        shape = frame_shape(int(height), int(width), pixel_format)
        self.det, self.cam, self.depth, self.to_host, self.group = det, camera_matrix, int(depth), to_host, group
        self.device = torch.device(det.opt.device)
        if self.device.type != "cuda":
            raise RuntimeError("BatchPipeline needs a CUDA device (the hot path has no CPU fallback)")
        self.batch, self.height, self.width = int(batch), int(height), int(width)
        with torch.cuda.device(self.device):
            self.copy_stream = torch.cuda.Stream()
            self.side_stream = torch.cuda.Stream()
            self.slots = [_Slot(batch, shape, det.opt.K, self.device, world) for _ in range(self.depth)]
        self._queue = collections.deque()
        self._next = 0

    @property
    def in_flight(self):
        return len(self._queue)

    def submit(self, frames):
        """frames: uint8 [B,H,W,3] (or [B,3H/2,W] in a YUV pixel_format) numpy array or CPU tensor (pinned memory makes
        the upload asynchronous)."""
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
        self.det.run_batch(slot.u8, self.cam, to_host=False, out=(slot.pbuf.poses, slot.pbuf.n_valid),
                           pixel_format=self.pixel_format, distortion=self.distortion)
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


class _TrackSet(object):
    """One of the `depth` buffer sets of TrackPipeline: per local slot a device frame buffer and a pinned staging
    buffer (grown to the largest frame seen), and the track records of one step."""

    def __init__(self, rows, T, device, world):
        self.dev = {}
        self.staging = {}
        self.buf = PoseBuffer(rows, T, device, world=world, R=_lib.CP_TRACK_RECORD)
        self.h2d_done = torch.cuda.Event()
        self.compute_done = torch.cuda.Event()
        self.side_done = torch.cuda.Event()
        self.used = False

    def device_frame(self, i, shape, device):
        n = int(np.prod(shape))
        if i not in self.dev or self.dev[i].numel() < n:
            self.dev[i] = torch.empty((n,), dtype=torch.uint8, device=device)
        return self.dev[i][:n].view(shape)

    def staged_frame(self, i, shape):
        n = int(np.prod(shape))
        if i not in self.staging or self.staging[i].numel() < n:
            self.staging[i] = torch.empty((n,), dtype=torch.uint8).pin_memory()
        return self.staging[i][:n].view(shape)


class TrackPipeline(object):
    """Double-buffered `run_batch(list, track=True)` over `slots` video slots: the frames of step i+1 are uploaded
    (through pinned staging) on a copy stream while step i computes, and the track records of step i are read back one
    submit later.  With world > 1 (under torchrun) rank `rank` runs the slots shard_range(slots, rank, world) and one
    all-gather per step collects everyone's records (`dist.slot_layout`).  pixel_format "nv12" / "i420": every frame is
    YUV 4:2:0, uint8 [3H/2,W].  distortion: one LensDistortion for every slot, or a list of one per slot (None: an
    undistorted camera); a camera changed by submit(camera_matrix=) gets its own map (built once, then cached)."""

    def __init__(self, det, slots, camera_matrix, world=1, rank=0, depth=2, to_host=True, group=None, pixel_format="bgr",
                 distortion=None):
        self.pixel_format = check_pixel_format(pixel_format)
        self.distortion = slot_distortions(distortion, int(slots), "TrackPipeline")
        self.det, self.depth, self.to_host, self.group = det, int(depth), to_host, group
        self.device = torch.device(det.opt.device)
        if self.device.type != "cuda":
            raise RuntimeError("TrackPipeline needs a CUDA device (the hot path has no CPU fallback)")
        self.slots, self.world, self.rank = int(slots), int(world), int(rank)
        self.lo, self.hi = shard_range(self.slots, self.rank, self.world)
        self.rows, self.order = slot_layout(self.slots, self.world)
        from .detector import camera_per_frame
        self.cams = np.stack(camera_per_frame(camera_matrix, self.slots))
        self.T = _lib.CP_MAX_K
        with torch.cuda.device(self.device):
            self.copy_stream = torch.cuda.Stream()
            self.side_stream = torch.cuda.Stream()
            self.sets = [_TrackSet(self.rows, self.T, self.device, self.world) for _ in range(self.depth)]
        self._queue = collections.deque()
        self._next = 0

    @property
    def in_flight(self):
        return len(self._queue)

    def _local(self, values, name):
        from .detector import check_slot_list
        values = check_slot_list(values, self.slots, name)
        return None if values is None else values[self.lo:self.hi]

    def submit(self, frames, new_video=None, pre_dets=None, frame_ids=None, camera_matrix=None):
        """frames: one entry per slot (all `slots`, on every rank): uint8 [H,W,3] (or [3H/2,W] in a YUV pixel_format)
        numpy array or CPU tensor (pinned memory makes the upload asynchronous), or None for an idle slot.  new_video /
        pre_dets / frame_ids as in
        run_batch(list, track=True); camera_matrix: [3,3] or [slots,3,3] from this step on (e.g. when a slot starts
        a video from another camera)."""
        if len(self._queue) >= self.depth:
            raise RuntimeError("TrackPipeline: collect() the oldest step before submitting step %d" % (self.depth + 1))
        from .detector import camera_per_frame, check_frames
        if camera_matrix is not None:
            self.cams = np.stack(camera_per_frame(camera_matrix, self.slots))
        frames = self._local(frames, "frame")
        check_frames(frames, allow_idle=True, pixel_format=self.pixel_format)
        st = self.sets[self._next]
        self._next = (self._next + 1) % self.depth
        compute = torch.cuda.current_stream(self.device)
        srcs = []
        for i, f in enumerate(frames):
            if f is None:
                srcs.append(None)
                continue
            f = torch.from_numpy(f) if isinstance(f, np.ndarray) else f
            if not f.is_cuda and not f.is_pinned():      # pageable source: stage it, so the upload is asynchronous
                if st.used:
                    st.h2d_done.synchronize()            # the set's previous upload has left the staging buffers
                stage = st.staged_frame(i, tuple(f.shape))
                stage.copy_(f)
                f = stage
            srcs.append(f)
        dev_frames = []
        with torch.cuda.stream(self.copy_stream):
            if st.used:
                self.copy_stream.wait_event(st.compute_done)        # do not overwrite frames a queued step still reads
            for i, f in enumerate(srcs):
                if f is None:
                    dev_frames.append(None)
                    continue
                d = st.device_frame(i, tuple(f.shape), self.device)
                d.copy_(f, non_blocking=True)
                dev_frames.append(d)
            st.h2d_done.record(self.copy_stream)
        compute.wait_event(st.h2d_done)
        if st.used:
            compute.wait_event(st.side_done)             # the set's previous gather / download have read its records
        n = self.hi - self.lo
        if n > 0:
            self.det.run_batch(dev_frames, self.cams[self.lo:self.hi], to_host=False, track=True,
                               out=(st.buf.poses[:n], st.buf.n_valid[:n]), new_video=self._local(new_video, "new_video"),
                               pre_dets=self._local(pre_dets, "pre_dets"), frame_ids=self._local(frame_ids, "frame_ids"),
                               pixel_format=self.pixel_format,
                               distortion=None if self.distortion is None else self.distortion[self.lo:self.hi])
        st.compute_done.record(compute)
        st.used = True
        with torch.cuda.stream(self.side_stream):
            self.side_stream.wait_event(st.compute_done)
            st.buf.all_gather(self.group)
            if self.to_host:
                st.buf.to_host(sync=False)
            st.side_done.record(self.side_stream)
        self._queue.append(st)

    def collect(self):
        """(tracks [slots, T, 320], n_tracks [slots]) of the oldest submitted step, in slot order: numpy arrays when
        `to_host`, else CUDA tensors."""
        st = self._queue.popleft()
        if self.to_host:
            st.buf._evt.synchronize()
            tracks, n = st.buf.host_views()
            return tracks[self.order].copy(), n[self.order].copy()
        torch.cuda.current_stream(self.device).wait_event(st.side_done)
        tracks, n = st.buf.views(st.buf.gathered)
        if self.order == list(range(tracks.shape[0])):
            return tracks.clone(), n.clone()
        idx = torch.tensor(self.order, device=tracks.device)
        return tracks.index_select(0, idx), n.index_select(0, idx)
