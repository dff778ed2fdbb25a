"""Live video in CUDA graphs: `slots` cameras, each with a frame size, a pixel format and a camera matrix, one step per
call replayed from a captured graph.  `_SlotGraph` is what every such graph shares -- the frame sizes and cameras, the
meta rows and affines, the frame buffers and frame table, the int32 control block of a step with idle slots, the
capture (the graphs of `_steps()`, or one per live count 1..S on one memory pool) and the call (the frame copies, the
control copy and one replay).  A graph class defines its step: the opt it refuses (`_refuse`), its buffers
(`_buffers`), the launches of a step (`_step`) and its outputs (`_out`).  `DetectGraph` / `MultiCategoryDetectGraph`
here replay run_batch of a detection model; `TrackGraph` / `MultiCategoryTrackGraph` (tracker.py) the tracking step."""
import ctypes
import warnings

import numpy as np
import torch

from . import _lib
from .engine import MJPEG, _ptr, _stream


def _frame_sizes(frame_hw, S, who):
    """frame_hw of a graph of S slots -> ([(H, W)], per_slot): one size for every slot, or one per slot."""
    per_slot = (isinstance(frame_hw, (list, tuple, np.ndarray)) and len(frame_hw) > 0
                and all(isinstance(v, (list, tuple, np.ndarray)) for v in frame_hw))
    if per_slot and len(frame_hw) != S:
        raise ValueError("%s: frame_hw is one (H, W) for every slot or one per slot, got %d for %d slots"
                         % (who, len(frame_hw), S))
    sizes = []
    for hw in (frame_hw if per_slot else [frame_hw]):
        if len(hw) != 2 or int(hw[0]) < 1 or int(hw[1]) < 1:
            raise ValueError("%s: frame_hw is one (H, W) for every slot or one per slot, got %r" % (who, frame_hw))
        sizes.append((int(hw[0]), int(hw[1])))
    return sizes, per_slot


class _SlotGraph(object):
    """The capture and call machinery of the live-video graphs (see the module docstring).  Subclasses define
    _refuse(opt, who), _buffers(opt, meta, trans), _steps(), _step(p) and set self._out in _buffers."""

    _host_list = "run_batch(list)"                    # where idle slots and mixed sizes run without a graph
    _mjpeg = ()                                       # the "mjpeg" slots, whose step decodes their frames first

    def _refuse(self, opt, who):
        """Raise for an opt the step does not take, before any device work."""
        raise NotImplementedError

    def _plan(self, det, S, ih, iw):
        """(plan, decode parameters, categories or None) of the graph: a copy of det's plan and weights, taken now.
        det: an ObjectPoseDetector (one category) or a MultiCategoryDetector / MultiCategoryTracker (its categories)."""
        from .detector import MultiCategoryDetector
        from .engine import Engine, decode_params
        if isinstance(det, MultiCategoryDetector):
            c, M = det._plan_cfg, len(det.categories)
            eng = Engine(c["arch"], c["heads"], c["head_conv"], S, ih, iw, self.device.index, tracking=c["tracking"],
                         tracking_task_gru=c["tracking_task_gru"], precision=c["precision"], models=M,
                         reuse_activations=True, batch_invariant=c["batch_invariant"])
            for m, sd in enumerate(det._weights):
                eng.load_state_dict(sd, model=m)
            return eng, (list(det._prms) if M > 1 else det._prms[0]), list(det.categories)
        m = det.model
        eng = Engine(m._arch(), m.heads, m.head_conv, S, ih, iw, self.device.index, tracking=m.tracking_inputs,
                     tracking_task_gru=m.use_convGRU and m.tracking_task, precision=m.precision, reuse_activations=True,
                     batch_invariant=m.batch_invariant)
        eng.load_state_dict(m.state_dict())
        return eng, decode_params(det.opt, test_scale=1.0), None

    def _build(self, det, slots, frame_hw, camera_matrix, pixel_format, idle_slots=False, distortion=None,
               max_frame_bytes=None):
        """Checks, buffers and the captured steps; everything that refuses comes before any device work."""
        from .detector import affine_from_center_scale, camera_per_frame
        from .engine import check_pixel_format, frame_shape, make_meta, map_pointers, slot_formats
        from .lens import slot_distortions, undistort_map, undistorted_cameras
        who, opt = type(self).__name__, det.opt
        self._refuse(opt, who)
        S = int(slots)
        if S < 1:
            raise ValueError("%s: slots must be >= 1, got %d" % (who, S))
        dists = slot_distortions(distortion, S, who)
        if dists is not None and (getattr(opt, "fix_short", 0) > 0 or not getattr(opt, "fix_res", True)):
            raise NotImplementedError("%s: distortion undistorts into the fix_res input; the keep_res and fix_short "
                                      "pre-process take no distortion" % who)
        sizes, self.per_slot = _frame_sizes(frame_hw, S, who)
        self.idle_slots = bool(idle_slots)
        if isinstance(pixel_format, (list, tuple)) and not self.per_slot:
            raise ValueError("%s: one pixel_format per slot goes with one frame_hw per slot; with one frame_hw every "
                             "slot takes one name, got %r" % (who, list(pixel_format)))
        # "mjpeg" slots are BGR slots whose frames the step decodes first; no other code learns the name
        names = list(pixel_format) if isinstance(pixel_format, (list, tuple)) else [pixel_format] * S
        self._mjpeg = [b for b, f in enumerate(names) if isinstance(f, str) and f == MJPEG] if len(names) == S else []
        if self._mjpeg:
            shown = pixel_format
            pixel_format = (["bgr" if b in self._mjpeg else f for b, f in enumerate(names)]
                            if isinstance(pixel_format, (list, tuple)) else "bgr")
        max_bytes = self._max_frame_bytes(max_frame_bytes, sizes if self.per_slot else sizes * S, who)
        fmts = slot_formats(pixel_format, S, who) if self.per_slot else [check_pixel_format(pixel_format)]
        # one name repeated is that name: the same table, launches and bits
        self.pixel_format = fmts[0] if len(set(fmts)) == 1 else fmts
        shapes = [frame_shape(h, w, f) for (h, w), f in zip(sizes, fmts)]
        cams = np.stack(camera_per_frame(camera_matrix, S))
        if dists is not None:                             # every map is built now, on the host, before device work
            host_maps = [None if d is None else undistort_map(d, cams[b], sizes[b if self.per_slot else 0],
                                                              (opt.input_h, opt.input_w)) for b, d in enumerate(dists)]
            cams = undistorted_cameras(dists, cams)       # the meta rows carry K_new
        if self.per_slot:
            self.frame_hw, self.frame_shape = sizes, shapes
        else:
            self.frame_hw, self.frame_shape = sizes[0], (S,) + shapes[0]
            sizes = sizes * S
        self._slot_hw, self._slot_shapes = sizes, shapes if self.per_slot else shapes * S
        self.L = L = _lib.load()
        self.slots, self.device = S, torch.device("cuda", torch.cuda.current_device())
        dev = self.device
        ih, iw = opt.input_h, opt.input_w
        self.eng, self.prm, self.categories = self._plan(det, S, ih, iw)
        M = 1 if self.categories is None else len(self.categories)
        self.streams = M * S                             # row (tracker stream) m * S + s: slot s of category m
        # every slot's row of run_batch: its fix_res c, s and meta row and the affine of its size
        meta, trans = np.zeros((S, _lib.CP_META_DOUBLES), np.float64), np.zeros((S, 6), np.float64)
        for b, (h, w) in enumerate(sizes):
            c, sc = np.array([w / 2., h / 2.], np.float32), float(max(h, w))
            meta[b] = make_meta(1, c, sc, w, h, cams[b]).numpy()[0]
            trans[b] = affine_from_center_scale(c, sc, iw, ih).reshape(6)
        self.meta = torch.from_numpy(meta).to(dev)                   # the network's rows, one per frame
        self._meta_host, self._distorted = meta, dists is not None    # what a per-step camera_matrix starts from
        self._mean = (ctypes.c_float * 3)(*[float(v) for v in opt.mean])
        self._std = (ctypes.c_float * 3)(*[float(v) for v in opt.std])
        mixed = isinstance(self.pixel_format, list)       # per-slot formats: a table of them, one per-frame launch
        self._fmt = _lib.CP_PIX_PER_FRAME if mixed else _lib.PIXEL_FORMAT_CODES[self.pixel_format]
        if self._mjpeg:
            self.pixel_format = shown if isinstance(shown, str) or len(set(shown)) > 1 else shown[0]
        # a frame table with one frame_hw per slot, idle slots or lens distortion (with one frame_hw: S equal sizes)
        self._table = self.per_slot or self.idle_slots or dists is not None
        if self._table:
            n = [int(np.prod(s)) for s in self._slot_shapes]
            offs = np.concatenate([[0], np.cumsum(n)[:-1]]).astype(np.int64)
            self.frames = torch.zeros((int(sum(n)),), dtype=torch.uint8, device=dev)
            self._slot_frames = [self.frames[o:o + k].view(s) for o, k, s in zip(offs, n, self._slot_shapes)]
            self.table = torch.zeros((int(L.cp_preprocess_frame_table_bytes(S)),), dtype=torch.uint8, device=dev)
            hw = np.ascontiguousarray(sizes, np.int32)
            p64, p32 = offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
            ptr = trans.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
            with torch.cuda.device(dev):
                if dists is not None:
                    # the maps live as long as the graph that reads them
                    self._maps = [None if m is None else torch.from_numpy(m).to(dev) for m in host_maps]
                    codes = np.array([_lib.PIXEL_FORMAT_CODES[f] for f in fmts], np.int32) if mixed else None
                    _lib.check(L.cp_preprocess_frame_table_maps(
                        self.frames.numel(), p64, p32, self._fmt,
                        None if codes is None else codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                        map_pointers(self._maps, S, ih, iw, dev, who), S, ih, iw, ptr, _ptr(self.table), _stream()),
                        "cp_preprocess_frame_table_maps")
                    self._fmt |= _lib.CP_PIX_REMAP
                elif mixed:
                    codes = np.array([_lib.PIXEL_FORMAT_CODES[f] for f in fmts], np.int32)
                    _lib.check(L.cp_preprocess_frame_table_formats(self.frames.numel(), p64, p32,
                                                                   codes.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                                                   S, ih, iw, ptr, _ptr(self.table), _stream()),
                               "cp_preprocess_frame_table_formats")
                else:
                    _lib.check(L.cp_preprocess_frame_table(self.frames.numel(), p64, p32, self._fmt, S, ih, iw, ptr,
                                                           _ptr(self.table), _stream()), "cp_preprocess_frame_table")
        else:
            self.frames = torch.zeros(self.frame_shape, dtype=torch.uint8, device=dev)
            offs = np.arange(S, dtype=np.int64) * int(np.prod(shapes[0]))
        if self._mjpeg:
            self._jpeg_buffers(max_bytes, offs)
        if self.idle_slots:
            # one int32 control block per call (_control): start flags [M*S], rows [S] (the slot of each live row), ids
            # [M*S] (the row m * S + slot of each live row of each category) and inv [M*S] (the live row of each
            # category's slot, or -1); a step at live count n reads the first n rows and M * n ids
            MS = self.streams
            self.ctrl = torch.zeros((3 * MS + S,), dtype=torch.int32, device=dev)
            self.start, self.rows = self.ctrl[:MS], self.ctrl[MS:MS + S]
            self.ids, self.inv = self.ctrl[MS + S:2 * MS + S], self.ctrl[2 * MS + S:]
            self.meta_rows = torch.zeros((S, _lib.CP_META_DOUBLES), dtype=torch.float64, device=dev)  # the live rows'
        self._buffers(opt, meta, trans)
        # the captured steps: _steps(), or with idle slots p = every live count 1..S
        steps = range(1, S + 1) if self.idle_slots else self._steps()
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):            # warm-up outside the capture
            for p in steps:
                if self.idle_slots:
                    self.ctrl.copy_(torch.from_numpy(self._control(list(range(p)), np.ones(S, np.int32))))
                self._step(p)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self._warmed()
        self.graphs, pool = [], None
        for p in steps:
            g = torch.cuda.CUDAGraph(keep_graph=True)
            with torch.cuda.graph(g, pool=pool):
                self._step(p)
            g.instantiate()
            self.graphs.append(g)
            if self.idle_slots:                  # the S graphs replay in turn on one stream: one memory pool
                pool = g.pool()
        self._parity = 0
        self._fresh = True
        self._started = [False] * S

    def _warmed(self):
        """After the warm-up steps, before the capture."""

    # ---- MJPEG slots -------------------------------------------------------------------------------------------------
    def _max_frame_bytes(self, max_frame_bytes, sizes, who):
        """The encoded bytes each slot takes: max_frame_bytes (one int or one per slot), by default H * W * 3."""
        if max_frame_bytes is None:
            return [h * w * 3 for h, w in sizes]
        if not self._mjpeg:
            raise ValueError("%s: max_frame_bytes caps the encoded frames of \"mjpeg\" slots, and no slot is one"
                             % who)
        per = list(max_frame_bytes) if isinstance(max_frame_bytes, (list, tuple, np.ndarray)) else \
            [max_frame_bytes] * len(sizes)
        if len(per) != len(sizes) or any(int(v) != v or not 1 <= int(v) < 1 << 28 for v in per):
            raise ValueError("%s: max_frame_bytes is one int or one per slot, each 1 .. 2^28 - 1, got %r"
                             % (who, max_frame_bytes))
        return [int(v) for v in per]

    def _jpeg_buffers(self, max_bytes, offs):
        """The slot decode's sizes, device block, encoded-byte buffer, workspace and error words; the block starts with
        every slot skipped."""
        L, S, dev = self.L, self.slots, self.device
        self._jhw = np.ascontiguousarray(self._slot_hw, np.int32)
        self._jmax = np.ascontiguousarray(max_bytes, np.int64)
        self._jbyte_offs = np.concatenate([[0], np.cumsum(self._jmax)[:-1]]).astype(np.int64)
        self._jout = np.ascontiguousarray(offs, np.int64)
        self._jblock_host = np.zeros(int(L.cp_jpeg_slots_block_bytes(S)), np.uint8)
        ws = L.cp_jpeg_slots_workspace_bytes(S, self._jhw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                             self._jmax.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 0)
        if ws == 0:
            _lib.check(-1, "cp_jpeg_slots_workspace_bytes")
        self._jws = torch.empty((int(ws),), dtype=torch.uint8, device=dev)
        self._jbytes = torch.zeros((int(self._jmax.sum()),), dtype=torch.uint8, device=dev)
        self._jblock = torch.zeros((self._jblock_host.size,), dtype=torch.uint8, device=dev)
        self.decode_errors = torch.zeros((S,), dtype=torch.int32, device=dev)
        self._prepare([None] * S)
        self._jblock.copy_(torch.from_numpy(self._jblock_host))

    def _encoded(self, b, f):
        """The encoded frame of MJPEG slot b, checked on the host: (its bytes as a CPU tensor, its CpJpegHeader)."""
        from .engine import jpeg_bytes, jpeg_parse
        who = type(self).__name__
        if torch.is_tensor(f) and f.is_cuda:
            raise ValueError("%s: slot %d is an \"mjpeg\" slot, whose header is parsed on the host: pass its frame "
                             "from host memory, not as a CUDA tensor" % (who, b))
        data = jpeg_bytes(f)
        if data is None:
            raise ValueError("%s: slot %d is an \"mjpeg\" slot: its frame is the encoded bytes (bytes, a 1-D uint8 "
                             "numpy array or CPU tensor), got %s" % (who, b, type(f).__name__))
        if len(data) > self._jmax[b]:
            raise ValueError("%s: slot %d takes encoded frames of at most max_frame_bytes = %d bytes, got %d"
                             % (who, b, self._jmax[b], len(data)))
        h = jpeg_parse(data)
        if h.status:
            raise ValueError("%s: slot %d is a JPEG the device decoder does not take: %s"
                             % (who, b, _lib.JPEG_REFUSALS.get(h.status, h.status)))
        if (h.out_h, h.out_w) != tuple(self._slot_hw[b]):
            raise ValueError("%s: slot %d decodes to %d x %d, its frame_hw is %s"
                             % (who, b, h.out_h, h.out_w, tuple(self._slot_hw[b])))
        if torch.is_tensor(f):
            return f.contiguous(), h
        with warnings.catch_warnings():                  # read-only bytes: only ever the source of a copy
            warnings.simplefilter("ignore")
            return torch.from_numpy(data), h

    def _prepare(self, encoded):
        """cp_jpeg_slots_prepare of one call into the host block: encoded[s] is (bytes, header) or None (skipped)."""
        S = self.slots
        hs = (_lib.CpJpegHeader * S)()
        nbytes = np.zeros(S, np.int64)
        for s, e in enumerate(encoded):
            if e is not None:
                hs[s], nbytes[s] = e[1], e[0].numel()
        p64 = ctypes.POINTER(ctypes.c_int64)
        _lib.check(self.L.cp_jpeg_slots_prepare(S, self._jhw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                                self._jmax.ctypes.data_as(p64), 0, hs, nbytes.ctypes.data_as(p64),
                                                self._jout.ctypes.data_as(p64),
                                                self._jblock_host.ctypes.data_as(ctypes.c_void_p)),
                   "cp_jpeg_slots_prepare")

    def _upload_encoded(self, frames):
        """The block and the encoded frames of one call copied in (before the replay); returns frames with the MJPEG
        slots' entries None, so that only the other slots' frames are copied as they are."""
        enc = [frames[b] if b in self._mjpeg else None for b in range(self.slots)]
        self._prepare(enc)
        # pageable sources are staged before copy_ returns, without waiting for the device
        self._jblock.copy_(torch.from_numpy(self._jblock_host), non_blocking=True)
        for b, e in enumerate(enc):
            if e is not None:
                o = int(self._jbyte_offs[b])
                self._jbytes[o:o + e[0].numel()].copy_(e[0], non_blocking=True)
        return [None if b in self._mjpeg else f for b, f in enumerate(frames)]

    def _decode(self):
        """The slot decode of a step, ahead of the pre-process: every live MJPEG slot's BGR frame into its region."""
        if self._mjpeg:
            p32, p64 = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_int64)
            _lib.check(self.L.cp_jpeg_decode_slots_dev(
                _ptr(self._jblock), self.slots, self._jhw.ctypes.data_as(p32), self._jmax.ctypes.data_as(p64), 0,
                _ptr(self._jbytes), _ptr(self.frames), _ptr(self._jws), ctypes.c_size_t(self._jws.numel()),
                _ptr(self.decode_errors), _stream()), "cp_jpeg_decode_slots_dev")

    def _mask(self, n_valid, n, rows=None):
        """n_valid of a step's n rows zeroed for every slot (rows[r], or r) whose frame did not decode exactly."""
        if self._mjpeg:
            _lib.check(self.L.cp_jpeg_mask_counts_dev(_ptr(self.decode_errors), _ptr(rows), n,
                                                      self.streams // self.slots, _ptr(n_valid), _stream()),
                       "cp_jpeg_mask_counts_dev")

    # ---- launches the steps share ------------------------------------------------------------------------------------
    def _preprocess(self, out, start=None, prev=None):
        """The pre-process of every slot into out [S,3,h,w]; with start flags, a starting slot's input also goes to
        prev."""
        L, S, (ih, iw) = self.L, self.slots, out.shape[2:]
        if self._table:
            _lib.check(L.cp_preprocess_slots_ragged_dev(_ptr(self.frames), _ptr(self.table), self._fmt, S, ih, iw,
                                                        self._mean, self._std, _ptr(start), _ptr(out), _ptr(prev),
                                                        _stream()), "cp_preprocess_slots_ragged_dev")
        else:
            H, W = self.frame_hw
            _lib.check(L.cp_preprocess_slots_dev(_ptr(self.frames), self._fmt, S, H, W, ih, iw, None, self._mean,
                                                 self._std, _ptr(start), _ptr(out), _ptr(prev), _stream()),
                       "cp_preprocess_slots_dev")

    def _preprocess_rows(self, n, out, start=None, store=None, prev=None):
        """The pre-process of the n live rows (slot rows[k] into out[k]); with store and prev, the previous-frame
        exchange through the per-slot store."""
        ih, iw = out.shape[2:]
        _lib.check(self.L.cp_preprocess_slots_rows_dev(_ptr(self.frames), _ptr(self.table), self._fmt, _ptr(self.rows), n,
                                                       ih, iw, self._mean, self._std, _ptr(start), _ptr(store), _ptr(out),
                                                       _ptr(prev), _stream()), "cp_preprocess_slots_rows_dev")

    def _gather(self, src, dst, rows, m):
        """dst[i] = src[m[i]] (zeros where m[i] < 0) for i < rows, whole rows of src's first axis."""
        _lib.check(self.L.cp_gather_rows_dev(_ptr(src), _ptr(dst), src[0].numel() * src.element_size(), rows, _ptr(m),
                                             _stream()), "cp_gather_rows_dev")

    def _rows_view(self, t, n):
        """The first rows of a buffer of the plan's lead axes, as lead(n) + inner (a step of n live slots)."""
        lead = self.eng._lead(n)
        inner = tuple(t.shape[len(lead):])
        return t.view(-1)[:int(np.prod(lead + inner))].view(lead + inner)

    # ---- the call ----------------------------------------------------------------------------------------------------
    def _control(self, live, start):
        """The control block of a step over the slots `live` (in row order), start: int32 [S] (slots that start)."""
        S, MS = self.slots, self.streams
        M, n = MS // S, len(live)
        rows = np.zeros(S, np.int32)
        rows[:n] = live
        ids = np.zeros(MS, np.int32)
        ids[:M * n] = [m * S + i for m in range(M) for i in live]
        inv = np.full(MS, -1, np.int32)
        inv[ids[:M * n]] = np.arange(M * n, dtype=np.int32)
        return np.concatenate([np.tile(start, M), rows, ids, inv]).astype(np.int32)

    def _camera_rows(self, camera_matrix):
        """The meta rows of a call's camera_matrix ([3,3] for every slot or [S,3,3], a numpy array or a CPU tensor):
        every slot's row with its camera fields replaced, or None when it is None.  Refused before any device work: a
        graph built with distortion= (its undistortion maps were built from the build-time cameras), another shape, a
        non-finite value, a CUDA tensor."""
        if camera_matrix is None:
            return None
        who, S = type(self).__name__, self.slots
        if self._distorted:
            raise ValueError("%s was built with distortion=: its undistortion maps come from the cameras it was built "
                             "with, so it takes no per-step camera_matrix; build a graph for the new cameras" % who)
        if torch.is_tensor(camera_matrix):
            if camera_matrix.device.type != "cpu":
                raise ValueError("%s: camera_matrix is read on the host: pass a numpy array or a CPU tensor, got a "
                                 "tensor on %s" % (who, camera_matrix.device))
            camera_matrix = camera_matrix.numpy()
        try:
            cam = np.asarray(camera_matrix, np.float64)
        except (TypeError, ValueError):
            cam = None
        if cam is None or cam.shape not in ((3, 3), (S, 3, 3)):
            raise ValueError("%s: camera_matrix must be [3,3] or one [3,3] per slot ([%d,3,3]), got %s"
                             % (who, S, type(camera_matrix).__name__ if cam is None else cam.shape))
        if not np.isfinite(cam).all():
            raise ValueError("%s: camera_matrix holds a non-finite value" % who)
        rows = self._meta_host.copy()
        rows[:, 5:14] = np.broadcast_to(cam.reshape(-1, 9), (S, 9))
        return rows

    def _camera_meta(self):
        """The device meta rows a per-step camera replaces: the network's rows (a tracking graph's also hold the tracker
        streams' rows, one per category)."""
        return self.meta

    def _set_cameras(self, rows):
        """One copy of the meta rows `rows` (_camera_rows) to the device, on the current stream ahead of the replay;
        they stay in force until the next camera_matrix."""
        dst = self._camera_meta()
        src = np.tile(rows, (dst.shape[0] // self.slots, 1))
        # a pageable source: staged before copy_ returns, without waiting for the device
        dst.copy_(torch.from_numpy(src), non_blocking=True)
        self._meta_host = rows

    def reset(self):
        """Forget every slot's tracks and previous frame: the next call starts a video in every slot (with idle slots:
        each slot's next live frame starts its video)."""
        self._fresh = True
        self._started = [False] * self.slots

    def _frames(self, frames):
        """The frames of one call, checked against the slots' shapes: one tensor, or one per slot (with idle slots: one
        per slot, None for an idle one)."""
        who = type(self).__name__
        if self._mjpeg and (not isinstance(frames, (list, tuple)) or len(frames) != self.slots):
            what = "%d entries" % len(frames) if isinstance(frames, (list, tuple)) else type(frames).__name__
            raise ValueError("%s has \"mjpeg\" slots: frames is a list of %d entries, the encoded bytes of each "
                             "\"mjpeg\" slot%s, got %s" % (who, self.slots, " (None for an idle slot)"
                                                             if self.idle_slots else "", what))
        if self.idle_slots and not isinstance(frames, (list, tuple)):
            if self.per_slot or not (torch.is_tensor(frames) or isinstance(frames, np.ndarray)):
                raise ValueError("%s was built with idle slots: frames is a list of %d frames (None for an idle slot)%s, "
                                 "got %s" % (who, self.slots, "" if self.per_slot else " or one uint8 %s array"
                                             % list(self.frame_shape), type(frames).__name__))
            frames = torch.from_numpy(frames) if isinstance(frames, np.ndarray) else frames
            if frames.dtype != torch.uint8 or tuple(frames.shape) != self.frame_shape:
                raise ValueError("%s: frames must be uint8 %s (%s), got %s %s" % (who, list(self.frame_shape),
                                                                                 self.pixel_format, frames.dtype,
                                                                                 tuple(frames.shape)))
            return list(frames)                         # every slot live
        if not self.per_slot and not self.idle_slots and not self._mjpeg:
            if isinstance(frames, np.ndarray):
                frames = torch.from_numpy(frames)
            if not torch.is_tensor(frames) or frames.dtype != torch.uint8 or tuple(frames.shape) != self.frame_shape:
                what = ("%s %s" % (frames.dtype, tuple(frames.shape))) if torch.is_tensor(frames) else type(frames).__name__
                raise ValueError("%s steps every slot at one frame size: frames must be uint8 %s (%s), got %s; idle "
                                 "slots and mixed sizes run through %s or a %s built with one frame_hw per slot"
                                 % (who, list(self.frame_shape), self.pixel_format, what, self._host_list, who))
            return [frames]
        if not isinstance(frames, (list, tuple)) or len(frames) != self.slots:
            what = "%d frames" % len(frames) if isinstance(frames, (list, tuple)) else type(frames).__name__
            raise ValueError("%s was built with %s: frames is a list of %d frames, got %s"
                             % (who, "idle slots" if self.idle_slots else "one frame_hw per slot", self.slots, what))
        out = []
        for b, f in enumerate(frames):
            if f is None:
                if self.idle_slots:
                    out.append(None)
                    continue
                raise ValueError("%s steps every slot: slot %d is idle; idle slots run through %s"
                                 % (who, b, self._host_list))
            if b in self._mjpeg:
                out.append(self._encoded(b, f))
                continue
            if isinstance(f, np.ndarray):
                f = torch.from_numpy(f)
            if not torch.is_tensor(f) or f.dtype != torch.uint8 or tuple(f.shape) != self._slot_shapes[b]:
                what = ("%s %s" % (f.dtype, tuple(f.shape))) if torch.is_tensor(f) else type(f).__name__
                raise ValueError("%s: slot %d takes uint8 %s frames (%s, frame_hw %s), got %s"
                                 % (who, b, list(self._slot_shapes[b]), self.pixel_format[b] if isinstance(
                                     self.pixel_format, list) else self.pixel_format, self._slot_hw[b], what))
            out.append(f)
        return out

    def _replay(self, frames, start=None, cameras=None):
        """Copies the checked frames of a call (and, when given, the start flags: int32 [S], and the meta rows of a
        camera_matrix: _camera_rows) and replays the step; with idle slots, _call_rows.  Returns self._out."""
        if cameras is not None:
            with torch.cuda.device(self.device):
                self._set_cameras(cameras)
        if self.idle_slots:
            return self._call_rows(frames, start)
        with torch.cuda.device(self.device):
            if self._mjpeg:
                frames = self._upload_encoded(frames)
            for dst, f in zip(self._slot_frames if self.per_slot else [self.frames.view(self.frame_shape)], frames):
                if f is not None:
                    dst.copy_(f, non_blocking=True)
            if start is not None:
                # one flag per tracker stream, the same in every category; a pageable source: staged before copy_
                # returns, without waiting for the device
                self.start.copy_(torch.from_numpy(np.tile(start, self.streams // self.slots)), non_blocking=True)
            self.graphs[self._parity].replay()
        self._parity = (self._parity + 1) % len(self.graphs)
        self._fresh = False
        return self._out

    def _call_rows(self, frames, start):
        """A call with idle slots: frames[i] None idles slot i.  With start flags (a tracking step), a live slot starts
        its video when it has not started since the graph was built or reset, or when start[i] (new_video); an idle slot
        is not stepped.  Copies the live frames and the control block, then replays the graph of the live count; with no
        live slot, zeros the outputs and launches no graph."""
        live = [i for i, f in enumerate(frames) if f is not None]
        with torch.cuda.device(self.device):
            if not live:
                for t in self._out:
                    t.zero_()
                return self._out
            if start is None:
                start = np.zeros(self.slots, np.int32)
            else:
                start = np.array([i in live and (bool(start[i]) or not self._started[i]) for i in range(self.slots)],
                                 np.int32)
            if self._mjpeg:
                frames = self._upload_encoded(frames)
            for i in live:
                if frames[i] is not None:
                    self._slot_frames[i].copy_(frames[i], non_blocking=True)
            # a pageable source: staged before copy_ returns, without waiting for the device
            self.ctrl.copy_(torch.from_numpy(self._control(live, start)), non_blocking=True)
            self.graphs[len(live) - 1].replay()
        for i in live:
            self._started[i] = True
        self._fresh = False
        return self._out


class DetectGraph(_SlotGraph):
    """run_batch of a detection model (CenterPose, no opt.tracking_task) replayed from a CUDA graph: `slots` cameras,
    each with a frame size, a pixel format and a camera matrix.  A step is the pre-process of every slot's frame and the
    network + decode + PnP (cp_infer) writing straight into the output buffers, captured once; a call is one copy per
    frame and one graph launch, and the host does not wait for the device.  g(frames) -> (poses [S,K,192], n_valid [S])
    int32: views of the graph's own buffers, overwritten by the next call.  Every step is bit for bit run_batch on the
    same frames by a detector whose plan holds S frames (run_batch reuses a larger plan once it has made one, and the
    split-K choice follows the plan's capacity): its array form with one frame_hw, its list form with one frame_hw per
    slot.

    det: an ObjectPoseDetector of a detection opt, any architecture and precision run_batch takes.  The graph holds its
    own copy of the plan and the model's weights (taken now) and its own buffers; det.run_batch may be called between
    graph calls.  Refused before any device work (ValueError or NotImplementedError; they run through run_batch or
    run()): a tracking opt (TrackGraph), test_scales other than [1], the keep_res / fix_short pre-process, and new_video /
    pre_dets on a call (a detection step keeps nothing from one frame to the next).  Several categories go through
    MultiCategoryDetectGraph.

    frame_hw, camera_matrix, pixel_format and the frames of a call are those of TrackGraph: one (H, W) for every slot
    (frames uint8 [S,H,W,3], or [S,3H/2,W] for "nv12" / "i420", [S,H,W,C] for a camera format, [S,H,W] for "gray" and
    the Bayer mosaics) or a list of S sizes (a
    list of S frames, packed into one device buffer and pre-processed through a frame table built now; pixel_format may
    then be a list of one name per slot); [3,3] or [S,3,3] cameras.  Frames may be in pinned host memory (keep them
    unchanged until the step's outputs are read) or on the device.

    idle_slots=True: a call takes a list of S entries, None for an idle camera (with one frame_hw, a uint8 [S, ...]
    array still means every slot live).  Every step is bit for bit run_batch(list) of the live frames with their
    cameras, scattered to their slots: an idle slot comes back with n_valid 0 and zero rows, and an all-idle call returns
    zeros and launches nothing.  One step is captured per live count L = 1..S (the network runs at batch L, as in
    run_batch, and split-K makes batch-L bits differ from batch-S bits); a call is one copy per live frame, one copy of an
    int32 control block (the row / slot maps) and one graph launch.

    distortion: the lens distortion of the cameras (lens.LensDistortion), one for every slot or a list of one per slot
    (None: an undistorted camera), as run_batch(distortion=) takes it.  The maps (lens.undistort_map) and a frame table
    with them are built with the graph, which then always pre-processes through the table; every step is bit for bit
    run_batch(..., distortion=) on the same frames.

    pixel_format "mjpeg" (one name, or in a per-slot list): an MJPEG camera, encoded baseline JPEG frames of the slot's
    decoded size (bytes, a 1-D uint8 numpy array or CPU tensor); a call then takes a list of S entries.  The step
    decodes them on the device first (cp_jpeg_decode_slots_dev) and is bit for bit run_batch(list,
    pixel_format="jpeg").  max_frame_bytes (one int or one per slot, default H * W * 3) caps a slot's encoded size.  A
    frame the header parser refuses, of another decoded size or over max_frame_bytes is a ValueError naming the slot;
    a bitstream error sets the slot's word in decode_errors (int32 [S], device) and its n_valid to 0 for that step."""

    _host_list = "run_batch(list) of the live frames"

    def __init__(self, det, slots, frame_hw, camera_matrix, pixel_format="bgr", idle_slots=False, distortion=None,
                 max_frame_bytes=None):
        from .detector import MultiCategoryDetector, ObjectPoseDetector
        if isinstance(det, MultiCategoryDetector):
            raise NotImplementedError("DetectGraph detects one category; several run through a MultiCategoryDetectGraph")
        if not isinstance(det, ObjectPoseDetector):
            raise NotImplementedError("DetectGraph takes an ObjectPoseDetector, got %s" % type(det).__name__)
        self._build(det, slots, frame_hw, camera_matrix, pixel_format, idle_slots, distortion, max_frame_bytes)

    def _refuse(self, opt, who):
        if getattr(opt, "tracking_task", False):
            raise ValueError("%s runs a detection model; a tracking model (opt.tracking_task) runs through %s"
                             % (who, "MultiCategoryTrackGraph" if who.startswith("MultiCategory") else "TrackGraph"))
        if [float(v) for v in getattr(opt, "test_scales", [1.0])] != [1.0]:
            raise NotImplementedError("%s runs at test_scales=[1]; multi-scale detection runs through run()" % who)
        if getattr(opt, "fix_short", 0) > 0 or not getattr(opt, "fix_res", True):
            raise NotImplementedError("%s pre-processes in the fix_res mode only, as run_batch(list); keep_res and "
                                      "fix_short run through run()" % who)

    def _steps(self):
        return (0,)

    def _buffers(self, opt, meta, trans):
        S, MS, dev, lead = self.slots, self.streams, self.device, self.eng._lead(self.slots)
        self.x = torch.zeros((S, 3, opt.input_h, opt.input_w), dtype=torch.float32, device=dev)
        K = (self.prm[0] if isinstance(self.prm, list) else self.prm).K
        self.poses = torch.zeros(lead + (K, _lib.CP_POSE_RECORD), dtype=torch.float32, device=dev)
        self.n_valid = torch.zeros(lead, dtype=torch.int32, device=dev)
        if self.idle_slots:                              # the step's compact rows, before the scatter to the slots
            self.poses_rows, self.n_valid_rows = torch.zeros_like(self.poses), torch.zeros_like(self.n_valid)
        out_lead = (S,) if self.categories is None else (MS // S, S)
        self._out = (self.poses.view(out_lead + self.poses.shape[-2:]), self.n_valid.view(out_lead))

    def _step(self, p):
        """The launches of one step: the pre-process of every slot and the network + decode + PnP into the outputs; with
        idle slots, the step of p live slots (_step_rows)."""
        with torch.cuda.device(self.device):
            if self.idle_slots:
                return self._step_rows(p)
            self._decode()
            self._preprocess(self.x)
            self.eng.infer(self.x, self.meta, self.prm, poses=self.poses, n_valid=self.n_valid)
            self._mask(self.n_valid, self.slots)

    def _step_rows(self, n):
        """A step of n live slots: the row-mapped pre-process, the gather of the live rows' meta rows, the network at
        batch n into the compact rows and their scatter to the slots (zeros for idle slots).  Which slots are live is
        data in the control block; n fixes the shapes."""
        MS = self.streams
        self._decode()
        self._preprocess_rows(n, self.x)
        self._gather(self.meta, self.meta_rows, n, self.rows)
        self.eng.infer(self.x[:n], self.meta_rows[:n], self.prm, poses=self._rows_view(self.poses_rows, n),
                       n_valid=self._rows_view(self.n_valid_rows, n))
        self._mask(self._rows_view(self.n_valid_rows, n), n, self.rows)
        rec = self.poses.shape[-2:]
        self._gather(self.poses_rows.view((MS,) + rec), self.poses.view((MS,) + rec), MS, self.inv)
        self._gather(self.n_valid_rows.view(MS, 1), self.n_valid.view(MS, 1), MS, self.inv)

    def __call__(self, frames, new_video=None, pre_dets=None, camera_matrix=None):
        """The next frame of every camera -> (poses [S,K,192], n_valid [S]) ([M,S,...] in MultiCategoryDetectGraph):
        views of the graph's own buffers, overwritten by the next call.  frames: one array (one frame_hw) or a list of
        one frame per slot (one frame_hw per slot, or idle slots: None for an idle camera).  camera_matrix: None (the
        cameras in force), or [3,3] / [S,3,3] (numpy or a CPU tensor), the cameras of this step and the later ones
        (cameras whose intrinsics change with focus, as phones report them per frame); every step is run_batch with the
        cameras in force.  A graph built with distortion= refuses it."""
        if new_video is not None or pre_dets is not None:
            raise ValueError("%s keeps nothing from one frame to the next: new_video and pre_dets are tracking "
                             "arguments (TrackGraph, run_batch(track=True))" % type(self).__name__)
        frames = self._frames(frames)
        return self._replay(frames, cameras=self._camera_rows(camera_matrix))


class MultiCategoryDetectGraph(DetectGraph):
    """DetectGraph over a MultiCategoryDetector: its M categories detect in the same `slots` cameras, one pre-process of
    the shared frames and one multi-model network + decode call (cp_infer_multi; cp_infer for M = 1) per step, each
    category with its own visible_thresh and balance coefficient.  Every step's (poses [M,S,K,192], n_valid [M,S]), in
    mdet.categories order, are bit for bit those of mdet.run_batch on the same frames by a detector whose plan holds S
    frames (idle slots: mdet.run_batch(list) of the live frames, scattered to their slots).  The graph owns its plan
    (every category's weights, copied from mdet now) and buffers; mdet.run_batch may be called between graph calls.
    Refused as in DetectGraph; a MultiCategoryTracker goes to MultiCategoryTrackGraph."""

    _host_list = "MultiCategoryDetector.run_batch(list) of the live frames"

    def __init__(self, mdet, slots, frame_hw, camera_matrix, pixel_format="bgr", idle_slots=False, distortion=None,
                 max_frame_bytes=None):
        from .detector import MultiCategoryDetector, MultiCategoryTracker
        if isinstance(mdet, MultiCategoryTracker):
            raise ValueError("MultiCategoryDetectGraph needs a MultiCategoryDetector; a MultiCategoryTracker runs "
                             "through MultiCategoryTrackGraph")
        if not isinstance(mdet, MultiCategoryDetector):
            raise NotImplementedError("MultiCategoryDetectGraph takes a MultiCategoryDetector; one category's "
                                      "ObjectPoseDetector goes to DetectGraph")
        self._build(mdet, slots, frame_hw, camera_matrix, pixel_format, idle_slots, distortion, max_frame_bytes)
