"""`Tracker` -- the CenterPoseTrack state (/root/reference/src/lib/utils/tracker.py:15-302) on the device.

The reference keeps a Python list of dicts per video and runs association, a 32-state filterpy Kalman filter per
object, the scale pool and a second PnP on the host every frame; here the state of `streams` independent videos lives
in device memory and one native call (`cp_tracker_step`) advances all of them from the fixed-shape pose records that
`cp_decode_pnp` / `cp_infer` emit, with the greedy or (opt.hungarian) the optimal association.  `cp_tracker_render_ex`
draws the previous-frame heat maps (`BaseDetector._get_additional_inputs`, base_detector.py:150-388) straight into the
network's `pre_hm` / `pre_hm_hp` inputs, from the tracks, from the ground truth (opt.gt_pre_hm_hmhp /
gt_pre_hm_hmhp_first) or empty (opt.empty_pre_hm).  `cp_tracker_seed` is init_track with meta['pre_dets'].  The Python
side packs the reference's `pre_dets` dicts into seed records and rebuilds its dict structures for callers that want
them (`tracks`).
"""
import ctypes

import numpy as np
import torch

from . import _lib
from .engine import _VISIBLE, _ptr, _stream
from .graph import _SlotGraph


def _opt(opt, name, default):
    return getattr(opt, name, default)


def _stream_map(stream_ids, batch):
    """A host int32 [batch] stream map for the _ex entry points (NULL = the identity).  The library validates it."""
    if stream_ids is None:
        return None
    ids = [int(s) for s in stream_ids]
    if len(ids) != batch:
        raise ValueError("%d stream ids for a batch of %d" % (len(ids), batch))
    return (ctypes.c_int32 * batch)(*ids)


def track_to_dict(row):
    """One CP_TRACK_RECORD row -> the reference's track dict (the keys run() / the debugger / the evaluator read)."""
    from .detector import record_to_result
    L = _lib
    t = np.asarray(row, np.float32)
    d = record_to_result(t[:L.CP_POSE_RECORD])
    d["tracking_id"] = int(t[L.T_ID])
    d["age"] = int(t[L.T_AGE])
    d["active"] = int(t[L.T_ACTIVE])
    d["kps_fusion_mean"] = t[L.T_KPS_FUSION_MEAN:L.T_KPS_FUSION_MEAN + 16].astype(np.float64)
    d["kps_fusion_std"] = t[L.T_KPS_FUSION_STD:L.T_KPS_FUSION_STD + 16].astype(np.float64)
    d["kps_mean_kf"] = t[L.T_KPS_MEAN_KF:L.T_KPS_MEAN_KF + 16].astype(np.float64).reshape(8, 2)
    d["kps_std_kf"] = [float(v) for v in t[L.T_KPS_STD_KF:L.T_KPS_STD_KF + 16]]
    d["obj_scale_kf"] = t[L.T_OBJ_SCALE_KF:L.T_OBJ_SCALE_KF + 3].astype(np.float64)
    d["obj_scale_uncertainty_kf"] = t[L.T_OBJ_SCALE_UNC_KF:L.T_OBJ_SCALE_UNC_KF + 3].astype(np.float64)
    d["pnp2_status"] = int(t[L.T_PNP2_STATUS])
    d["in_boxes"] = bool(int(t[L.T_IN_BOXES]))
    d["kps_conf_avg_kf"] = float(t[L.T_CONF_AVG])
    if d["pnp2_status"] == L.PNP_OK:
        d["kps_pnp_kf"] = t[L.T_KPS_PNP_KF:L.T_KPS_PNP_KF + 18].astype(np.float64).reshape(9, 2)
        d["kps_3d_cam_kf"] = t[L.T_KPS_3D_CAM_KF:L.T_KPS_3D_CAM_KF + 27].astype(np.float64).reshape(9, 3)
    return d


def tracks_to_results(rows, n, width, height):
    """[T,320] rows of one stream -> (results list of dicts, boxes list of tuples) shaped like Tracker.step's return
    (tracker.py:271-295): a box = (kps_pnp_kf, kps_3d_cam_kf, obj_scale, kps_ori_kf, track)."""
    res = [track_to_dict(rows[i]) for i in range(int(n))]
    boxes = []
    for d in res:
        if d["in_boxes"] and "kps_pnp_kf" in d:
            kp = np.asarray(d["kps"], np.float64).reshape(-1, 2)
            po = np.vstack([kp.mean(0, keepdims=True), kp]).copy()
            po[:, 0] /= width
            po[:, 1] /= height
            d["kps_ori_kf"] = po
            boxes.append((d["kps_pnp_kf"], d["kps_3d_cam_kf"], np.array(d["obj_scale"]), po, d))
    return res, boxes


def _need(d, key):
    if key not in d:
        raise ValueError("pre_dets entry has no %r, which the reference tracker reads with these options" % key)
    return d[key]


def seed_records(dets, opt):
    """meta['pre_dets'] (a list of the reference's dicts) -> fp32 [len, CP_SEED_RECORD] (cp_seed_field layout).  A key
    the reference would read with these options but which the dict lacks raises ValueError naming it."""
    L = _lib
    kalman, scale_pool = bool(_opt(opt, "kalman", True)), bool(_opt(opt, "scale_pool", True))
    use_pnp = bool(_opt(opt, "use_pnp", True))
    out = np.zeros((len(dets), L.CP_SEED_RECORD), np.float32)

    def put(r, off, n, v):
        r[off:off + n] = np.asarray(v, np.float64).reshape(-1)[:n]
    for r, d in zip(out, dets):
        r[L.P_SCORE] = float(_need(d, "score"))
        bbox = _need(d, "bbox")
        put(r, L.P_BBOX, 4, bbox)
        r[L.P_CLS] = int(_need(d, "cls"))
        if "ct" in d:
            put(r, L.P_CT, 2, d["ct"])
            r[L.S_HAS_CT] = 1
        if kalman:                               # init_kf (tracker.py:55-79)
            put(r, L.S_KPS_FUSION_MEAN, 16, _need(d, "kps_fusion_mean"))
            put(r, L.S_KPS_FUSION_STD, 16, _need(d, "kps_fusion_std"))
            put(r, L.P_TRACKING_HP, 16, _need(d, "tracking_hp"))
        if scale_pool:                           # the scale pool (tracker.py:45-47)
            put(r, L.P_OBJ_SCALE_UNC, 3, _need(d, "obj_scale_uncertainty"))
        if scale_pool or use_pnp:
            put(r, L.P_OBJ_SCALE, 3, _need(d, "obj_scale"))
        if use_pnp and not kalman and scale_pool:
            put(r, L.P_KPS, 16, _need(d, "kps"))  # the second PnP reads track['kps'] without the filter (tracker.py:246)
        for key, off, n in (("kps", L.P_KPS, 16), ("kps_displacement_mean", L.P_KPS_DISP_MEAN, 16),
                            ("kps_heatmap_mean", L.P_KPS_HM_MEAN, 16), ("kps_heatmap_std", L.P_KPS_HM_STD, 16),
                            ("kps_heatmap_height", L.P_KPS_HM_HEIGHT, 8), ("kps_displacement_std", L.P_KPS_DISP_STD, 16),
                            ("obj_scale", L.P_OBJ_SCALE, 3), ("obj_scale_uncertainty", L.P_OBJ_SCALE_UNC, 3),
                            ("tracking", L.P_TRACKING, 2), ("tracking_hp", L.P_TRACKING_HP, 16),
                            ("kps_fusion_mean", L.S_KPS_FUSION_MEAN, 16), ("kps_fusion_std", L.S_KPS_FUSION_STD, 16),
                            ("kps_3d_cam", L.P_KPS_3D_CAM, 27), ("kps_pnp", L.P_KPS_PNP, 18)):
            if key in d:
                put(r, off, n, d[key])
        if "location" in d and "quaternion_xyzw" in d:    # a dict that already went through pnp_shell
            r[L.P_STATUS] = L.PNP_OK
            put(r, L.P_LOCATION, 3, d["location"])
            put(r, L.P_QUAT, 4, d["quaternion_xyzw"])
            if "projected_cuboid" in d:
                put(r, L.P_PROJ_CUBOID, 16, d["projected_cuboid"])
        if "kps_gt" in d:
            put(r, L.S_KPS_GT, 18, d["kps_gt"])
            r[L.S_HAS_KPS_GT] = 1
        if "kps_pnp_kf" in d:
            put(r, L.S_KPS_PNP_KF, 18, d["kps_pnp_kf"])
            r[L.S_HAS_KPS_PNP_KF] = 1
    return out


def _tracker_config(opt, cat, streams, max_tracks, device_index):
    """cp_tracker_config of category `cat` (its visible_thresh and opt.conf_border[cat])."""
    border = _opt(opt, "conf_border", {cat: [3, 9]})
    border = border[cat] if isinstance(border, dict) else border
    cfg = _lib.CpTrackerConfig()
    cfg.streams, cfg.max_tracks = streams, max_tracks
    cfg.kalman = int(bool(_opt(opt, "kalman", True)))
    cfg.scale_pool = int(bool(_opt(opt, "scale_pool", True)))
    cfg.use_pnp = int(bool(_opt(opt, "use_pnp", True)))
    cfg.hps_uncertainty = int(bool(_opt(opt, "hps_uncertainty", True)))
    cfg.max_age = int(_opt(opt, "max_age", 5))
    cfg.visible_thresh = _VISIBLE[cat]
    cfg.opencv_return = int(bool(_opt(opt, "show_axes", False)))
    cfg.render_hm_mode = int(_opt(opt, "render_hm_mode", 1))
    cfg.render_hmhp_mode = int(_opt(opt, "render_hmhp_mode", 2))
    cfg.device = device_index
    cfg.new_thresh = float(_opt(opt, "new_thresh", 0.3))
    cfg.pre_thresh = float(_opt(opt, "pre_thresh", -1))
    cfg.R = float(_opt(opt, "R", 20))
    cfg.conf_lo, cfg.conf_hi = float(border[0]), float(border[1])
    cfg.hungarian = int(bool(_opt(opt, "hungarian", False)))
    return cfg


class Tracker(object):
    """`streams` video streams of opt.c, or, with `categories` (a list of category names), `streams` slots of every
    category in one tracker (cp_tracker_create_multi): tracker stream m * streams + s is slot s of categories[m], with
    that category's visible_thresh and opt.conf_border[category] (when conf_border is a dict).  The device entry points
    then address all len(categories) * streams streams (self.streams), one step advancing every one of them."""

    def __init__(self, opt, streams=1, device=None, max_tracks=_lib.CP_MAX_K, categories=None):
        self.L = _lib.load()
        self.opt = opt
        self.max_tracks = int(max_tracks)
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.categories = list(categories) if categories is not None else [_opt(opt, "c", "chair")]
        if not 1 <= len(self.categories) <= _lib.CP_MAX_MODELS:
            raise ValueError("Tracker: 1..%d categories, got %d" % (_lib.CP_MAX_MODELS, len(self.categories)))
        for c in self.categories if categories is not None else ():
            if c not in _VISIBLE:
                raise ValueError("Tracker: unknown category '%s' (cuboid_pnp_shell.py:59-66)" % c)
        self.slots = int(streams)                        # streams per category
        self.streams = self.slots * len(self.categories)
        cfgs = [_tracker_config(opt, c, self.slots, self.max_tracks, self.device.index) for c in self.categories]
        self._cfg = cfgs[0]
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            if categories is None:
                rc = self.L.cp_tracker_create(ctypes.byref(cfgs[0]), ctypes.byref(h))
            else:
                rc = self.L.cp_tracker_create_multi((_lib.CpTrackerConfig * len(cfgs))(*cfgs), len(cfgs), ctypes.byref(h))
            _lib.check(rc, "cp_tracker_create")
        self._h = h
        self.meta = None
        self._rows = None          # host copy of the latest step: (rows [B,T,320], n [B])
        self._dev = None           # device tensors of the latest step
        self._dicts = None
        # per stream, since the latest seeding and before the next step: None (not seeded), or the missing key that the
        # reference would raise on when drawing these seeds from the tracks (or "" when none is missing), and whether
        # every seed carries 'kps_gt'
        self._seeded = [None] * self.streams
        self._seeded_gt = [False] * self.streams

    def close(self):
        if getattr(self, "_h", None):
            self.L.cp_tracker_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- reference surface -------------------------------------------------------------------------------------
    def reset(self, index=-1):
        """Tracker.reset (tracker.py:50-52)."""
        with torch.cuda.device(self.device):
            _lib.check(self.L.cp_tracker_reset(self._h, int(index), _stream()), "cp_tracker_reset")
        self._rows = self._dev = self._dicts = None
        for b in range(self.streams):
            if index < 0 or b == index:
                self._seeded[b], self._seeded_gt[b] = None, False

    def init_track(self, meta):
        """Tracker.init_track (tracker.py:21-48) for stream 0: with meta['pre_dets'] the stream is reset and one track
        is started per dict with score > new_thresh (ground-truth seeding, eval_video_official.py:422-456)."""
        self.meta = meta
        if meta is not None and "pre_dets" in meta:
            self.seed([meta["pre_dets"]] + [None] * (self.streams - 1))

    def seed(self, pre_dets):
        """init_track with pre_dets for several streams: pre_dets[b] is the list of dicts for stream b, or None to leave
        stream b untouched (one cp_tracker_seed_ex call over the streams that are seeded)."""
        pre_dets = list(pre_dets)
        if len(pre_dets) > self.streams:
            raise ValueError("%d seed lists for a tracker of %d streams" % (len(pre_dets), self.streams))
        ids = [b for b, p in enumerate(pre_dets) if p is not None]
        B = len(ids)
        if B == 0:
            return
        S = max(1, max(len(pre_dets[b]) for b in ids))
        if S > self.max_tracks:
            raise ValueError("%d seeds exceed max_tracks = %d" % (S, self.max_tracks))
        recs = np.zeros((B, S, _lib.CP_SEED_RECORD), np.float32)
        n = np.full(B, -1, np.int32)
        hmhp = int(_opt(self.opt, "render_hmhp_mode", 2))
        filt = bool(_opt(self.opt, "kalman", True)) or bool(_opt(self.opt, "scale_pool", True))
        pre_thresh, new_thresh = float(_opt(self.opt, "pre_thresh", -1)), float(_opt(self.opt, "new_thresh", 0.3))
        for i, b in enumerate(ids):
            dets = list(pre_dets[b])
            if dets:
                recs[i, :len(dets)] = seed_records(dets, self.opt)
            n[i] = len(dets)
            kept = [d for d in dets if float(d["score"]) > new_thresh]
            missing = ""
            for d in kept:
                if float(d["score"]) < pre_thresh:
                    continue
                if hmhp in (0, 1) and "kps_ori" not in d:
                    missing = "kps_ori"
                elif hmhp in (2, 3) and filt and "kps_pnp_kf" not in d and "kps_mean_kf" not in d:
                    missing = "kps_mean_kf"          # base_detector.py:245: the reference raises KeyError here
            self._seeded[b] = missing
            self._seeded_gt[b] = all("kps_gt" in d for d in kept)
        seeds = torch.from_numpy(recs).to(self.device)
        nt = torch.from_numpy(n).to(self.device)
        with torch.cuda.device(self.device):
            rc = self.L.cp_tracker_seed_ex(self._h, B, _stream_map(ids, B), _ptr(seeds), _ptr(nt), S, _stream())
        _lib.check(rc, "cp_tracker_seed")
        seeds._cp_keep = nt
        self._keep = seeds                       # the copy is stream-ordered; keep the buffers alive until the next call
        self._rows = self._dev = self._dicts = None

    @property
    def tracks(self):
        """The reference's `self.tracker.tracks` of stream 0 (list of dicts), rebuilt from the latest step."""
        if self._dicts is None:
            if self._dev is None:
                return []
            rows, n = self._host()
            self._dicts = [track_to_dict(rows[0, i]) for i in range(int(n[0]))]
        return self._dicts

    # ---- device entry points -----------------------------------------------------------------------------------
    def _host(self):
        if self._rows is None:
            tr, n = self._dev
            self._rows = (tr.cpu().numpy(), n.cpu().numpy())
        return self._rows

    def step_records(self, poses, n_valid, meta, out=None, stream_ids=None):
        """poses [B,K,192] / n_valid [B] / meta [B,16] CUDA tensors (as cp_infer emits them) -> (tracks [B,T,320],
        n_tracks [B]) CUDA tensors.  Stream b of the tracker consumes poses[b], or stream stream_ids[b] when a map is
        given; streams the map does not list are not stepped and keep their state untouched."""
        B, K, R = poses.shape
        if R != _lib.CP_POSE_RECORD or B > self.streams:
            raise ValueError("poses %s does not fit a tracker of %d streams" % (tuple(poses.shape), self.streams))
        for t, dt in ((poses, torch.float32), (n_valid, torch.int32), (meta, torch.float64)):
            if t.device != self.device or t.dtype != dt or not t.is_contiguous():
                raise ValueError("tracker inputs must be contiguous %s tensors on %s" % (dt, self.device))
        if out is None:
            out = (torch.empty((B, self.max_tracks, _lib.CP_TRACK_RECORD), dtype=torch.float32, device=self.device),
                   torch.empty((B,), dtype=torch.int32, device=self.device))
        with torch.cuda.device(self.device):
            rc = self.L.cp_tracker_step_ex(self._h, B, _stream_map(stream_ids, B), _ptr(poses), _ptr(n_valid), K, _ptr(meta),
                                           _ptr(out[0]), _ptr(out[1]), _stream())
        _lib.check(rc, "cp_tracker_step")
        self._dev, self._rows, self._dicts = out, None, None
        for s in (range(B) if stream_ids is None else stream_ids):
            self._seeded[s], self._seeded_gt[s] = None, False
        return out

    def render(self, meta, trans_input, inp_h, inp_w, out=None, modes=None, stream_ids=None):
        """Previous-frame heat maps of every stream: (pre_hm [B,1,h,w], pre_hm_hp [B,8,h,w]) fp32 CUDA.  modes: None
        (all drawn from the tracks) or one cp_render_mode per stream: RENDER_TRACKS, RENDER_GT (the ground-truth
        branch, on a stream seeded since its last step) or RENDER_EMPTY (opt.empty_pre_hm).  stream_ids: image b draws
        tracker stream stream_ids[b] (default: stream b)."""
        B = meta.shape[0]
        sid = list(range(B)) if stream_ids is None else [int(s) for s in stream_ids]
        if len(sid) != B:
            raise ValueError("render: %d stream ids for %d images" % (len(sid), B))
        mode_arr = None
        if modes is not None:
            modes = [int(m) for m in modes]
            if len(modes) != B:
                raise ValueError("render: %d modes for %d streams" % (len(modes), B))
            mode_arr = (ctypes.c_int32 * B)(*modes)
        for b, s in enumerate(sid):
            if not 0 <= s < self.streams:
                raise ValueError("render: stream id %d out of range 0..%d" % (s, self.streams - 1))
            m = modes[b] if modes is not None else _lib.RENDER_TRACKS
            if m == _lib.RENDER_GT and not (self._seeded[s] is not None and self._seeded_gt[s]):
                raise ValueError("the ground-truth render of stream %d needs tracks seeded from pre_dets with 'kps_gt'" % s)
            if m == _lib.RENDER_TRACKS and self._seeded[s]:
                raise ValueError("drawing the seeds of stream %d from the tracks reads %r, which a pre_dets entry lacks"
                                 % (s, self._seeded[s]))
        tr = torch.as_tensor(np.asarray(trans_input, np.float64).reshape(-1, 6)) if not torch.is_tensor(trans_input) else trans_input
        if tr.shape[0] == 1 and B > 1:
            tr = tr.expand(B, 6)
        tr = tr.to(self.device, torch.float64).contiguous()
        meta = meta.to(self.device, torch.float64).contiguous()
        if out is None:
            out = (torch.empty((B, 1, inp_h, inp_w), dtype=torch.float32, device=self.device),
                   torch.empty((B, 8, inp_h, inp_w), dtype=torch.float32, device=self.device))
        with torch.cuda.device(self.device):
            rc = self.L.cp_tracker_render_ex2(self._h, B, _stream_map(stream_ids, B), _ptr(meta), _ptr(tr), int(inp_h),
                                              int(inp_w), mode_arr, _ptr(out[0]), _ptr(out[1]), _stream())
        _lib.check(rc, "cp_tracker_render_ex")
        out[0]._cp_keep = (meta, tr)
        return out


class TrackGraph(_SlotGraph):
    """The array form of ObjectPoseDetector.run_batch(track=True) replayed from CUDA graphs: `slots` video slots with a
    pixel format and a camera each, every slot stepping on every call.  A step is the pre-process, the reset of the slots
    whose video starts, the previous-frame render, the network + decode + PnP and the tracker step, captured once; a call
    is one copy per frame buffer, one copy of the start flags and one graph launch, and the host does not wait for the
    device.  Every step's (tracks [S,T,320], n_tracks [S]) are bit for bit those of run_batch(track=True) on a fresh
    detector fed the same frames (with new_video as run_batch(list) takes it).

    The previous network input needs no copy: the step alternates between two input buffers, and the graph of odd steps
    is that of even steps with the two swapped.  A slot that starts a video (on the first call, after reset(), or with
    new_video[i]) has its network input written to the previous-frame buffer too, by the pre-process itself.

    det: an ObjectPoseDetector of a tracking opt (opt.tracking_task).  The graph holds its own copy of the plan and the
    model's weights (taken now), its own tracker and buffers: building it leaves det._slots untouched, and det.run_batch
    (track=True) and this graph may be called in any order, each keeping its own slot state.  Greedy or opt.hungarian
    association, opt.empty_pre_hm and the heat maps drawn from the tracks follow opt as in run_batch.  Refused (ValueError
    or NotImplementedError; they stay on run_batch): test_scales other than [1], the ground-truth heat maps
    (opt.gt_pre_hm_hmhp / gt_pre_hm_hmhp_first), pre_dets seeding, and idle slots unless idle_slots=True.  Several
    categories go through MultiCategoryTrackGraph; a detection model through DetectGraph (graph.py), which shares this
    graph's frame handling, capture and call.

    frame_hw: one (H, W) for every slot, or a list of S (H_s, W_s).  camera_matrix: [3,3] for every slot or [S,3,3].
      - One size: a call takes the frames as one array, uint8 [S,H,W,3] for pixel_format "bgr", [S,3H/2,W] for "nv12" /
        "i420" (H, W even), [S,H,W,C] for a camera format ("rgb24", "rgba", "bgra", "yuyv422", "uyvy422"), [S,H,W] for
        a sensor format ("gray", "bayer_rggb8", "bayer_bggr8", "bayer_gbrg8", "bayer_grbg8"), [S,3H/2,W] for a phone
        format ("nv21", "yv12", "nv12_full", "nv21_full", "i420_full", "yv12_full"); one copy and the uniform
        pre-process (cp_preprocess_slots_dev).
      - One size per slot: a call takes a list of S frames, uint8 [H_s,W_s,3] or [3H_s/2,W_s] (...), each copied into
        its own region of one packed device buffer; the step is that of run_batch(list, track=True) with every slot
        present, the pre-process reading a frame table built once now (cp_preprocess_slots_ragged_dev).  pixel_format
        may then be a list of one name per slot (cameras of different kinds): the table holds each slot's format and
        one launch converts every slot's frame in its own format; one name repeated is that name.
    Frames may be on the host (pinned memory keeps the copy asynchronous; the caller must not overwrite them until the
    step's outputs are read) or on the device.

    idle_slots=True: a call takes a list of S entries, a frame of that slot's size and format or None for an idle slot
    (with one frame_hw, a uint8 [S, ...] array still means every slot live).  Every step is bit for bit
    run_batch(list, track=True) of a fresh detector on the same list: an idle slot comes back with n_tracks 0 and zero
    rows, and its stream, tracks and previous frame are left as they were; a slot's first live frame (after building or
    reset()) starts its video, and new_video[i] restarts a live slot and is ignored on an idle one; an all-idle call
    returns zeros and launches nothing.  One step is captured per live count L = 1..S (the network runs at batch L, as
    in run_batch), so building costs S warm-up steps and S captures; a call is one copy per live frame, one copy of an
    int32 control block (start flags and the row / stream maps) and one graph launch.  Each slot's previous frame is
    kept in a per-slot store that the pre-process exchanges in place.

    distortion: the lens distortion of the cameras, one lens.LensDistortion for every slot or one per slot (None: an
    undistorted camera), as run_batch(track=True, distortion=) takes it.  The maps and a frame table with them are
    built with the graph, which then always pre-processes through the table; every step is bit for bit
    run_batch(..., track=True, distortion=) on the same frames."""

    _host_step = "run_batch(track=True)"              # where what the graph refuses runs
    _host_list = "run_batch(list, track=True)"

    def __init__(self, det, slots, frame_hw, camera_matrix, pixel_format="bgr", idle_slots=False, distortion=None,
                 max_frame_bytes=None):
        from .detector import ObjectPoseDetector
        if not isinstance(det, ObjectPoseDetector) or det._track_categories() is not None:
            raise NotImplementedError("TrackGraph tracks one category; several run through MultiCategoryTracker.run_batch "
                                      "or a MultiCategoryTrackGraph")
        self._build(det, slots, frame_hw, camera_matrix, pixel_format, idle_slots, distortion, max_frame_bytes)

    def _refuse(self, opt, who):
        if not getattr(opt, "tracking_task", False):
            raise ValueError("%s needs a tracking model (opt.tracking_task)" % who)
        if [float(v) for v in getattr(opt, "test_scales", [1.0])] != [1.0]:
            raise NotImplementedError("%s runs at test_scales=[1]; multi-scale tracking runs through run()" % who)
        if getattr(opt, "gt_pre_hm_hmhp", False) or getattr(opt, "gt_pre_hm_hmhp_first", False):
            raise NotImplementedError("%s draws the previous-frame heat maps from the tracks; the ground-truth heat maps "
                                      "(opt.gt_pre_hm_hmhp / gt_pre_hm_hmhp_first) run through %s" % (who, self._host_step))

    def _steps(self):
        return (0, 1)                            # the input buffers swapped on odd steps

    def _buffers(self, opt, meta, trans):
        """The tracker of M x S streams (stream m * S + s: slot s of category m), the previous frames, the rendered heat
        maps and the outputs; every slot's meta row and affine repeated per category."""
        S, MS, dev = self.slots, self.streams, self.device
        M, ih, iw = MS // S, opt.input_h, opt.input_w
        self.tracker = Tracker(opt, streams=S, device=dev, categories=self.categories)
        if M > 1:                                        # the network's rows are category 0's: one buffer to update
            self.meta_all = torch.from_numpy(np.tile(meta, (M, 1))).to(dev)
            self.meta = self.meta_all[:S]
        else:
            self.meta_all = self.meta
        self.trans = torch.from_numpy(np.tile(trans, (M, 1))).to(dev)
        mode = _lib.RENDER_EMPTY if getattr(opt, "empty_pre_hm", False) else _lib.RENDER_TRACKS
        self.modes = torch.full((MS,), mode, dtype=torch.int32, device=dev)
        if self.idle_slots:
            self.store = torch.zeros((S, 3, ih, iw), dtype=torch.float32, device=dev)   # every slot's previous frame
            # the live rows' meta rows and affines of every category, gathered from the per-slot rows above
            self.meta_trk = torch.zeros((MS, _lib.CP_META_DOUBLES), dtype=torch.float64, device=dev)
            self.trans_trk = torch.zeros((MS, 6), dtype=torch.float64, device=dev)
        else:
            self.start = torch.ones((MS,), dtype=torch.int32, device=dev)
        self.x = [torch.zeros((S, 3, ih, iw), dtype=torch.float32, device=dev) for _ in range(2)]
        lead = self.eng._lead(S)                         # the plan's per-model axes: (S,) or (M, S)
        self.pre_hm = torch.zeros(lead + (1, ih, iw), dtype=torch.float32, device=dev)
        self.pre_hm_hp = torch.zeros(lead + (8, ih, iw), dtype=torch.float32, device=dev)
        K = (self.prm[0] if isinstance(self.prm, list) else self.prm).K
        self.poses = torch.zeros(lead + (K, _lib.CP_POSE_RECORD), dtype=torch.float32, device=dev)
        self.n_valid = torch.zeros(lead, dtype=torch.int32, device=dev)
        self.tracks = torch.zeros((MS, self.tracker.max_tracks, _lib.CP_TRACK_RECORD), dtype=torch.float32, device=dev)
        self.n_tracks = torch.zeros((MS,), dtype=torch.int32, device=dev)
        if self.idle_slots:                              # the step's compact rows, before the scatter to the slots
            self.tracks_rows, self.n_tracks_rows = torch.zeros_like(self.tracks), torch.zeros_like(self.n_tracks)
        out_lead = (S,) if self.categories is None else (M, S)
        self._out = (self.tracks.view(out_lead + self.tracks.shape[1:]), self.n_tracks.view(out_lead))

    def _camera_meta(self):
        return self.meta_all

    def _warmed(self):
        if self.idle_slots:                      # the warm-ups stepped every stream: start from nothing
            self.tracker.reset()
            torch.cuda.synchronize(self.device)

    def _step(self, p):
        """The launches of one step: network input in x[p], previous frames in x[1 - p]; with idle slots, the step of p
        live slots (_step_rows)."""
        if self.idle_slots:
            return self._step_rows(p)
        L, st, h = self.L, _stream(), self.tracker._h
        MS, (ih, iw), cur, prev = self.streams, self.x[p].shape[2:], self.x[p], self.x[1 - p]
        with torch.cuda.device(self.device):
            _lib.check(L.cp_tracker_reset_dev(h, MS, _ptr(self.start), st), "cp_tracker_reset_dev")
            self._decode()
            self._preprocess(cur, self.start, prev)
            _lib.check(L.cp_tracker_render_dev(h, MS, _ptr(self.meta_all), _ptr(self.trans), ih, iw, _ptr(self.modes),
                                               _ptr(self.pre_hm), _ptr(self.pre_hm_hp), st), "cp_tracker_render_dev")
            self.eng.infer(cur, self.meta, self.prm, prev, self.pre_hm, self.pre_hm_hp, poses=self.poses,
                           n_valid=self.n_valid)
            self._mask(self.n_valid, self.slots)
            _lib.check(L.cp_tracker_step(h, MS, _ptr(self.poses), _ptr(self.n_valid), self.poses.shape[-2],
                                         _ptr(self.meta_all), _ptr(self.tracks), _ptr(self.n_tracks), st), "cp_tracker_step")

    def _step_rows(self, n):
        """The launches of a step of n live slots: the reset of the starting streams, the row-mapped pre-process with
        the previous-frame exchange, the gathers of the live rows' meta rows and affines, the render, the network at
        batch n, the tracker step over the live streams and the scatter of their tracks to the slots (zeros for idle
        slots).  Which slots are live is data in the control block; n fixes the shapes."""
        L, st, h, MS = self.L, _stream(), self.tracker._h, self.streams
        M, cur, prev = MS // self.slots, self.x[0], self.x[1]
        (ih, iw), Mn = cur.shape[2:], M * n
        pre_hm, pre_hm_hp = self._rows_view(self.pre_hm, n), self._rows_view(self.pre_hm_hp, n)
        poses, n_valid = self._rows_view(self.poses, n), self._rows_view(self.n_valid, n)
        with torch.cuda.device(self.device):
            _lib.check(L.cp_tracker_reset_dev(h, MS, _ptr(self.start), st), "cp_tracker_reset_dev")
            self._decode()
            self._preprocess_rows(n, cur, self.start, self.store, prev)
            self._gather(self.meta, self.meta_rows, n, self.rows)
            self._gather(self.meta_all, self.meta_trk, Mn, self.ids)
            self._gather(self.trans, self.trans_trk, Mn, self.ids)
            _lib.check(L.cp_tracker_render_dev2(h, Mn, _ptr(self.ids), _ptr(self.meta_trk), _ptr(self.trans_trk), ih, iw,
                                                _ptr(self.modes), _ptr(pre_hm), _ptr(pre_hm_hp), st),
                       "cp_tracker_render_dev2")
            self.eng.infer(cur[:n], self.meta_rows[:n], self.prm, prev[:n], pre_hm, pre_hm_hp, poses=poses,
                           n_valid=n_valid)
            self._mask(n_valid, n, self.rows)
            _lib.check(L.cp_tracker_step_dev(h, Mn, _ptr(self.ids), _ptr(poses), _ptr(n_valid), poses.shape[-2],
                                             _ptr(self.meta_trk), _ptr(self.tracks_rows), _ptr(self.n_tracks_rows), st),
                       "cp_tracker_step_dev")
            self._gather(self.tracks_rows, self.tracks, MS, self.inv)
            self._gather(self.n_tracks_rows.view(MS, 1), self.n_tracks.view(MS, 1), MS, self.inv)

    def __call__(self, frames, new_video=None, pre_dets=None, camera_matrix=None):
        """The next frame of every slot -> (tracks [S,T,320], n_tracks [S]) ([M,S,...] in MultiCategoryTrackGraph):
        views of the graph's own buffers, overwritten by the next call.  frames: one array (one frame_hw) or a list of
        one frame per slot (one frame_hw per slot).  new_video: None or one bool per slot (slot i starts a new video
        with this frame).  camera_matrix: None (the cameras in force), or [3,3] / [S,3,3] (numpy or a CPU tensor), the
        cameras of this step and the later ones, read by the network's PnP and the tracker's alike; every step is
        run_batch(track=True) with the cameras in force.  A graph built with distortion= refuses it."""
        who = type(self).__name__
        if pre_dets is not None:
            raise NotImplementedError("%s does not seed tracks; pre_dets seeding runs through %s" % (who, self._host_step))
        frames = self._frames(frames)
        start = np.full(self.slots, int(self._fresh), np.int32)
        if new_video is not None:
            new_video = [bool(v) for v in new_video]
            if len(new_video) != self.slots:
                raise ValueError("%s: %d new_video entries for %d slots" % (who, len(new_video), self.slots))
            start |= np.array(new_video, np.int32)
        return self._replay(frames, start, self._camera_rows(camera_matrix))


class MultiCategoryTrackGraph(TrackGraph):
    """TrackGraph over a MultiCategoryTracker: its M categories track in the same `slots` video slots, and every step's
    (tracks [M,S,T,320], n_tracks [M,S]), in trk.categories order, are bit for bit those of trk.run_batch on the same
    frames (its array form with one frame_hw, its list form with every slot present with one frame_hw per slot).  The
    step is TrackGraph's: one pre-process of the shared frames, the reset of the M x S tracker streams of the slots that
    start a video, one render of every category's previous-frame heat maps, one multi-model network + decode call
    (cp_infer_multi_track) and one tracker step over the M x S streams, each category with its own visible_thresh, balance
    coefficient and opt.conf_border.

    The graph owns its plan (every category's weights, copied from trk now), its tracker and buffers: trk._slots is left
    untouched, and trk.run_batch and this graph may be called in any order.  Refused as in TrackGraph; several categories
    of one graph need a MultiCategoryTracker (a MultiCategoryDetector is not a tracking model).  idle_slots=True as in
    TrackGraph, bit for bit trk.run_batch(list) with None for the idle slots."""

    _host_step = "MultiCategoryTracker.run_batch"
    _host_list = "MultiCategoryTracker.run_batch(list)"

    def __init__(self, trk, slots, frame_hw, camera_matrix, pixel_format="bgr", idle_slots=False, distortion=None,
                 max_frame_bytes=None):
        from .detector import MultiCategoryDetector, MultiCategoryTracker
        if not isinstance(trk, MultiCategoryTracker):
            if isinstance(trk, MultiCategoryDetector):
                raise ValueError("MultiCategoryTrackGraph needs a MultiCategoryTracker; a MultiCategoryDetector is not a "
                                 "tracking model")
            raise NotImplementedError("MultiCategoryTrackGraph takes a MultiCategoryTracker; one category's "
                                      "ObjectPoseDetector goes to TrackGraph")
        self._build(trk, slots, frame_hw, camera_matrix, pixel_format, idle_slots, distortion, max_frame_bytes)
