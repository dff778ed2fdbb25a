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


class TrackGraph(object):
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
    categories go through MultiCategoryTrackGraph.

    frame_hw: one (H, W) for every slot, or a list of S (H_s, W_s).  camera_matrix: [3,3] for every slot or [S,3,3].
      - One size: a call takes the frames as one array, uint8 [S,H,W,3] for pixel_format "bgr", [S,3H/2,W] for "nv12" /
        "i420" (H, W even); one copy and the uniform pre-process (cp_preprocess_slots_dev).
      - One size per slot: a call takes a list of S frames, uint8 [H_s,W_s,3] or [3H_s/2,W_s], each copied into its own
        region of one packed device buffer; the step is that of run_batch(list, track=True) with every slot present, the
        pre-process reading a frame table built once now (cp_preprocess_slots_ragged_dev).
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
    kept in a per-slot store that the pre-process exchanges in place."""

    _host_step = "run_batch(track=True)"              # where what the graph refuses runs
    _host_list = "run_batch(list, track=True)"

    def __init__(self, det, slots, frame_hw, camera_matrix, pixel_format="bgr", idle_slots=False):
        from .detector import ObjectPoseDetector
        if not isinstance(det, ObjectPoseDetector) or det._track_categories() is not None:
            raise NotImplementedError("TrackGraph tracks one category; several run through MultiCategoryTracker.run_batch "
                                      "or a MultiCategoryTrackGraph")
        self._build(det, slots, frame_hw, camera_matrix, pixel_format, idle_slots)

    def _plan(self, det, S, ih, iw):
        """(plan, decode parameters, tracker, categories or None) of the graph: a copy of det's plan and weights."""
        from .engine import Engine, decode_params
        m = det.model
        eng = Engine(m._arch(), m.heads, m.head_conv, S, ih, iw, self.device.index, tracking=m.tracking_inputs,
                     tracking_task_gru=m.use_convGRU and m.tracking_task, precision=m.precision, reuse_activations=True)
        eng.load_state_dict(m.state_dict())
        return eng, decode_params(det.opt, test_scale=1.0), Tracker(det.opt, streams=S, device=self.device), None

    def _build(self, det, slots, frame_hw, camera_matrix, pixel_format, idle_slots=False):
        """Checks, buffers and the captured steps (two, or one per live count with idle_slots); everything that refuses
        comes before any device work."""
        from .detector import affine_from_center_scale, camera_per_frame
        from .engine import check_pixel_format, frame_shape, make_meta
        who, opt = type(self).__name__, det.opt
        if not getattr(opt, "tracking_task", False):
            raise ValueError("%s needs a tracking model (opt.tracking_task)" % who)
        if [float(v) for v in getattr(opt, "test_scales", [1.0])] != [1.0]:
            raise NotImplementedError("%s runs at test_scales=[1]; multi-scale tracking runs through run()" % who)
        if getattr(opt, "gt_pre_hm_hmhp", False) or getattr(opt, "gt_pre_hm_hmhp_first", False):
            raise NotImplementedError("%s draws the previous-frame heat maps from the tracks; the ground-truth heat maps "
                                      "(opt.gt_pre_hm_hmhp / gt_pre_hm_hmhp_first) run through %s" % (who, self._host_step))
        S = int(slots)
        if S < 1:
            raise ValueError("%s: slots must be >= 1, got %d" % (who, S))
        sizes, self.per_slot = _frame_sizes(frame_hw, S, who)
        self.idle_slots = bool(idle_slots)
        self.pixel_format = check_pixel_format(pixel_format)
        shapes = [frame_shape(h, w, pixel_format) for h, w in sizes]
        cams = np.stack(camera_per_frame(camera_matrix, S))
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
        self.eng, self.prm, self.tracker, self.categories = self._plan(det, S, ih, iw)
        M = 1 if self.categories is None else len(self.categories)
        MS = self.streams = M * S                        # tracker stream m * S + s: slot s of category m
        # every slot's row of run_batch: its fix_res c, s and meta row and the affine of its size, repeated per category
        meta, trans = np.zeros((S, _lib.CP_META_DOUBLES), np.float64), np.zeros((S, 6), np.float64)
        for b, (h, w) in enumerate(sizes):
            c, sc = np.array([w / 2., h / 2.], np.float32), float(max(h, w))
            meta[b] = make_meta(1, c, sc, w, h, cams[b]).numpy()[0]
            trans[b] = affine_from_center_scale(c, sc, iw, ih).reshape(6)
        self.meta = torch.from_numpy(meta).to(dev)                   # the network's rows, one per frame
        self.meta_all = self.meta if M == 1 else torch.from_numpy(np.tile(meta, (M, 1))).to(dev)
        self.trans = torch.from_numpy(np.tile(trans, (M, 1))).to(dev)
        mode = _lib.RENDER_EMPTY if getattr(opt, "empty_pre_hm", False) else _lib.RENDER_TRACKS
        self.modes = torch.full((MS,), mode, dtype=torch.int32, device=dev)
        self._mean = (ctypes.c_float * 3)(*[float(v) for v in opt.mean])
        self._std = (ctypes.c_float * 3)(*[float(v) for v in opt.std])
        self._fmt = {"bgr": _lib.CP_PIX_BGR, "nv12": _lib.CP_PIX_NV12, "i420": _lib.CP_PIX_I420}[self.pixel_format]
        if self.per_slot or self.idle_slots:                # a frame table (with idle slots: of S equal sizes too)
            n = [int(np.prod(s)) for s in self._slot_shapes]
            offs = np.concatenate([[0], np.cumsum(n)[:-1]]).astype(np.int64)
            self.frames = torch.zeros((int(sum(n)),), dtype=torch.uint8, device=dev)
            self._slot_frames = [self.frames[o:o + k].view(s) for o, k, s in zip(offs, n, self._slot_shapes)]
            self.table = torch.zeros((int(L.cp_preprocess_frame_table_bytes(S)),), dtype=torch.uint8, device=dev)
            hw = np.ascontiguousarray(sizes, np.int32)
            with torch.cuda.device(dev):
                _lib.check(L.cp_preprocess_frame_table(self.frames.numel(), offs.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                                       hw.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), self._fmt, S, ih,
                                                       iw, trans.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                       _ptr(self.table), _stream()), "cp_preprocess_frame_table")
        else:
            self.frames = torch.zeros(self.frame_shape, dtype=torch.uint8, device=dev)
        if self.idle_slots:
            # one int32 control block per call: start flags [M*S] (per tracker stream), rows [S] (the slot of each live
            # row), ids [M*S] (the tracker stream of each live row of each category) and inv [M*S] (the row of each
            # stream, or -1); a step at live count n reads the first n rows and M * n ids
            self.ctrl = torch.zeros((3 * MS + S,), dtype=torch.int32, device=dev)
            self.start, self.rows = self.ctrl[:MS], self.ctrl[MS:MS + S]
            self.ids, self.inv = self.ctrl[MS + S:2 * MS + S], self.ctrl[2 * MS + S:]
            self.store = torch.zeros((S, 3, ih, iw), dtype=torch.float32, device=dev)   # every slot's previous frame
            # the live rows' meta rows and affines, gathered from the per-slot rows above
            self.meta_rows = torch.zeros((S, _lib.CP_META_DOUBLES), dtype=torch.float64, device=dev)
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
        # the captured steps: p = 0, 1 (the input buffers swapped), or with idle slots p = every live count 1..S
        steps = range(1, S + 1) if self.idle_slots else (0, 1)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):            # warm-up outside the capture; the first call resets every slot
            for p in steps:
                if self.idle_slots:
                    self.ctrl.copy_(torch.from_numpy(self._control(list(range(p)), np.ones(S, np.int32))))
                self._step(p)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        if self.idle_slots:                      # the warm-ups stepped every stream: start from nothing
            self.tracker.reset()
            torch.cuda.synchronize(dev)
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

    def _step(self, p):
        """The launches of one step: network input in x[p], previous frames in x[1 - p]; with idle slots, the step of p
        live slots (_step_rows)."""
        if self.idle_slots:
            return self._step_rows(p)
        L, st, h = self.L, _stream(), self.tracker._h
        S, MS, (ih, iw), cur, prev = self.slots, self.streams, self.x[p].shape[2:], self.x[p], self.x[1 - p]
        with torch.cuda.device(self.device):
            _lib.check(L.cp_tracker_reset_dev(h, MS, _ptr(self.start), st), "cp_tracker_reset_dev")
            if self.per_slot:
                _lib.check(L.cp_preprocess_slots_ragged_dev(_ptr(self.frames), _ptr(self.table), self._fmt, S, ih, iw,
                                                            self._mean, self._std, _ptr(self.start), _ptr(cur),
                                                            _ptr(prev), st), "cp_preprocess_slots_ragged_dev")
            else:
                H, W = self.frame_hw
                _lib.check(L.cp_preprocess_slots_dev(_ptr(self.frames), self._fmt, S, H, W, ih, iw, None, self._mean,
                                                     self._std, _ptr(self.start), _ptr(cur), _ptr(prev), st),
                           "cp_preprocess_slots_dev")
            _lib.check(L.cp_tracker_render_dev(h, MS, _ptr(self.meta_all), _ptr(self.trans), ih, iw, _ptr(self.modes),
                                               _ptr(self.pre_hm), _ptr(self.pre_hm_hp), st), "cp_tracker_render_dev")
            self.eng.infer(cur, self.meta, self.prm, prev, self.pre_hm, self.pre_hm_hp, poses=self.poses,
                           n_valid=self.n_valid)
            _lib.check(L.cp_tracker_step(h, MS, _ptr(self.poses), _ptr(self.n_valid), self.poses.shape[-2],
                                         _ptr(self.meta_all), _ptr(self.tracks), _ptr(self.n_tracks), st), "cp_tracker_step")

    def _step_rows(self, n):
        """The launches of a step of n live slots: the reset of the starting streams, the row-mapped pre-process with
        the previous-frame exchange, the gathers of the live rows' meta rows and affines, the render, the network at
        batch n, the tracker step over the live streams and the scatter of their tracks to the slots (zeros for idle
        slots).  Which slots are live is data in the control block; n fixes the shapes."""
        L, st, h, S, MS = self.L, _stream(), self.tracker._h, self.slots, self.streams
        M, cur, prev = MS // S, self.x[0], self.x[1]
        (ih, iw), Mn, lead = cur.shape[2:], M * n, self.eng._lead(n)

        def view(t):                          # the first rows of a buffer of the plan's lead axes, as lead(n) + inner
            inner = tuple(t.shape[len(lead):])
            return t.view(-1)[:int(np.prod(lead + inner))].view(lead + inner)

        def gather(src, dst, rows, m):
            _lib.check(L.cp_gather_rows_dev(_ptr(src), _ptr(dst), src[0].numel() * src.element_size(), rows, _ptr(m),
                                            st), "cp_gather_rows_dev")
        pre_hm, pre_hm_hp, poses, n_valid = view(self.pre_hm), view(self.pre_hm_hp), view(self.poses), view(self.n_valid)
        with torch.cuda.device(self.device):
            _lib.check(L.cp_tracker_reset_dev(h, MS, _ptr(self.start), st), "cp_tracker_reset_dev")
            _lib.check(L.cp_preprocess_slots_rows_dev(_ptr(self.frames), _ptr(self.table), self._fmt, _ptr(self.rows), n,
                                                      ih, iw, self._mean, self._std, _ptr(self.start), _ptr(self.store),
                                                      _ptr(cur), _ptr(prev), st), "cp_preprocess_slots_rows_dev")
            gather(self.meta, self.meta_rows, n, self.rows)
            gather(self.meta_all, self.meta_trk, Mn, self.ids)
            gather(self.trans, self.trans_trk, Mn, self.ids)
            _lib.check(L.cp_tracker_render_dev2(h, Mn, _ptr(self.ids), _ptr(self.meta_trk), _ptr(self.trans_trk), ih, iw,
                                                _ptr(self.modes), _ptr(pre_hm), _ptr(pre_hm_hp), st),
                       "cp_tracker_render_dev2")
            self.eng.infer(cur[:n], self.meta_rows[:n], self.prm, prev[:n], pre_hm, pre_hm_hp, poses=poses,
                           n_valid=n_valid)
            _lib.check(L.cp_tracker_step_dev(h, Mn, _ptr(self.ids), _ptr(poses), _ptr(n_valid), poses.shape[-2],
                                             _ptr(self.meta_trk), _ptr(self.tracks_rows), _ptr(self.n_tracks_rows), st),
                       "cp_tracker_step_dev")
            gather(self.tracks_rows, self.tracks, MS, self.inv)
            gather(self.n_tracks_rows.view(MS, 1), self.n_tracks.view(MS, 1), MS, self.inv)

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

    def reset(self):
        """Forget every slot's tracks and previous frame: the next call starts a video in every slot (with idle slots:
        each slot's next live frame starts its video)."""
        self._fresh = True
        self._started = [False] * self.slots

    def _frames(self, frames):
        """The frames of one call, checked against the slots' shapes: one tensor, or one per slot (with idle slots: one
        per slot, None for an idle one)."""
        who = type(self).__name__
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
        if not self.per_slot and not self.idle_slots:
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
            if isinstance(f, np.ndarray):
                f = torch.from_numpy(f)
            if not torch.is_tensor(f) or f.dtype != torch.uint8 or tuple(f.shape) != self._slot_shapes[b]:
                what = ("%s %s" % (f.dtype, tuple(f.shape))) if torch.is_tensor(f) else type(f).__name__
                raise ValueError("%s: slot %d takes uint8 %s frames (%s, frame_hw %s), got %s"
                                 % (who, b, list(self._slot_shapes[b]), self.pixel_format, self._slot_hw[b], what))
            out.append(f)
        return out

    def __call__(self, frames, new_video=None, pre_dets=None):
        """The next frame of every slot -> (tracks [S,T,320], n_tracks [S]) ([M,S,...] in MultiCategoryTrackGraph):
        views of the graph's own buffers, overwritten by the next call.  frames: one array (one frame_hw) or a list of
        one frame per slot (one frame_hw per slot).  new_video: None or one bool per slot (slot i starts a new video
        with this frame)."""
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
        if self.idle_slots:
            return self._call_rows(frames, start)
        start = np.tile(start, self.streams // self.slots)       # one flag per tracker stream, the same in every category
        with torch.cuda.device(self.device):
            for dst, f in zip(self._slot_frames if self.per_slot else [self.frames], frames):
                dst.copy_(f, non_blocking=True)
            # a pageable source: staged before copy_ returns, without waiting for the device
            self.start.copy_(torch.from_numpy(start), non_blocking=True)
            self.graphs[self._parity].replay()
        self._parity ^= 1
        self._fresh = False
        return self._out

    def _call_rows(self, frames, start):
        """A call with idle slots: frames[i] None idles slot i.  A live slot starts its video when it has not started
        since the graph was built or reset, or when start[i] (new_video); an idle slot is not stepped and keeps its
        tracks and previous frame.  Copies the live frames and the control block, then replays the graph of the live
        count; with no live slot, zeros the outputs and launches no graph."""
        live = [i for i, f in enumerate(frames) if f is not None]
        with torch.cuda.device(self.device):
            if not live:
                self.tracks.zero_()
                self.n_tracks.zero_()
                return self._out
            start = np.array([i in live and (bool(start[i]) or not self._started[i]) for i in range(self.slots)], np.int32)
            for i in live:
                self._slot_frames[i].copy_(frames[i], non_blocking=True)
            # a pageable source: staged before copy_ returns, without waiting for the device
            self.ctrl.copy_(torch.from_numpy(self._control(live, start)), non_blocking=True)
            self.graphs[len(live) - 1].replay()
        for i in live:
            self._started[i] = True
        self._fresh = False
        return self._out


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

    def __init__(self, trk, slots, frame_hw, camera_matrix, pixel_format="bgr", idle_slots=False):
        from .detector import MultiCategoryDetector, MultiCategoryTracker
        if not isinstance(trk, MultiCategoryTracker):
            if isinstance(trk, MultiCategoryDetector):
                raise ValueError("MultiCategoryTrackGraph needs a MultiCategoryTracker; a MultiCategoryDetector is not a "
                                 "tracking model")
            raise NotImplementedError("MultiCategoryTrackGraph takes a MultiCategoryTracker; one category's "
                                      "ObjectPoseDetector goes to TrackGraph")
        self._build(trk, slots, frame_hw, camera_matrix, pixel_format, idle_slots)

    def _plan(self, trk, S, ih, iw):
        from .engine import Engine
        c, M = trk._plan_cfg, len(trk.categories)
        eng = Engine(c["arch"], c["heads"], c["head_conv"], S, ih, iw, self.device.index, tracking=c["tracking"],
                     tracking_task_gru=c["tracking_task_gru"], precision=c["precision"], models=M,
                     reuse_activations=True)
        for m, sd in enumerate(trk._weights):
            eng.load_state_dict(sd, model=m)
        prm = list(trk._prms) if M > 1 else trk._prms[0]
        return eng, prm, Tracker(trk.opt, streams=S, device=self.device, categories=trk.categories), list(trk.categories)
