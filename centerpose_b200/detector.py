"""`ObjectPoseDetector` on the H100-native hot path -- the drop-in for
/root/reference/src/lib/detectors/{base_detector,object_pose,detector_factory}.py.

`run()` keeps the reference's one-image semantics and its 12-key return dict
(base_detector.py:390-772): load -> pre_process -> network -> decode ->
post_process -> merge -> PnP.  A uint8 BGR image is uploaded once and
pre-processed on the device at every test scale, bit for bit what the cv2 code
of `pre_process` gives (which stays, as the public method and for pre-processed
input); everything after it runs in libcenterpose_b200.so too.  The only host
work left is rebuilding the reference's Python result structures from the
fixed-shape pose records (`records_to_results`).  `run_batch()` is the batched
entry point the reference does not have (B = 32 / 256 configurations of
BASELINE.json).
"""
import copy
import json
import os
import time

import numpy as np
import torch

from . import _lib
from .engine import (JPEG, Engine, check_pixel_format, decode_params, decode_pnp, frame_layout, image_size, is_jpeg,
                     jpeg_bytes, jpeg_decode, jpeg_error_text, jpeg_parse, make_meta, preprocess, preprocess_formats,
                     preprocess_remap, slot_formats)
from .lens import MapCache, slot_distortions, undistorted_cameras
from .model import _load_checkpoint, create_model, load_model
from .tracker import Tracker, tracks_to_results


# ----------------------------------------------------------------------------- records -> reference structures
def record_to_result(rec):
    """One CP_POSE_RECORD row -> the reference's per-detection dict
    (post_process.py:27-63 + cuboid_pnp_shell.py:27-54)."""
    L = _lib
    r = np.asarray(rec, np.float32)
    d = {
        "score": float(r[L.P_SCORE]),
        "cls": int(r[L.P_CLS]),
        "obj_scale": r[L.P_OBJ_SCALE:L.P_OBJ_SCALE + 3].copy(),
        "obj_scale_uncertainty": r[L.P_OBJ_SCALE_UNC:L.P_OBJ_SCALE_UNC + 3].copy(),
        "kps_displacement_std": r[L.P_KPS_DISP_STD:L.P_KPS_DISP_STD + 16].copy(),
        "bbox": r[L.P_BBOX:L.P_BBOX + 4].astype(np.float64),
        "ct": [float(r[L.P_CT]), float(r[L.P_CT + 1])],
        "kps": r[L.P_KPS:L.P_KPS + 16].astype(np.float64),
        "tracking": r[L.P_TRACKING:L.P_TRACKING + 2].copy(),
        "tracking_hp": r[L.P_TRACKING_HP:L.P_TRACKING_HP + 16].copy(),
        "kps_displacement_mean": r[L.P_KPS_DISP_MEAN:L.P_KPS_DISP_MEAN + 16].astype(np.float64),
        "kps_heatmap_mean": r[L.P_KPS_HM_MEAN:L.P_KPS_HM_MEAN + 16].astype(np.float64),
        "kps_heatmap_std": r[L.P_KPS_HM_STD:L.P_KPS_HM_STD + 16].copy(),
        "kps_heatmap_height": r[L.P_KPS_HM_HEIGHT:L.P_KPS_HM_HEIGHT + 8].copy(),
    }
    st = int(r[L.P_STATUS])
    d["pnp_status"] = st
    if st in (L.PNP_OK, L.PNP_INVISIBLE):
        d["location"] = [float(v) for v in r[L.P_LOCATION:L.P_LOCATION + 3]]
        d["quaternion_xyzw"] = r[L.P_QUAT:L.P_QUAT + 4].astype(np.float64)
        d["projected_cuboid"] = r[L.P_PROJ_CUBOID:L.P_PROJ_CUBOID + 16].astype(np.float64).reshape(8, 2)
        d["kps_3d_cam"] = r[L.P_KPS_3D_CAM:L.P_KPS_3D_CAM + 27].astype(np.float64).reshape(9, 3)
        d["kps_pnp"] = r[L.P_KPS_PNP:L.P_KPS_PNP + 18].astype(np.float64).reshape(9, 2)
        d["reprojection_error"] = float(r[L.P_REPROJ])
    return d


def records_to_results(poses, n_valid, width, height):
    """poses [K,192], n_valid -> (results ndarray-of-dicts, boxes list) exactly
    shaped like base_detector.py:498,548-654."""
    res = [record_to_result(poses[i]) for i in range(int(n_valid))]
    boxes = []
    for d in res:
        if d["pnp_status"] == _lib.PNP_OK:
            kp = d["kps"].reshape(-1, 2)
            po = np.vstack([kp.mean(0, keepdims=True), kp]).copy()
            po[:, 0] /= width
            po[:, 1] /= height
            boxes.append((d["kps_pnp"], d["kps_3d_cam"], np.array(d["obj_scale"]), po, d))
    return np.array(res, dtype=object), boxes


def dets_to_dict(dets):
    """dets [B,K,128] -> the 13 arrays of decode.py:348-361."""
    L = _lib
    a = np.asarray(dets, np.float32)
    f = lambda off, n: a[..., off:off + n].copy()
    return {
        "bboxes": f(L.D_BBOX, 4), "scores": f(L.D_SCORE, 1), "kps": f(L.D_KPS, 16), "clses": f(L.D_CLS, 1),
        "obj_scale": f(L.D_OBJ_SCALE, 3), "obj_scale_uncertainty": f(L.D_OBJ_SCALE_UNC, 3),
        "tracking": f(L.D_TRACKING, 2), "tracking_hp": f(L.D_TRACKING_HP, 16),
        "kps_displacement_mean": f(L.D_KPS_DISP_MEAN, 16), "kps_displacement_std": f(L.D_KPS_DISP_STD, 16),
        "kps_heatmap_mean": f(L.D_KPS_HM_MEAN, 16), "kps_heatmap_std": f(L.D_KPS_HM_STD, 16),
        "kps_heatmap_height": f(L.D_KPS_HM_HEIGHT, 8),
    }


def affine_from_center_scale(c, s, out_w, out_h, inv=False):
    """The rot=0 case of utils/image.py:35-68: three float32 control points
    (centre, centre + (0, -s/2), and the perpendicular third point) handed to
    cv2.getAffineTransform, which is what the reference calls."""
    import cv2
    src = np.zeros((3, 2), np.float32)
    dst = np.zeros((3, 2), np.float32)
    src[0] = c
    src[1] = np.asarray(c, np.float32) + np.array([0, s * -0.5], np.float32)
    dst[0] = [out_w * 0.5, out_h * 0.5]
    dst[1] = np.array([out_w * 0.5, out_h * 0.5], np.float32) + np.array([0, out_w * -0.5], np.float32)
    for p in (src, dst):
        d = p[0] - p[1]
        p[2] = p[1] + np.array([-d[1], d[0]], np.float32)
    return cv2.getAffineTransform(dst, src) if inv else cv2.getAffineTransform(src, dst)


def scale_width(s):
    """The scale of a pre_process meta as one number: `s` is max(h, w) in the fix_res mode and the (w, h) pair in the
    keep_res and fix_short modes, of which get_affine_transform uses only the width (image.py:44-45).  The meta row
    and so the decode's s / max(w, h) ratio take the same width (post_process.py:33,45,48,60 would broadcast a (w, h)
    pair against the 16 keypoint values and fail)."""
    return float(s[0]) if isinstance(s, np.ndarray) and s.ndim else float(s)


def camera_per_frame(camera_matrix, B):
    """camera_matrix [3,3] (shared) or [B,3,3] / a list of B [3,3] -> B float64 [3,3] matrices."""
    cam = np.asarray(camera_matrix, np.float64)
    if cam.shape == (3, 3):
        return [cam] * B
    if cam.shape != (B, 3, 3):
        raise ValueError("camera_matrix must be [3,3] or one [3,3] per frame ([%d,3,3]), got %s" % (B, cam.shape))
    return list(cam)


class JpegFrame:
    """An encoded JPEG frame of run_batch(list, pixel_format="jpeg"): its bytes (uint8 numpy) and parsed header; shape is
    that of the decoded BGR image (after the EXIF orientation)."""

    def __init__(self, data, header):
        self.data, self.header = data, header
        self.shape = (header.out_h, header.out_w, 3)


def jpeg_frames(frames, pixel_format):
    """run_batch(list) with pixel_format "jpeg" (or a list naming it for some frames): each such frame (bytes, a 1-D uint8
    numpy array or CPU tensor; None for an idle slot) parsed into a JpegFrame, its format replaced by "bgr".  A refused
    header raises ValueError naming the frame and the reason, before any device work.  Other calls are returned as
    they are."""
    names = list(pixel_format) if isinstance(pixel_format, (list, tuple)) else [pixel_format] * len(frames)
    if JPEG not in [f for f in names if isinstance(f, str)]:
        return frames, pixel_format
    if len(names) != len(frames):
        raise ValueError("run_batch: pixel_format is one name or one per frame, got %d names for %d frames"
                         % (len(names), len(frames)))
    frames = list(frames)
    for b, f in enumerate(frames):
        if names[b] != JPEG:
            continue
        names[b] = "bgr"
        if f is None:
            continue
        data = jpeg_bytes(f)
        if data is None:
            raise TypeError("run_batch: frame %d is a %s; pixel_format \"jpeg\" takes encoded bytes, a 1-D uint8 numpy "
                            "array or CPU tensor" % (b, type(f).__name__))
        h = jpeg_parse(data)
        if h.status:
            raise ValueError("run_batch: frame %d is a JPEG the device decoder does not take: %s"
                             % (b, _lib.JPEG_REFUSALS.get(h.status, h.status)))
        frames[b] = JpegFrame(data, h)
    return frames, names


def check_frames(frames, allow_idle, pixel_format="bgr"):
    """The frames of a ragged batch: uint8 [H,W,3] numpy arrays or tensors, or the buffers of another pixel_format
    (engine.check_pixel_format), one name for every frame or a list with one per frame (None = an idle slot when
    allowed)."""
    if not isinstance(pixel_format, (list, tuple)):
        check_pixel_format(pixel_format)
    if len(frames) == 0:
        raise ValueError("run_batch: an empty list of frames")
    fmts = slot_formats(pixel_format, len(frames))
    for b, f in enumerate(frames):
        if f is None:
            if not allow_idle:
                raise ValueError("run_batch: frame %d is None (idle slots need track=True)" % b)
            continue
        if isinstance(f, JpegFrame):
            continue
        if not isinstance(f, (np.ndarray, torch.Tensor)):
            raise TypeError("run_batch: frame %d is a %s, not a numpy array or tensor" % (b, type(f).__name__))
        dt = f.dtype
        if dt not in (np.uint8, torch.uint8):
            raise TypeError("run_batch: frame %d is %s; the ragged path takes uint8 %s frames"
                            % (b, dt, frame_layout(fmts[b])))
        image_size(f.shape, fmts[b], "run_batch: frame %d" % b)


def check_slot_list(values, S, name, kind=None):
    """A per-slot argument: None, or a list of S entries."""
    if values is None:
        return None
    values = list(values)
    if len(values) != S:
        raise ValueError("run_batch: %d %s entries for %d slots" % (len(values), name, S))
    return [kind(v) for v in values] if kind is not None else values


def _returned(pair, to_host):
    return (pair[0].cpu().numpy(), pair[1].cpu().numpy()) if to_host else pair


class _SlotState(object):
    """run_batch(track=True): the tracker of S slot streams (of every category, with `categories`: stream m * S + s is
    slot s of category m), each slot's previous network input (`pre`, [S,3,h,w], None before the first step; never
    written in place, so it may be the network input of the previous step itself; shared by the categories) and
    whether each slot has had a frame since the state was made."""

    def __init__(self, opt, S, device, categories=None):
        self.streams = S
        self.tracker = Tracker(opt, streams=S, device=device, categories=categories)
        self.pre = None
        self.started = [False] * S


# ----------------------------------------------------------------------------- detector
class ObjectPoseDetector(object):
    def __init__(self, opt, model=None):
        if opt.gpus[0] < 0:
            raise RuntimeError("centerpose_b200 runs on a CUDA device only (--gpus -1 is the reference's CPU path)")
        opt.device = torch.device("cuda")
        self.opt = opt
        print("Creating model...")
        self.model = model if model is not None else create_model(opt.arch, opt.heads, opt.head_conv, opt)
        if getattr(opt, "load_model", ""):
            self.model = load_model(self.model, opt.load_model)
        self.model = self._to_device(self.model)
        self.model.eval()
        self.mean = np.array(opt.mean, dtype=np.float32).reshape(1, 1, 3)
        self.std = np.array(opt.std, dtype=np.float32).reshape(1, 1, 3)
        self.max_per_image = 100
        self.num_classes = opt.num_classes
        self.scales = opt.test_scales
        self.opt = opt
        self.pause = True
        self.pre_images = None
        self.tracker = None
        self.flip_idx = getattr(opt, "flip_idx", None)
        if getattr(opt, "refined_Kalman", False):
            raise NotImplementedError("opt.refined_Kalman (utils/tracker_baseline.py, CenterPose + Kalman baseline) is not "
                                      "on the accelerated path; use --tracking_task (CenterPoseTrack)")
        if getattr(opt, "tracking_task", False):
            # base_detector.py:53-54: the tracker state lives on the device (centerpose_b200/tracker.py)
            self.tracker = Tracker(opt, streams=1, device=opt.device)
        self._slots = None             # run_batch(track=True): per-slot tracker and previous frames (_SlotState)
        self._meta_key = None          # run_batch: bytes of the host meta rows last uploaded to _meta_dev
        self._meta_dev = None
        self._packed = None            # run_batch(list): device buffer the ragged frames are packed into
        self._affines = {}             # (h, w) -> fix_res trans_input of that frame size
        self._maps = MapCache()        # run_batch(distortion=): the device map of each camera
        self._stage = None             # run(): the pinned staging buffer and the device buffer of the frame
        self._frame_dev = None
        self._jpeg_dev = None          # run(): the device copy of a JPEG file's bytes

    def _to_device(self, t):
        """base_detector.py:41,436: everything the network touches lives on opt.device (always CUDA here)."""
        return t.to(self.opt.device)

    # base_detector.py:91-148 -- the reference's cv2 pre-processing (host side), all three modes
    def pre_process(self, image, scale, input_meta={}):
        import cv2
        (new_height, new_width), meta = self._pre_meta(image.shape[0], image.shape[1], scale, input_meta)
        inp_height, inp_width = meta["inp_height"], meta["inp_width"]
        resized = cv2.resize(image, (new_width, new_height))
        inp = cv2.warpAffine(resized, meta["trans_input"], (inp_width, inp_height), flags=cv2.INTER_LINEAR)
        inp = ((inp / 255. - self.mean) / self.std).astype(np.float32)
        images = torch.from_numpy(inp.transpose(2, 0, 1).reshape(1, 3, inp_height, inp_width))
        return images, meta

    def _pre_meta(self, height, width, scale, input_meta):
        """The geometry of pre_process for a height x width frame at `scale`, in each mode: ((new_height, new_width), the
        size cv2.resize takes the frame to; meta, with pre_dets / camera_matrix / id copied from input_meta)."""
        new_height = int(height * scale)
        new_width = int(width * scale)
        if self.opt.fix_short > 0:
            if height < width:
                inp_height = self.opt.fix_short
                inp_width = (int(width / height * self.opt.fix_short) + 63) // 64 * 64
            else:
                inp_height = (int(height / width * self.opt.fix_short) + 63) // 64 * 64
                inp_width = self.opt.fix_short
            c = np.array([width / 2, height / 2], dtype=np.float32)
            s = np.array([width, height], dtype=np.float32)
        elif self.opt.fix_res:
            inp_height, inp_width = self.opt.input_h, self.opt.input_w
            c = np.array([new_width / 2., new_height / 2.], dtype=np.float32)
            s = max(height, width) * 1.0
        else:
            inp_height = (new_height | self.opt.pad) + 1
            inp_width = (new_width | self.opt.pad) + 1
            c = np.array([new_width // 2, new_height // 2], dtype=np.float32)
            s = np.array([inp_width, inp_height], dtype=np.float32)
        s0 = scale_width(s)                                                # the affine only uses the width (image.py:44)
        trans_input = affine_from_center_scale(c, s0, inp_width, inp_height)
        out_height = inp_height // self.opt.down_ratio
        out_width = inp_width // self.opt.down_ratio
        trans_output = affine_from_center_scale(c, s0, out_width, out_height)
        meta = {"c": c, "s": s, "height": height, "width": width, "out_height": out_height,
                "out_width": out_width, "inp_height": inp_height, "inp_width": inp_width,
                "trans_input": trans_input, "trans_output": trans_output}
        for k in ("pre_dets", "camera_matrix", "id"):
            if k in input_meta:
                meta[k] = input_meta[k]
        return (new_height, new_width), meta

    def _check_scales(self, h, w):
        """A test scale that resizes the h x w frame below 1 px is refused before any device work."""
        for scale in self.scales:
            if int(h * scale) < 1 or int(w * scale) < 1:
                raise ValueError("run: test scale %g resizes the %d x %d frame to %d x %d pixels"
                                 % (scale, h, w, int(h * scale), int(w * scale)))

    def _device_frame(self, image):
        """run()'s frame on the device, or None for the host pre_process: a uint8 [H,W,3] numpy image is uploaded once
        per call, as [1,H,W,3], through a pinned staging buffer into a device buffer, both kept and grown (run()
        synchronises before it returns, so both are free again at the next call).  A test scale that resizes the frame
        below 1 px is refused first."""
        if not (isinstance(image, np.ndarray) and image.dtype == np.uint8 and image.ndim == 3 and image.shape[2] == 3):
            return None
        self._check_scales(*image.shape[:2])
        n = image.size
        if self._stage is None or self._stage.numel() < n or self._frame_dev.numel() < n:
            self._stage = torch.empty((n,), dtype=torch.uint8, pin_memory=True)
            self._frame_dev = torch.empty((n,), dtype=torch.uint8, device=self.opt.device)
        np.copyto(self._stage[:n].numpy().reshape(image.shape), image)
        frame = self._frame_dev[:n]
        frame.copy_(self._stage[:n], non_blocking=True)
        return frame.view((1,) + image.shape)

    def _device_jpeg(self, data, header):
        """run()'s frame decoded on the device from the bytes of a supported JPEG (cp_jpeg_decode, bit for bit
        cv2.imread): the bytes go up once through the pinned staging buffer, the decoded frame lands in the device frame
        buffer as [1,H,W,3].  None when the bitstream is corrupt (the frame's error word, read back once): run() then
        decodes on the host as before."""
        h, w = header.out_h, header.out_w
        self._check_scales(h, w)
        n, m = len(data), h * w * 3
        if self._stage is None or self._stage.numel() < n:
            self._stage = torch.empty((n,), dtype=torch.uint8, pin_memory=True)
        if self._frame_dev is None or self._frame_dev.numel() < m:
            self._frame_dev = torch.empty((m,), dtype=torch.uint8, device=self.opt.device)
        if self._jpeg_dev is None or self._jpeg_dev.numel() < n:
            self._jpeg_dev = torch.empty((n,), dtype=torch.uint8, device=self.opt.device)
        np.copyto(self._stage[:n].numpy(), data)
        self._jpeg_dev[:n].copy_(self._stage[:n], non_blocking=True)
        errors = jpeg_decode([header], self._jpeg_dev, [0], self._frame_dev, [0])
        if int(errors.item()):
            return None
        return self._frame_dev[:m].view(1, h, w, 3)

    def _device_pre_process(self, frame, scale, input_meta):
        """pre_process on the device of the uploaded frame ([1,H,W,3] uint8 CUDA, _device_frame): the same images (here
        a [1,3,inp_height,inp_width] CUDA tensor) and meta, bit for bit -- cv2.resize fused into the warp
        (cp_preprocess_resize_affine) in all three modes."""
        (new_height, new_width), meta = self._pre_meta(frame.shape[1], frame.shape[2], scale, input_meta)
        images = preprocess(frame, meta["inp_height"], meta["inp_width"], self.opt.mean, self.opt.std,
                            trans_input=meta["trans_input"], resize_hw=(new_height, new_width))
        return images, meta

    def _track_policy(self, start, frame_id, pre_dets):
        """base_detector.py:440-465 for one stream and frame: (the pre_dets to seed the stream from, or None; the
        cp_render_mode of its previous-frame heat maps).  A stream is seeded when its video starts and on ground-truth
        frames (opt.gt_pre_hm_hmhp: every frame; opt.gt_pre_hm_hmhp_first: frame_id 0; :451-454), whose heat maps are
        drawn from the ground truth; with opt.empty_pre_hm they are empty (_get_additional_inputs, :165-166)."""
        gt = bool(getattr(self.opt, "gt_pre_hm_hmhp", False))
        if not gt and getattr(self.opt, "gt_pre_hm_hmhp_first", False):
            if frame_id is None:
                raise ValueError("opt.gt_pre_hm_hmhp_first needs the frame index, meta['id']")
            gt = int(frame_id) == 0
        if getattr(self.opt, "empty_pre_hm", False):
            mode = _lib.RENDER_EMPTY
        else:
            mode = _lib.RENDER_GT if gt else _lib.RENDER_TRACKS
        return (pre_dets if start or gt else None), mode

    def _meta_tensor(self, meta, batch=1):
        cam = meta.get("camera_matrix")
        if cam is None:
            if self.opt.use_pnp:
                raise ValueError("meta_inp['camera_matrix'] is required when opt.use_pnp is set (demo.py:141-147)")
            cam = np.eye(3)
        return make_meta(batch, meta["c"], scale_width(meta["s"]), meta["width"], meta["height"], cam)

    def process(self, images, pre_images=None, pre_hms=None, pre_hm_hp=None, pre_inds=None, return_time=False,
                meta=None, scale=1.0):
        """object_pose.py:131-165: network + sigmoid + decode.  Returns
        (output, dets[, forward_time]); the pose records of the fused stage are
        kept on `self._last` (host) / `self._last_dev` (device) for post_process / merge / PnP / tracking."""
        torch.cuda.synchronize()
        output = self.model(images, pre_images, pre_hms, pre_hm_hp)[-1]
        torch.cuda.synchronize()
        forward_time = time.time()
        prm = decode_params(self.opt, test_scale=float(scale))
        metat = self._meta_tensor(meta if meta is not None else self._dummy_meta(images), images.shape[0]).to(images.device)
        dets, poses, n_valid = decode_pnp(output, metat, prm, want_dets=True)
        output["hm"] = output["hm"].sigmoid_()
        if self.opt.hm_hp and not self.opt.mse_loss:
            output["hm_hp"] = output["hm_hp"].sigmoid_()
        output.update({"pre_inds": pre_inds})
        self._last_dev = (poses, n_valid, metat)
        self._last = (poses.cpu().numpy(), n_valid.cpu().numpy())
        dets = dets_to_dict(dets.cpu().numpy())
        if return_time:
            return output, dets, forward_time
        return output, dets

    def _dummy_meta(self, images):
        h, w = images.shape[2], images.shape[3]
        return {"c": np.array([w / 2., h / 2.], np.float32), "s": float(max(h, w)), "width": w, "height": h,
                "camera_matrix": np.eye(3)}

    def run(self, image_or_path_or_tensor, filename=None, meta_inp={}, preprocessed_flag=False):
        """base_detector.py:390-772.  One image per call, the reference's 12-key return dict.  A uint8 [H,W,3] image
        (passed, or read from a path) is uploaded once and pre-processed on the device at every test scale
        (_device_frame, _device_pre_process: bit for bit pre_process, so `pre` covers the upload and the launches);
        pre-processed input and other dtypes or shapes go through pre_process on the host.  After that everything runs
        in libcenterpose_b200.so; post_process / merge_outputs / PnP are part of the fused decode call, so their stamps
        are 0 and `dec` carries the whole post-network stage."""
        import cv2
        load_time, pre_time, net_time, dec_time, post_time = 0, 0, 0, 0, 0
        merge_time, track_time, pnp_time, tot_time = 0, 0, 0, 0
        tracking = bool(getattr(self.opt, "tracking_task", False))
        if tracking and (len(self.scales) != 1 or self.scales[0] != 1.0):
            raise NotImplementedError("CenterPoseTrack runs at test_scales=[1] (the reference re-initialises the tracker "
                                      "state once per scale, base_detector.py:440-449)")
        start_time = time.time()
        pre_processed = preprocessed_flag
        encoded = None              # the bytes of a JPEG file or of encoded input, decoded on the device
        from_path = type(image_or_path_or_tensor) == type("")   # before `filename` may replace it (a label, not a file)
        if isinstance(image_or_path_or_tensor, (bytes, bytearray)) or (
                isinstance(image_or_path_or_tensor, np.ndarray) and image_or_path_or_tensor.ndim == 1
                and image_or_path_or_tensor.dtype == np.uint8):
            encoded, image = jpeg_bytes(image_or_path_or_tensor), None
            if filename is not None:
                image_or_path_or_tensor = filename
        elif isinstance(image_or_path_or_tensor, np.ndarray):
            image = image_or_path_or_tensor
            if filename is not None:
                image_or_path_or_tensor = filename
        elif type(image_or_path_or_tensor) == type(""):
            image = None
            try:
                with open(image_or_path_or_tensor, "rb") as fp:
                    head = fp.read(3)
                    if is_jpeg(head):
                        encoded = np.frombuffer(head + fp.read(), np.uint8)
            except OSError:
                pass
            if encoded is None:
                image = cv2.imread(image_or_path_or_tensor)
        else:
            image = image_or_path_or_tensor["image"][0].numpy()
            pre_processed = True
        loaded_time = time.time()
        load_time += loaded_time - start_time
        # a uint8 BGR frame goes to the device once and every scale pre-processes it there; `pre` covers the upload.
        # A supported JPEG is decoded there instead (bit for bit cv2.imread); a refused or corrupt one is decoded by cv2.
        frame = None
        if encoded is not None:
            header = jpeg_parse(encoded) if is_jpeg(encoded) else None
            if header is not None and header.status == 0:
                frame = self._device_jpeg(encoded, header)
            if frame is None:
                image = cv2.imread(image_or_path_or_tensor) if from_path else cv2.imdecode(encoded, cv2.IMREAD_COLOR)
            else:
                debug = int(getattr(self.opt, "debug", 0) or 0)
                image = frame[0].cpu().numpy() if debug >= 1 else None
        if frame is None and not pre_processed:
            frame = self._device_frame(image)
        pre_time += time.time() - loaded_time

        # base_detector.py:421-497: one pass per test scale.  merge_outputs (object_pose.py:184-197) reads detections[0],
        # i.e. only the FIRST scale contributes results (with the soft-NMS forced on when several scales are listed); the
        # other passes still run because run() returns the `output` maps of the last one.
        first = None
        for si, scale in enumerate(self.scales):
            scale_start_time = time.time()
            if frame is not None:
                images, meta = self._device_pre_process(frame, scale, meta_inp)
            elif not pre_processed:
                images, meta = self.pre_process(image, scale, meta_inp)
            else:
                images = torch.from_numpy(np.expand_dims(image, axis=0))
                meta = meta_inp
            images = self._to_device(images)

            pre_hms, pre_hm_hp, pre_inds = None, None, None
            if tracking:
                start = self.pre_images is None
                seed, mode = self._track_policy(start, meta.get("id"), meta.get("pre_dets"))
                if start:                                         # base_detector.py:444-449
                    print("Initialize tracking!")
                    self.pre_images = images
                if start or seed is not None:
                    self.tracker.init_track(meta)
                if self.opt.pre_hm or self.opt.pre_hm_hp:         # :456-462, rendered on the device from the tracker state
                    if "trans_input" not in meta:
                        raise ValueError("tracking needs meta['trans_input'] (pre_process provides it)")
                    metat = self._meta_tensor(meta).to(images.device)
                    pre_hms, pre_hm_hp = self.tracker.render(metat, meta["trans_input"], images.shape[2], images.shape[3],
                                                             modes=[mode])
            torch.cuda.synchronize()
            pre_process_time = time.time()
            pre_time += pre_process_time - scale_start_time

            output, dets, forward_time = self.process(images, self.pre_images if tracking else None, pre_hms, pre_hm_hp,
                                                      pre_inds, return_time=True, meta=meta, scale=scale)
            torch.cuda.synchronize()
            net_time += forward_time - pre_process_time
            decode_time = time.time()
            dec_time += decode_time - forward_time
            if si == 0:
                first = (self._last, self._last_dev, meta)
        self._last, self._last_dev, meta = first

        # post_process + merge + PnP already happened inside cp_decode_pnp; unpack the records
        poses, n_valid = self._last
        results, boxes = records_to_results(poses[0], n_valid[0], meta["width"], meta["height"])
        if not self.opt.use_pnp:
            boxes = []
        post_process_time = time.time()
        post_time += post_process_time - decode_time
        pnp_process_time = post_process_time

        if tracking:                                          # :660-665 (gaussian_fusion :502-544 runs inside the step)
            pd, nd, md = self._last_dev
            self.tracker.step_records(pd, nd, md)
            rows, nt = self.tracker._host()
            results, boxes = tracks_to_results(rows[0], nt[0], meta["width"], meta["height"])
            if not self.opt.use_pnp:
                boxes = []
            self.pre_images = images
        end_time = time.time()
        track_time += end_time - pnp_process_time
        tot_time += end_time - start_time

        dict_out = self.build_dict_out(meta, results, boxes)
        self.last_dict_out = dict_out
        debug = int(getattr(self.opt, "debug", 0) or 0)
        if debug >= 1 and debug < 4:
            self.show_results(None, image, results)
        elif debug == 4:
            self.save_results(None, image, results, image_or_path_or_tensor, dict_out)
        elif debug == 6:
            self.save_results_eval(None, image, results, image_or_path_or_tensor, dict_out)
        return {"results": results, "boxes": boxes, "output": output, "tot": tot_time, "load": load_time,
                "pre": pre_time, "net": net_time, "dec": dec_time, "post": post_time, "merge": merge_time,
                "pnp": pnp_time, "track": track_time}

    # ------------------------------------------------------------------ result emitters (SURVEY.md row f-3)
    def build_dict_out(self, meta, results, boxes):
        """The JSON payload of base_detector.py:672-754: camera matrix + one object per track (tracking) or per box."""
        opt = self.opt
        dict_out = {"camera_data": [], "objects": []}
        if "camera_matrix" in meta:
            dict_out["camera_data"] = np.asarray(meta["camera_matrix"]).tolist()
        lst = lambda v: np.asarray(v).tolist()      # noqa: E731
        if getattr(opt, "tracking_task", False):
            for tr in results:
                sc = np.asarray(tr["obj_scale"], np.float64)
                obj = {"class": opt.c, "ct": tr["ct"], "bbox": lst(tr["bbox"]), "confidence": tr["score"],
                       "kps_displacement_mean": lst(tr["kps_displacement_mean"]), "kps_heatmap_mean": lst(tr["kps_heatmap_mean"]),
                       "kps_heatmap_std": lst(tr["kps_heatmap_std"]), "kps_heatmap_height": lst(tr["kps_heatmap_height"]),
                       "obj_scale": (sc / sc[1]).tolist(), "tracking_id": tr["tracking_id"]}
                if opt.use_pnp:
                    if "location" in tr:
                        obj["location"] = tr["location"]
                        obj["quaternion_xyzw"] = lst(tr["quaternion_xyzw"])
                    if "kps_pnp" in tr:
                        obj["kps_pnp"] = lst(tr["kps_pnp"])
                        obj["kps_3d_cam"] = lst(tr["kps_3d_cam"])
                if getattr(opt, "obj_scale_uncertainty", False):
                    obj["obj_scale_uncertainty"] = lst(tr["obj_scale_uncertainty"])
                if getattr(opt, "kalman", False):
                    obj["kps_mean_kf"] = lst(tr["kps_mean_kf"])
                    obj["kps_std_kf"] = tr["kps_std_kf"]
                    if opt.use_pnp and "kps_pnp_kf" in tr:
                        obj["kps_pnp_kf"] = lst(tr["kps_pnp_kf"])
                        obj["kps_3d_cam_kf"] = lst(tr["kps_3d_cam_kf"])
                if getattr(opt, "scale_pool", False):
                    sk = np.asarray(tr["obj_scale_kf"], np.float64)
                    obj["obj_scale_kf"] = (sk / sk[1]).tolist()
                    obj["obj_scale_uncertainty_kf"] = lst(tr["obj_scale_uncertainty_kf"])
                if getattr(opt, "hps_uncertainty", False):
                    obj["kps_displacement_std"] = lst(tr["kps_displacement_std"])
                    obj["kps_fusion_mean"] = lst(tr["kps_fusion_mean"])
                    obj["kps_fusion_std"] = lst(tr["kps_fusion_std"])
                if getattr(opt, "tracking", False):
                    obj["tracking"] = lst(tr["tracking"])
                if getattr(opt, "tracking_hp", False):
                    obj["tracking_hp"] = lst(tr["tracking_hp"])
                dict_out["objects"].append(obj)
        else:
            for box in boxes:
                b = box[4]
                obj = {"class": opt.c, "ct": b["ct"], "bbox": lst(b["bbox"]), "confidence": b["score"],
                       "kps_displacement_mean": lst(b["kps_displacement_mean"]), "kps_heatmap_mean": lst(b["kps_heatmap_mean"]),
                       "kps_heatmap_std": lst(b["kps_heatmap_std"]), "kps_heatmap_height": lst(b["kps_heatmap_height"]),
                       "obj_scale": lst(b["obj_scale"])}
                if opt.use_pnp:
                    if "location" in b:
                        obj["location"] = b["location"]
                        obj["quaternion_xyzw"] = lst(b["quaternion_xyzw"])
                    if "kps_pnp" in b:
                        obj["kps_pnp"] = lst(b["kps_pnp"])
                        obj["kps_3d_cam"] = lst(b["kps_3d_cam"])
                dict_out["objects"].append(obj)
        return dict_out

    def _debugger(self, debugger):
        """The reference's Debugger (drawing) when its package is importable (drop-in use inside the reference tree);
        visualisation itself is outside the accelerated path, so without it only the JSON is written."""
        if debugger is not None:
            return debugger
        try:
            from lib.utils.debugger import Debugger
            return Debugger(dataset=self.opt.dataset, ipynb=(self.opt.debug == 3),
                            theme=getattr(self.opt, "debugger_theme", "white"))
        except Exception:
            return None

    def _draw(self, debugger, image, results, eval_mode=False):
        opt = self.opt
        debugger.add_img(image, img_id="out_img_pred")
        for bbox in results:
            if bbox["score"] > opt.vis_thresh and opt.reg_bbox:
                if getattr(opt, "tracking_task", False) and not eval_mode:
                    debugger.add_coco_bbox(bbox["bbox"], 0, bbox["score"], id=bbox["tracking_id"], img_id="out_img_pred")
                else:
                    debugger.add_coco_bbox(bbox["bbox"], 0, bbox["score"], img_id="out_img_pred")
                if "projected_cuboid" in bbox:
                    debugger.add_coco_hp(bbox["projected_cuboid"], img_id="out_img_pred", pred_flag="pnp")

    def show_results(self, debugger, image, results):
        """object_pose.py:280-317 (interactive display): needs the reference's Debugger."""
        dbg = self._debugger(debugger)
        if dbg is None:
            return
        self._draw(dbg, image, results)
        dbg.show_all_imgs(pause=self.pause)

    def save_results(self, debugger, image, results, image_or_path_or_tensor, dict_out=None):
        """object_pose.py:357-414: <demo_save>/<source name>/<frame>.json (+ the rendered image when a Debugger exists)."""
        opt = self.opt
        if os.path.isdir(opt.demo):
            target = os.path.join(opt.demo_save, os.path.basename(opt.demo))
        else:
            target = os.path.join(opt.demo_save, os.path.splitext(os.path.basename(opt.demo))[0])
        os.makedirs(target, exist_ok=True)
        dbg = self._debugger(debugger)
        if dbg is not None:
            self._draw(dbg, image, results)
            dbg.save_all_imgs_demo(image_or_path_or_tensor, path=target)
        if dict_out is not None:
            name = os.path.splitext(os.path.basename(image_or_path_or_tensor))[0]
            with open(os.path.join(target, name + ".json"), "w") as fp:
                json.dump(dict_out, fp)
            return os.path.join(target, name + ".json")

    def save_results_eval(self, debugger, image, results, image_or_path_or_tensor, dict_out=None, video_layout=False):
        """object_pose.py:319-355: demo/<checkpoint name>/[<video>/]<frame>.json, the layout the Objectron evaluator
        (tools/objectron_eval/eval_video_official.py:307-311) reads."""
        opt = self.opt
        if getattr(opt, "tracking_task", False) or getattr(opt, "eval_max_num", None) == 100:
            video_layout = True
        root = os.path.join("demo", os.path.splitext(os.path.basename(opt.load_model))[0])
        os.makedirs(root, exist_ok=True)
        key = image_or_path_or_tensor
        file_id = key[key.rfind("_") + 1:]
        folder = key[:key.rfind("_")]
        dbg = self._debugger(debugger)
        if dbg is not None:
            self._draw(dbg, image, results, eval_mode=True)
        if video_layout:
            vdir = os.path.join(root, folder)
            os.makedirs(vdir, exist_ok=True)
            if dbg is not None:
                dbg.save_all_imgs_eval(key, path=vdir, video_layout=True)
            path = os.path.join(vdir, file_id + ".json")
        else:
            if dbg is not None:
                dbg.save_all_imgs_eval(key, path=root, video_layout=False)
            path = os.path.join(root, "%s_%s.json" % (folder, file_id))
        if dict_out is not None:
            with open(path, "w") as fp:
                json.dump(dict_out, fp)
            return path

    # ------------------------------------------------------------------ batched API (not in the reference)
    def run_batch(self, frames, camera_matrix, pre_images=None, pre_hms=None, pre_hm_hp=None, to_host=True, track=False,
                  out=None, pre_dets=None, frame_ids=None, new_video=None, pixel_format="bgr", distortion=None):
        """frames: uint8 [B,H,W,3] (numpy / pinned CPU tensor / CUDA tensor) or a
        pre-processed fp32 [B,3,h,w] CUDA tensor.  One native cp_infer call for the
        whole batch.  Returns (poses [B,K,192], n_valid [B]) -- on the host when
        `to_host`, else as CUDA tensors.

        frames may also be a LIST of uint8 [H_b,W_b,3] frames of mixed sizes (numpy, CPU or CUDA tensors), with
        camera_matrix [3,3] or one per frame [B,3,3]: one ragged pre-process launch, one network + decode call, and
        every frame's records in its own pixels (its own c, s and meta row), exactly what run() gives for it.

        out: optional (poses, n_valid) CUDA tensors to write into (e.g. the views of a dist.PoseBuffer, so that the
        records land directly in the buffer of the all-gather / the pinned D2H copy).

        track=True (tracking models): the batch is B independent video streams, or SLOTS, and every call is their next
        frame.  The previous frames, the tracker state and the rendered previous-frame heat maps stay on the device;
        returns (tracks [B,T,320], n_tracks [B]) (layout: cp_track_field) instead.  pre_dets: None, or per slot the
        meta['pre_dets'] list of this frame (or None); frame_ids: per slot meta['id'] (needed with
        opt.gt_pre_hm_hmhp_first).  Per slot, seeding and the heat maps follow run(): seeded when its video starts and
        on ground-truth frames, drawn from the ground truth on those frames, empty with opt.empty_pre_hm.  A slot's
        video starts on its first frame after the state is made (first call, a new number of slots, reset_tracking()).
        Both forms go through one tracking step (`_track_step`); the array form is the case where every slot steps.
        With a list, a None frame idles its slot this call, new_video[i] starts a new video in slot i, and `out` (see
        `_run_slots`) is honoured; the array form ignores `out`.

        pixel_format="nv12" / "i420": the uint8 frames are YUV 4:2:0 as video decoders give them, uint8 [B,3H/2,W] (array
        form) or a list of uint8 [3H_b/2,W_b] (H and W even), converted on the device inside the pre-process: every
        result equals, bit for bit, that of the same call on cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420).  c, s and
        the meta rows come from the image size (H, W).  The camera formats "rgb24" (uint8 [B,H,W,3]), "rgba" / "bgra"
        ([B,H,W,4]) and "yuyv422" / "uyvy422" ([B,H,W,2], W even) are converted the same way, each bit for bit its
        cv2.cvtColor to BGR (COLOR_RGB2BGR, _RGBA2BGR, _BGRA2BGR, COLOR_YUV2BGR_YUYV, _UYVY).  So are the sensor
        formats, one uint8 plane per frame ([B,H,W] or a list of [H_b,W_b]): "gray" (COLOR_GRAY2BGR) and the Bayer
        mosaics "bayer_rggb8" / "bayer_bggr8" / "bayer_gbrg8" / "bayer_grbg8" (H and W at least 3), named after their
        top-left 2 x 2 block and demosaiced as cv2's bilinear COLOR_BayerBG2BGR / _RG / _GR / _GB.  With a list of frames,
        pixel_format may also be a list of one name per frame or slot (cameras of different kinds); a list of one name
        repeated is that name.

        distortion: the lens distortion of the cameras (lens.LensDistortion), one for every camera or a list of one per
        frame or slot, None for an undistorted camera.  A distorted camera's frames are undistorted inside the
        pre-process: its network input is, bit for bit, the normalised cv2.remap of the BGR frame through
        lens.undistort_map (built once per camera and kept on the device), and its meta row carries the
        new_camera_matrix K_new, so records are in the pixels of the undistorted image of camera K_new and poses in the
        camera frame.  Every result then equals that of the same call on those fp32 inputs with camera_matrix K_new.
        The array form goes through a frame table (cp_preprocess_remap) only when some camera is distorted.  Refused:
        distortion with pre-processed fp32 frames, and with the keep_res / fix_short pre-process."""
        if track and not getattr(self.opt, "tracking_task", False):
            raise ValueError("run_batch(track=True) needs a tracking model (opt.tracking_task)")
        if isinstance(frames, (list, tuple)):
            if pre_images is not None or pre_hms is not None or pre_hm_hp is not None:
                raise ValueError("run_batch(list): the previous frames and heat maps are kept per slot (track=True)")
            if track:
                return self._run_slots(frames, camera_matrix, to_host, out, pre_dets, frame_ids, new_video, pixel_format,
                                       distortion)
            if new_video is not None or pre_dets is not None or frame_ids is not None:
                raise ValueError("run_batch(list): new_video / pre_dets / frame_ids need track=True")
            dists = slot_distortions(distortion, len(frames))
            frames, pixel_format = jpeg_frames(frames, pixel_format)
            check_frames(frames, allow_idle=False, pixel_format=pixel_format)
            x, meta, _ = self._ragged_input(frames, camera_matrix, pixel_format, dists)
        else:
            if new_video is not None:
                raise ValueError("run_batch: new_video needs a list of slot frames")
            x, meta, c, s = self._array_input(frames, camera_matrix, pixel_format, distortion)
            B = x.shape[0]
            if track:
                pre_dets = self._slot_pre_dets(pre_dets, B)
                trans = affine_from_center_scale(c, s, x.shape[3], x.shape[2])
                return self._track_step(B, list(range(B)), x, self._meta_rows(meta), trans, None, pre_dets, frame_ids,
                                        to_host, None)
        eng = self.model.engine(x.shape[0], x.shape[2], x.shape[3], x.device)
        _, poses, n_valid = eng.infer(x, self._meta_rows(meta), decode_params(self.opt, test_scale=1.0), pre_images,
                                      pre_hms, pre_hm_hp, poses=out[0] if out is not None else None,
                                      n_valid=out[1] if out is not None else None)
        return _returned((poses, n_valid), to_host)

    def _array_input(self, frames, camera_matrix, pixel_format="bgr", distortion=None):
        """run_batch's array form: uint8 [B,H,W,3] frames, frames of another pixel_format (uint8 [B,3H/2,W], [B,H,W,C]) (or
        pre-processed fp32 [B,3,h,w]) -> (x [B,3,h,w] fp32 CUDA, meta rows [B,16] float64 host, c, s) with the fix_res
        affine of the image size; with a distorted camera (distortion), through _remap_input."""
        dev = self.opt.device
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        dists = slot_distortions(distortion, frames.shape[0] if frames.dim() else 0)
        if dists is not None:
            return self._remap_input(frames, camera_matrix, pixel_format, dists)
        if check_pixel_format(pixel_format) != "bgr":
            layout = frame_layout(pixel_format)
            if frames.dtype != torch.uint8 or frames.dim() != layout.count(",") + 2:
                raise ValueError("run_batch: %s frames are uint8 [B,%s, got %s %s"
                                 % (pixel_format, layout[1:], frames.dtype, tuple(frames.shape)))
            B = frames.shape[0]
            sh, sw = image_size(frames.shape[1:], pixel_format, "run_batch: each frame")
            fr = frames.to(dev, non_blocking=True).contiguous().reshape(-1)
            n = fr.numel() // max(B, 1)
            x = preprocess_formats(fr, np.arange(B, dtype=np.int64) * n, [(sh, sw)] * B, pixel_format, self.opt.input_h,
                                   self.opt.input_w, self.opt.mean, self.opt.std)
            c, s = np.array([sw / 2., sh / 2.], np.float32), float(max(sh, sw))
            iw, ih = sw, sh
        elif frames.dtype == torch.uint8:
            B, sh, sw, _ = frames.shape
            fr = frames.to(dev, non_blocking=True)
            x = preprocess(fr, self.opt.input_h, self.opt.input_w, self.opt.mean, self.opt.std)
            c, s = np.array([sw / 2., sh / 2.], np.float32), float(max(sh, sw))
            iw, ih = sw, sh
        else:
            x = frames.to(dev)
            B, _, ih, iw = x.shape
            c, s = np.array([iw / 2., ih / 2.], np.float32), float(max(ih, iw))
        meta = make_meta(B, c, s, iw, ih, camera_matrix).numpy()
        # the batched path pre-processes at scale 1 (what every shipped configuration uses); results of a multi-scale
        # opt are those of test_scales[0] (object_pose.py:188), which run() reproduces frame by frame
        if float(self.scales[0]) != 1.0:
            raise NotImplementedError("run_batch pre-processes at scale 1; use run() for test_scales[0] != 1")
        return x, meta, c, s

    def _remap_input(self, frames, camera_matrix, pixel_format, dists):
        """_array_input with distorted cameras: the uint8 frames of one size as a frame table, one cp_preprocess_remap
        launch (unmapped frames under the fix_res affine of the size, as the array form without distortion)."""
        self._check_undistort(pixel_format)
        if frames.dtype != torch.uint8:
            raise ValueError("run_batch: distortion undistorts camera frames (uint8); pre-processed fp32 input has no "
                             "frame to remap, got %s" % frames.dtype)
        layout = frame_layout(pixel_format)
        if frames.dim() != layout.count(",") + 2:
            raise ValueError("run_batch: %s frames are uint8 [B,%s, got %s" % (pixel_format, layout[1:], tuple(frames.shape)))
        B = frames.shape[0]
        sh, sw = image_size(frames.shape[1:], pixel_format, "run_batch: each frame")
        cams = camera_per_frame(camera_matrix, B)
        ih, iw = self.opt.input_h, self.opt.input_w
        maps = self._maps.maps(dists, cams, [(sh, sw)] * B, (ih, iw), self.opt.device)
        fr = frames.to(self.opt.device, non_blocking=True).contiguous().reshape(-1)
        n = fr.numel() // max(B, 1)
        x = preprocess_remap(fr, np.arange(B, dtype=np.int64) * n, [(sh, sw)] * B, pixel_format, maps, ih, iw,
                             self.opt.mean, self.opt.std)
        c, s = np.array([sw / 2., sh / 2.], np.float32), float(max(sh, sw))
        meta = make_meta(B, c, s, sw, sh, undistorted_cameras(dists, cams)).numpy()
        return x, meta, c, s

    def _check_undistort(self, pixel_format):
        """Refuses, before any device work, what the undistorting pre-process does not take."""
        if getattr(self.opt, "fix_short", 0) > 0 or not getattr(self.opt, "fix_res", True):
            raise NotImplementedError("run_batch: distortion undistorts into the fix_res input; the keep_res and "
                                      "fix_short pre-process take no distortion")
        if float(self.scales[0]) != 1.0:
            raise NotImplementedError("run_batch pre-processes at scale 1; use run() for test_scales[0] != 1")
        if not isinstance(pixel_format, (list, tuple)):
            check_pixel_format(pixel_format)

    # ------------------------------------------------------------------ ragged batches (lists of frames)
    def _ragged_input(self, frames, camera_matrix, pixel_format="bgr", dists=None):
        """Validated list of uint8 HWC frames (or frames of pixel_format: one name, or one per frame) -> (x [B,3,h,w]
        fp32 CUDA, meta rows [B,16] float64 host, trans_input [B,2,3] host).  The frames are copied into one device
        buffer and pre-processed by one cp_preprocess_formats launch with the same fix_res affine (c = image centre,
        s = max side) and meta row that pre_process / run() use.  dists (slot_distortions, one per frame): one
        cp_preprocess_remap launch instead, the distorted frames through their maps and with K_new in their meta rows."""
        if getattr(self.opt, "fix_short", 0) > 0 or not getattr(self.opt, "fix_res", True):
            raise NotImplementedError("run_batch(list) pre-processes in the fix_res mode only")
        if float(self.scales[0]) != 1.0:
            raise NotImplementedError("run_batch pre-processes at scale 1; use run() for test_scales[0] != 1")
        B = len(frames)
        cams = camera_per_frame(camera_matrix, B)
        fmts = slot_formats(pixel_format, B)
        if dists is not None:
            self._check_undistort(pixel_format)
        dev = self.opt.device
        ih, iw = self.opt.input_h, self.opt.input_w
        ts, hw, offs, off = [], np.zeros((B, 2), np.int32), np.zeros(B, np.int64), 0
        for b, f in enumerate(frames):
            t = torch.from_numpy(f) if isinstance(f, np.ndarray) else f
            ts.append(t)
            hw[b] = image_size(t.shape, fmts[b])
            offs[b] = off
            off += int(np.prod(t.shape))
        if self._packed is None or self._packed.numel() < off or self._packed.device != torch.device(dev):
            self._packed = torch.empty((max(off, 1),), dtype=torch.uint8, device=dev)
        for t, o in zip(ts, offs):
            if not isinstance(t, JpegFrame):
                self._packed[o:o + t.numel()].copy_(t.reshape(-1), non_blocking=True)
        self._decode_jpegs(frames, offs)
        trans = np.zeros((B, 2, 3), np.float64)
        meta = np.zeros((B, _lib.CP_META_DOUBLES), np.float64)
        for b in range(B):
            h, w = int(hw[b, 0]), int(hw[b, 1])
            c, sc = np.array([w / 2., h / 2.], np.float32), float(max(h, w))
            if (h, w) not in self._affines:
                self._affines[(h, w)] = affine_from_center_scale(c, sc, iw, ih)
            trans[b] = self._affines[(h, w)]
            meta[b] = make_meta(1, c, sc, w, h, cams[b] if dists is None else undistorted_cameras(dists[b:b + 1],
                                                                                                 cams[b:b + 1])).numpy()[0]
        if dists is None:
            x = preprocess_formats(self._packed, offs, hw, fmts, ih, iw, self.opt.mean, self.opt.std, trans_input=trans)
        else:
            maps = self._maps.maps(dists, cams, [tuple(v) for v in hw], (ih, iw), dev)
            x = preprocess_remap(self._packed, offs, hw, fmts, maps, ih, iw, self.opt.mean, self.opt.std,
                                 trans_input=trans)
        return x, meta, trans

    def _decode_jpegs(self, frames, offs):
        """The JpegFrames among frames decoded by one cp_jpeg_decode, frame b into self._packed at offs[b] as BGR.  A
        corrupt bitstream raises ValueError naming the frame (one small copy back of the error words)."""
        idx = [b for b, f in enumerate(frames) if isinstance(f, JpegFrame)]
        if not idx:
            return
        data = np.concatenate([frames[b].data for b in idx])
        starts = np.cumsum([0] + [len(frames[b].data) for b in idx[:-1]])
        enc = torch.from_numpy(data).to(self.opt.device, non_blocking=True)
        errors = jpeg_decode([frames[b].header for b in idx], enc, starts, self._packed, [offs[b] for b in idx])
        bad = errors.cpu().numpy()
        for k, b in enumerate(idx):
            if bad[k]:
                raise ValueError("run_batch: frame %d is a corrupt JPEG (%s)" % (b, jpeg_error_text(bad[k])))

    def _meta_rows(self, meta):
        """Host meta rows -> a device tensor, uploaded again only when the rows change (a fixed frame size and camera
        are uploaded once)."""
        key = meta.tobytes()
        if self._meta_key != key:
            self._meta_dev = torch.from_numpy(meta).to(self.opt.device)
            self._meta_key = key
        return self._meta_dev

    def _run_slots(self, frames, camera_matrix, to_host, out, pre_dets, frame_ids, new_video, pixel_format="bgr",
                   distortion=None):
        """run_batch(list, track=True): frames[i] is the next frame of the video in slot i, or None when slot i is idle
        this step (its tracker stream is not stepped and keeps its state).  new_video[i] marks the first frame of a
        video in slot i, which then behaves exactly like the first run() call of a fresh detector: the stream is reset,
        the frame is its own previous frame, it is seeded from pre_dets[i] when given, and its heat maps follow
        opt.gt_pre_hm_hmhp* / opt.empty_pre_hm.  Only the live slots go through the network (as one batch).

        Returns (tracks [S,T,320], n_tracks [S]) for the S slots, idle slots with n_tracks 0 and zero rows; out:
        optional (tracks, n_tracks) CUDA tensors of those shapes to write into."""
        S = len(frames)
        dists = slot_distortions(distortion, S)
        frames, pixel_format = jpeg_frames(frames, pixel_format)
        if dists is not None:
            self._check_undistort(pixel_format)
        check_frames(frames, allow_idle=True, pixel_format=pixel_format)
        cams = camera_per_frame(camera_matrix, S)
        new_video = check_slot_list(new_video, S, "new_video", bool)
        pre_dets = self._slot_pre_dets(pre_dets, S)
        frame_ids = check_slot_list(frame_ids, S, "frame_ids")
        out = self._track_out(out, S)
        live = [i for i in range(S) if frames[i] is not None]
        if not live:
            out[0].zero_()
            out[1].zero_()
            return _returned(out, to_host)
        fmts = slot_formats(pixel_format, S)
        x, meta, trans = self._ragged_input([frames[i] for i in live], np.stack([cams[i] for i in live]),
                                            [fmts[i] for i in live],
                                            slot_distortions([dists[i] for i in live], len(live)) if dists else None)
        return self._track_step(S, live, x, self._meta_rows(meta), trans, new_video, pre_dets, frame_ids, to_host, out)

    # ---- what a tracking step does per category: one category here; MultiCategoryTracker runs several through the
    # same step (_track_step) by overriding these
    def _track_categories(self):
        """None: one category, opt.c (outputs [S, ...]); else the categories of the step (outputs [M, S, ...])."""
        return None

    def _track_engine(self, S, x):
        """(the plan, its decode parameters) of a tracking step of S slots at the network input size of x."""
        return self.model.engine(S, x.shape[2], x.shape[3], x.device), decode_params(self.opt, test_scale=1.0)

    def _slot_pre_dets(self, pre_dets, S):
        """run_batch's pre_dets, checked: None or, per slot, a list of pre_dets dicts (or None)."""
        return check_slot_list(pre_dets, S, "pre_dets")

    def _cat_pre_dets(self, pre_dets):
        """Checked pre_dets -> one per-slot list (or None) per category."""
        return [pre_dets]

    def _track_out(self, out, S):
        """The (tracks, n_tracks) CUDA tensors a step of S slots writes: `out` when given (checked), else new ones."""
        lead = (S,) if self._track_categories() is None else (len(self._track_categories()), S)
        dev, T = self.opt.device, _lib.CP_MAX_K
        if out is None:
            return (torch.empty(lead + (T, _lib.CP_TRACK_RECORD), dtype=torch.float32, device=dev),
                    torch.empty(lead, dtype=torch.int32, device=dev))
        if (tuple(out[0].shape) != lead + (T, _lib.CP_TRACK_RECORD) or tuple(out[1].shape) != lead
                or out[0].dtype != torch.float32 or out[1].dtype != torch.int32):
            raise ValueError("run_batch: out must be (tracks %s fp32, n_tracks %s int32)"
                             % (list(lead + (T, _lib.CP_TRACK_RECORD)), list(lead)))
        return out

    def _track_step(self, S, live, x, metat, trans, new_video, pre_dets, frame_ids, to_host, out):
        """One tracking step of S slots, both forms of run_batch(track=True).  Row k of x (network input [n,3,h,w]),
        metat (device meta rows [n,16]) and trans (trans_input, [n,2,3] or one [2,3] for all) is the next frame of slot
        live[k]; new_video / pre_dets / frame_ids: None or per slot (pre_dets as _slot_pre_dets returns it).  Writes
        (tracks [S,T,320], n_tracks [S]) into out (None: new tensors; only when every slot is live), slots not in
        `live` with n_tracks 0 and zero rows.  With several categories (_track_categories) every category steps the same
        slots: tracker stream m * S + s, outputs [M, S, ...], one render, one network call and one tracker step for all."""
        cats = self._track_categories()
        M = 1 if cats is None else len(cats)
        if self._slots is None or self._slots.streams != S:
            self._slots = _SlotState(self.opt, S, self.opt.device, categories=cats)
        st = self._slots
        trk = st.tracker
        # looked up before the render, whose trans_input upload waits for the device: host work between that upload and
        # the network launch would leave the GPU idle
        eng, prm = self._track_engine(S, x)
        # previous frames of another size (an fp32 array input that changed size): every slot takes this frame as its
        # previous frame and is seeded as at a start, but keeps its tracks
        resized = st.pre is not None and st.pre.shape[1:] != x.shape[1:]
        if resized and len(live) < S:
            raise ValueError("run_batch: the network input changed size from %s to %s while slots are idle"
                             % (tuple(st.pre.shape[2:]), tuple(x.shape[2:])))
        new = [not st.started[i] or (new_video is not None and new_video[i]) for i in live]
        starts = [n or resized for n in new]
        seeds, modes = [None] * (M * S), []
        for m, pd in enumerate(self._cat_pre_dets(pre_dets)):
            for k, i in enumerate(live):
                seeds[m * S + i], mode = self._track_policy(starts[k], frame_ids[i] if frame_ids is not None else None,
                                                            pd[i] if pd is not None else None)
                modes.append(mode)
        for k, i in enumerate(live):
            if new[k]:                                        # base_detector.py:444-449: a fresh stream
                for m in range(M):
                    trk.reset(m * S + i)
                st.started[i] = True
        trk.seed(seeds)
        all_live = len(live) == S                             # every slot, in order: stream map NULL (the identity)
        if all(starts):
            pre = x
        elif all_live and not any(starts):
            pre = st.pre
        else:
            pre = torch.stack([x[k] if starts[k] else st.pre[i] for k, i in enumerate(live)])
        n = len(live)
        ids = None if all_live else [m * S + i for m in range(M) for i in live]
        if M > 1:            # one render of every category's images (category m's are rows m * n ...), one meta row each
            metat = metat.repeat(M, 1)
            if np.asarray(trans).ndim == 3:
                trans = np.tile(trans, (M, 1, 1))
        pre_hms, pre_hm_hp = trk.render(metat, trans, x.shape[2], x.shape[3], modes=modes, stream_ids=ids)
        if M > 1:
            pre_hms, pre_hm_hp = pre_hms.view((M, n) + pre_hms.shape[1:]), pre_hm_hp.view((M, n) + pre_hm_hp.shape[1:])
        _, poses, n_valid = eng.infer(x, metat[:n], prm, pre, pre_hms, pre_hm_hp)
        poses, n_valid = poses.reshape((M * n,) + poses.shape[-2:]), n_valid.reshape(M * n)
        if cats is not None:
            out = self._track_out(out, S) if out is not None or not all_live else out
        if all_live and cats is None:
            out = trk.step_records(poses, n_valid, metat, out=out)
            st.pre = x
        elif all_live:                                        # [M, S, ...] is the tracker's stream order
            flat = None if out is None else (out[0].view((M * S,) + out[0].shape[-2:]), out[1].view(M * S))
            flat = trk.step_records(poses, n_valid, metat, out=flat)
            out = out if out is not None else (flat[0].view((M, S) + flat[0].shape[1:]), flat[1].view(M, S))
            st.pre = x
        else:
            tr, nt = trk.step_records(poses, n_valid, metat, stream_ids=ids)
            row = {i: k for k, i in enumerate(live)}
            old = st.pre if st.pre is not None else x.new_zeros((S,) + tuple(x.shape[1:]))
            st.pre = torch.stack([x[row[i]] if i in row else old[i] for i in range(S)])
            zt, zn = tr.new_zeros(tr.shape[1:]), nt.new_zeros(())
            outs = [out] if cats is None else [(out[0][m], out[1][m]) for m in range(M)]
            for m, (o_tr, o_nt) in enumerate(outs):
                torch.stack([tr[m * n + row[i]] if i in row else zt for i in range(S)], out=o_tr)
                torch.stack([nt[m * n + row[i]] if i in row else zn for i in range(S)], out=o_nt)
        return _returned(out, to_host)

    def reset_tracking(self):
        """base_detector.py:774-776."""
        if self.tracker is not None:
            self.tracker.reset()
        self.pre_images = None
        self._slots = None


detector_factory = {"object_pose": ObjectPoseDetector}


# ----------------------------------------------------------------------------- several categories at once
class MultiCategoryDetector(ObjectPoseDetector):
    """One checkpoint per object category (upstream publishes one per category), all run over the same frames by one
    multi-model plan: every layer is one launch for all categories, followed by one decode.

    checkpoints: ordered mapping category -> checkpoint path, loaded with load_model (and its weights_only rule).  All
    checkpoints must have opt's architecture, heads and head_conv.  Category c decodes with decode_params(opt, c=c)
    (its visible_thresh and balance coefficient).  Only run_batch is offered: tracking, run(), process() and the result
    writers are single-category and raise here.  The checkpoints' weights stay on the host; on the device they exist
    only in the plan."""

    def __init__(self, opt, checkpoints):
        if getattr(opt, "tracking_task", False):
            raise ValueError("MultiCategoryDetector: tracking several categories runs through MultiCategoryTracker")
        _load_categories(self, opt, checkpoints, "MultiCategoryDetector")

    def engine(self, batch, height, width):
        """The multi-model plan for this input shape (created on first use, rebuilt for a larger batch), its activation
        arena packed by liveness (Engine reuse_activations)."""
        eng = self._eng
        if eng is None or eng.max_batch < batch or (eng.height, eng.width) != (height, width):
            if eng is not None:
                eng.close()
            dev = torch.device(self.opt.device)
            c = self._plan_cfg
            eng = Engine(c["arch"], c["heads"], c["head_conv"], max(batch, 1), height, width,
                         dev.index if dev.index is not None else torch.cuda.current_device(), tracking=c["tracking"],
                         tracking_task_gru=c["tracking_task_gru"], precision=c["precision"], models=len(self._weights),
                         reuse_activations=True, batch_invariant=c["batch_invariant"])
            for i, sd in enumerate(self._weights):
                eng.load_state_dict(sd, model=i)
            self._eng = eng
        return eng

    def run_batch(self, frames, camera_matrix, to_host=True, out=None, pixel_format="bgr", distortion=None):
        """run_batch of ObjectPoseDetector (a uint8 [B,H,W,3] array, or a list of mixed-size frames with one camera or
        one per frame; YUV 4:2:0 and camera formats with pixel_format, a list of names with a list of frames, and lens
        distortion with distortion, as there) for every category: the frames are pre-processed once.  Returns (poses [M,B,K,192], n_valid [M,B]) in `categories` order, also for M = 1; out:
        optional (poses, n_valid) CUDA tensors of those shapes to write into."""
        if isinstance(frames, (list, tuple)):
            dists = slot_distortions(distortion, len(frames))
            frames, pixel_format = jpeg_frames(frames, pixel_format)
            check_frames(frames, allow_idle=False, pixel_format=pixel_format)
            x, meta, _ = self._ragged_input(frames, camera_matrix, pixel_format, dists)
        else:
            x, meta, _, _ = self._array_input(frames, camera_matrix, pixel_format, distortion)
        eng = self.engine(x.shape[0], x.shape[2], x.shape[3])
        if len(self._prms) > 1:
            _, poses, n_valid = eng.infer(x, self._meta_rows(meta), self._prms,
                                          poses=out[0] if out is not None else None,
                                          n_valid=out[1] if out is not None else None)
        else:             # a one-model plan: cp_infer, outputs [B, ...] -> [1, B, ...]
            _, poses, n_valid = eng.infer(x, self._meta_rows(meta), self._prms[0],
                                          poses=out[0][0] if out is not None else None,
                                          n_valid=out[1][0] if out is not None else None)
            poses, n_valid = out if out is not None else (poses.unsqueeze(0), n_valid.unsqueeze(0))
        return _returned((poses, n_valid), to_host)


class MultiCategoryTracker(MultiCategoryDetector):
    """The tracking counterpart of MultiCategoryDetector: M CenterPoseTrack checkpoints (one per category, loaded and
    checked the same way) track their objects in the same S video slots.  One step is one pre-process, one render of
    every category's previous-frame heat maps, one multi-model network + decode call (cp_infer_multi_track) and one
    tracker step over the M x S streams (cp_tracker_create_multi); the previous frames are shared by the categories.
    Category c tracks with its visible_thresh, balance coefficient and opt.conf_border[c] (when conf_border is a dict).
    The slot policy (starts, seeding, render modes, previous frames) is that of ObjectPoseDetector.run_batch(track=True),
    run per category.  Not supported: opt.refined_Kalman and test_scales other than [1]."""

    def __init__(self, opt, checkpoints):
        if not getattr(opt, "tracking_task", False):
            raise ValueError("MultiCategoryTracker needs a tracking opt (opt.tracking_task); detection of several "
                             "categories runs through MultiCategoryDetector")
        if getattr(opt, "refined_Kalman", False):
            raise NotImplementedError("opt.refined_Kalman (utils/tracker_baseline.py, CenterPose + Kalman baseline) is not "
                                      "on the accelerated path; use --tracking_task (CenterPoseTrack)")
        if [float(v) for v in getattr(opt, "test_scales", [1.0])] != [1.0]:
            raise NotImplementedError("CenterPoseTrack runs at test_scales=[1] (the reference re-initialises the tracker "
                                      "state once per scale, base_detector.py:440-449)")
        _load_categories(self, opt, checkpoints, "MultiCategoryTracker")
        if not self._plan_cfg["tracking"]:
            raise ValueError("MultiCategoryTracker: the tracking model needs the pre_img / pre_hm / pre_hm_hp inputs")
        if self.tracker is not None:                # ObjectPoseDetector's one-stream tracker: the slots have their own
            self.tracker.close()
            self.tracker = None

    def run_batch(self, frames, camera_matrix, new_video=None, pre_dets=None, frame_ids=None, to_host=True, out=None,
                  pixel_format="bgr", distortion=None):
        """The next frame of every slot, for every category.  frames: uint8 [S,H,W,3] (every slot steps), or a list of S
        uint8 [H_s,W_s,3] frames of mixed sizes where None idles a slot this step, with camera_matrix [3,3] or one per
        slot.  new_video[i]: slot i starts a new video (every category).  pre_dets: None, or a mapping category -> per
        slot list of meta['pre_dets'] lists (None = that slot is not seeded); frame_ids: per slot meta['id'].
        Returns (tracks [M,S,T,320], n_tracks [M,S]) in `categories` order (idle slots: n_tracks 0, zero rows), on the
        host when `to_host`; out: optional (tracks, n_tracks) CUDA tensors of those shapes to write into.
        pixel_format "nv12" / "i420": YUV 4:2:0 frames, uint8 [S,3H/2,W] or [3H_s/2,W_s]; the camera and sensor
        formats, one name per slot with a list of frames, and distortion (one LensDistortion, or one per slot), as in
        ObjectPoseDetector.run_batch."""
        if isinstance(frames, (list, tuple)):
            return self._run_slots(frames, camera_matrix, to_host, out, pre_dets, frame_ids, new_video, pixel_format,
                                   distortion)
        if new_video is not None:
            raise ValueError("run_batch: new_video needs a list of slot frames")
        x, meta, c, s = self._array_input(frames, camera_matrix, pixel_format, distortion)
        S = x.shape[0]
        pre_dets = self._slot_pre_dets(pre_dets, S)
        frame_ids = check_slot_list(frame_ids, S, "frame_ids")
        trans = affine_from_center_scale(c, s, x.shape[3], x.shape[2])
        return self._track_step(S, list(range(S)), x, self._meta_rows(meta), trans, None, pre_dets, frame_ids, to_host,
                                self._track_out(out, S) if out is not None else None)

    def _track_categories(self):
        return self.categories

    def _track_engine(self, S, x):
        return self.engine(S, x.shape[2], x.shape[3]), (self._prms if len(self._prms) > 1 else self._prms[0])

    def _slot_pre_dets(self, pre_dets, S):
        if pre_dets is None:
            return None
        if not hasattr(pre_dets, "items"):
            raise ValueError("run_batch: pre_dets maps a category to its per-slot pre_dets lists")
        for c, v in pre_dets.items():
            if c not in self.categories:
                raise ValueError("run_batch: pre_dets for unknown category '%s' (categories: %s)" % (c, self.categories))
            if v is not None and len(list(v)) != S:
                raise ValueError("run_batch: pre_dets['%s'] has %d entries for %d slots" % (c, len(list(v)), S))
        return {c: (list(v) if v is not None else None) for c, v in pre_dets.items()}

    def _cat_pre_dets(self, pre_dets):
        return [(pre_dets or {}).get(c) for c in self.categories]

    def reset_tracking(self):
        """Forget every slot's tracks and previous frames (the next step starts every slot)."""
        self._slots = None


def _single_category(name):
    def refuse(self, *a, **k):
        raise NotImplementedError("%s.%s: only run_batch runs several categories; use an ObjectPoseDetector per "
                                  "category" % (type(self).__name__, name))
    refuse.__name__ = name
    return refuse


for _name in ("run", "process", "pre_process", "build_dict_out", "show_results", "save_results", "save_results_eval"):
    setattr(MultiCategoryDetector, _name, _single_category(_name))
setattr(MultiCategoryDetector, "reset_tracking", _single_category("reset_tracking"))
del _name


def _load_categories(det, opt, checkpoints, who):
    """The shared set-up of MultiCategoryDetector / MultiCategoryTracker: checks the categories and checkpoints, loads
    every checkpoint to the host and makes `det` an ObjectPoseDetector of opt without a device model (the multi-model
    plan, created by det.engine, holds the weights)."""
    cats = list(checkpoints.keys())
    if not 1 <= len(cats) <= _lib.CP_MAX_MODELS:
        raise ValueError("%s: 1..%d categories, got %d" % (who, _lib.CP_MAX_MODELS, len(cats)))
    for c in cats:
        decode_params(opt, c=c)                  # raises on an unknown category
    weights = []
    for c in cats:
        m = create_model(opt.arch, opt.heads, opt.head_conv, opt)
        _check_checkpoint(m, checkpoints[c], c, who)
        m = load_model(m, checkpoints[c])
        weights.append({k: v.detach().cpu() for k, v in m.state_dict().items()})
    det._plan_cfg = dict(arch=m._arch(), heads=m.heads, head_conv=m.head_conv, tracking=m.tracking_inputs,
                         tracking_task_gru=m.use_convGRU and m.tracking_task, precision=m.precision,
                         batch_invariant=m.batch_invariant)
    base = copy.copy(opt)
    base.load_model = ""
    ObjectPoseDetector.__init__(det, base, model=m)
    det.model = None                             # the plan holds the weights; only the host copies are kept
    det.categories = cats
    det._weights = weights
    det._prms = [decode_params(opt, c=c, test_scale=1.0) for c in cats]
    det._eng = None


def _check_checkpoint(model, path, category, who="MultiCategoryDetector"):
    """The checkpoint must hold exactly the tensors of `model` (same architecture, heads and head_conv): one plan runs
    every category's weights through the same schedule."""
    sd = _load_checkpoint(path)["state_dict"]
    got = {(k[7:] if k.startswith("module") and not k.startswith("module_list") else k): tuple(v.shape)
           for k, v in sd.items()}
    want = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    if got != want:
        diff = sorted(set(got.items()) ^ set(want.items()))[:4]
        raise ValueError("%s: the checkpoint of '%s' (%s) does not match the architecture, heads and "
                         "head_conv of opt (first differences: %s)" % (who, category, path, diff))
