"""Lens distortion: camera frames undistorted inside the pre-process.

A calibrated camera is its intrinsics K (the distorted camera, ROS `CameraInfo.K`), its distortion coefficients D
(`CameraInfo.D`) in one of three models (`CameraInfo.distortion_model`), and the pinhole camera K_new its frames are
undistorted to (`CameraInfo.P`'s left 3 x 3; default K, as cv2.undistort).  For a frame of size (h, w) and a network
input of (ih, iw), the pre-process of that frame is one bilinear resampling through a coordinate map:

    A        = the fix_res trans_input of the frame size (c = (w/2, h/2), s = max(h, w))
    P        = [A; 0 0 1] @ K_new
    mx, my   = cv2.initUndistortRectifyMap(K, D, None, P, (iw, ih), CV_32FC1)              plumb_bob, rational_polynomial
             = cv2.fisheye.initUndistortRectifyMap(K, D, eye(3), P, (iw, ih), CV_32FC1)    equidistant
    input    = normalise(cv2.remap(frame as BGR, mx, my, INTER_LINEAR, BORDER_CONSTANT, 0))

so the network sees the undistorted image of camera K_new under the usual fix_res affine.  The meta row carries K_new,
and records come out in the pixels of that undistorted image.  The map is built on the host with cv2, once per camera
(`MapCache`), and read by the pre-process kernel at every output pixel.  This fused path resamples once; it is not bit
for bit cv2.undistort at full resolution followed by the affine pre-process, which resamples twice.
"""
import collections

import numpy as np
import torch

# distortion_model -> the coefficient counts it takes (ROS CameraInfo: plumb_bob k1 k2 t1 t2 k3; rational_polynomial
# k1 k2 t1 t2 k3 k4 k5 k6; equidistant k1 k2 k3 k4, cv2.fisheye's model)
MODELS = {"plumb_bob": (4, 5), "rational_polynomial": (8,), "equidistant": (4,)}


def _matrix3(K, what):
    K = np.asarray(K, np.float64)
    if K.shape != (3, 3) or not np.all(np.isfinite(K)):
        raise ValueError("%s must be a finite 3x3 matrix, got %s" % (what, K.shape if K.shape != (3, 3) else K.tolist()))
    return K


class LensDistortion(object):
    """The distortion of one camera: coeffs (ROS CameraInfo.D) in `model` ("plumb_bob": 4 or 5 coefficients,
    "rational_polynomial": 8, "equidistant": 4), and the camera matrix the frames are undistorted to,
    new_camera_matrix (the left 3x3 of CameraInfo.P; None: the camera's own K).  The intrinsics K come from the call's
    camera_matrix, so one LensDistortion serves every camera with the same lens."""

    def __init__(self, coeffs, model="plumb_bob", new_camera_matrix=None):
        if model not in MODELS:
            raise ValueError("LensDistortion: model must be one of %s, got %r" % (", ".join(MODELS), model))
        D = np.asarray(coeffs, np.float64)
        if D.ndim != 1 or D.shape[0] not in MODELS[model]:
            raise ValueError("LensDistortion: %s takes %s coefficients, got shape %s"
                             % (model, " or ".join(str(n) for n in MODELS[model]), D.shape))
        if not np.all(np.isfinite(D)):
            raise ValueError("LensDistortion: the coefficients must be finite, got %s" % D.tolist())
        self.coeffs, self.model = D, model
        self.new_camera_matrix = None if new_camera_matrix is None else _matrix3(new_camera_matrix,
                                                                                "LensDistortion: new_camera_matrix")

    def __repr__(self):
        return "LensDistortion(%s, model=%r%s)" % (self.coeffs.tolist(), self.model, "" if self.new_camera_matrix is None
                                                   else ", new_camera_matrix=%s" % self.new_camera_matrix.tolist())

    def camera(self, K):
        """The camera matrix of the undistorted frames of a camera with intrinsics K (the meta row's camera)."""
        return _matrix3(K, "camera_matrix") if self.new_camera_matrix is None else self.new_camera_matrix

    def key(self, K, frame_hw, input_hw):
        """What the map of a camera with intrinsics K depends on."""
        return (np.asarray(K, np.float64).tobytes(), self.coeffs.tobytes(), self.model, self.camera(K).tobytes(),
                tuple(int(v) for v in frame_hw), tuple(int(v) for v in input_hw))


def undistort_map(dist, K, frame_hw, input_hw):
    """float32 [ih, iw, 2]: the (x, y) source position in a frame of size frame_hw of every network input pixel, the
    recipe of the module docstring (cv2 builds it)."""
    import cv2
    from .detector import affine_from_center_scale
    K = _matrix3(K, "camera_matrix")
    (h, w), (ih, iw) = (int(v) for v in frame_hw), (int(v) for v in input_hw)
    A = affine_from_center_scale(np.array([w / 2., h / 2.], np.float32), float(max(h, w)), iw, ih)
    P = np.vstack([A, [0.0, 0.0, 1.0]]) @ dist.camera(K)
    if dist.model == "equidistant":
        mx, my = cv2.fisheye.initUndistortRectifyMap(K, dist.coeffs, np.eye(3), P, (iw, ih), cv2.CV_32FC1)
    else:
        mx, my = cv2.initUndistortRectifyMap(K, dist.coeffs, None, P, (iw, ih), cv2.CV_32FC1)
    return np.ascontiguousarray(np.stack([mx, my], axis=-1), np.float32)


def slot_distortions(distortion, n, who="run_batch"):
    """distortion of n frames or slots -> None (no camera is distorted: the launches and bits of a call without it), or
    a list of n LensDistortion / None.  distortion: None, one LensDistortion for every camera, or a list of n."""
    if distortion is None:
        return None
    if isinstance(distortion, LensDistortion):
        return [distortion] * n
    if not isinstance(distortion, (list, tuple)):
        raise TypeError("%s: distortion is a LensDistortion or a list of one per frame or slot, got %s"
                        % (who, type(distortion).__name__))
    if len(distortion) != n:
        raise ValueError("%s: distortion is one LensDistortion or one per frame or slot, got %d for %d"
                         % (who, len(distortion), n))
    for d in distortion:
        if d is not None and not isinstance(d, LensDistortion):
            raise TypeError("%s: a distortion entry is a LensDistortion or None, got %s" % (who, type(d).__name__))
    return None if all(d is None for d in distortion) else list(distortion)


class MapCache(object):
    """Device maps (undistort_map) keyed by camera, lens, frame size and input size, built on first use.  Holds at
    most `capacity` maps (2 MB each at 512 x 512), dropping the least recently used; a dropped map is freed in stream
    order, after the launches already enqueued on the current stream."""

    def __init__(self, capacity=64):
        self.capacity = int(capacity)
        self._maps = collections.OrderedDict()

    def get(self, dist, K, frame_hw, input_hw, device):
        key = dist.key(K, frame_hw, input_hw) + (str(torch.device(device)),)
        m = self._maps.get(key)
        if m is None:
            m = torch.from_numpy(undistort_map(dist, K, frame_hw, input_hw)).to(device)
            self._maps[key] = m
            while len(self._maps) > self.capacity:
                self._maps.popitem(last=False)
        else:
            self._maps.move_to_end(key)
        return m

    def maps(self, dists, cams, frame_hws, input_hw, device):
        """One map per frame (None where dists[b] is None)."""
        return [None if d is None else self.get(d, cams[b], frame_hws[b], input_hw, device) for b, d in enumerate(dists)]


def undistorted_cameras(dists, cams):
    """The meta rows' cameras: K_new for a distorted camera, K for the others."""
    return np.stack([np.asarray(K, np.float64) if d is None else d.camera(K) for d, K in zip(dists, cams)])
