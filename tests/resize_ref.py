"""TEST INFRASTRUCTURE ONLY -- a numpy restatement of cv2.resize(src, (rw, rh)) (INTER_LINEAR) for uint8 images, the
rule the device resize fetch (ResizeFetch, csrc/ext_ops.cu) is held to.  OpenCV resize.cpp, third party:
opencv-python 4.13.0; INTER_RESIZE_COEF_BITS = 11, so the weights are integers summing to COEF_SCALE = 2048:
  * per axis, scale = 1 / (dst / src) in double; destination index d has
    f = (float)((d + 0.5) * scale - 0.5), s = floor(f), f -= s (float32),
    a0 = round_half_even((1 - f) * 2048), a1 = round_half_even(f * 2048) (float32 products);
  * horizontal: s < 0 -> s = 0, f = 0; s >= sw - 1 -> s = sw - 1, f = 0 (the second tap then has weight 0);
    S = src[s] a0 + src[s + 1] a1 as an int;
  * vertical: f is NOT clamped; the rows s and s + 1 are each clamped to [0, sh - 1];
    value = sat_u8((((b0 (S0 >> 4)) >> 16) + ((b1 (S1 >> 4)) >> 16) + 2) >> 2) (VResizeLinear<uchar>);
  * an unchanged size is a copy; a downscale to exactly one half follows the same rule."""
import numpy as np

COEF_SCALE = 2048


def axis_taps(src, dst):
    """(s int64, a0 int32, a1 int32) [dst] of one axis before any clamping: the first source index, the two weights."""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f)
    f = (f - s).astype(np.float32)
    a0 = np.rint((np.float32(1) - f) * np.float32(COEF_SCALE)).astype(np.int64)
    a1 = np.rint(f * np.float32(COEF_SCALE)).astype(np.int64)
    return s.astype(np.int64), a0.astype(np.int32), a1.astype(np.int32)


def resize_u8(src, rw, rh):
    """uint8 [sh, sw] or [sh, sw, C] -> uint8 [rh, rw(, C)], bit for bit cv2.resize(src, (rw, rh))."""
    src = np.asarray(src)
    if src.dtype != np.uint8 or src.ndim not in (2, 3):
        raise ValueError("resize_u8: expected a uint8 [H, W] or [H, W, C] image, got %s %s" % (src.dtype, src.shape))
    sh, sw = src.shape[:2]
    if rw <= 0 or rh <= 0 or sh <= 0 or sw <= 0:
        raise ValueError("resize_u8: sizes must be positive, got %d x %d -> %d x %d" % (sh, sw, rh, rw))
    if (rh, rw) == (sh, sw):
        return src.copy()
    v = src.astype(np.int32)                     # every product below fits: 2048 * (255 * 2048 >> 4) < 2^31
    # horizontal pass on every source row
    sx, a0, a1 = axis_taps(sw, rw)
    lo, hi = sx < 0, sx >= sw - 1
    sx = np.where(lo, 0, np.where(hi, sw - 1, sx))
    a0 = np.where(lo | hi, COEF_SCALE, a0)
    a1 = np.where(lo | hi, 0, a1)
    x1 = np.minimum(sx + 1, sw - 1)              # read only where a1 is 0
    ex = (slice(None),) + (None,) * (src.ndim - 2)
    S = v[:, sx] * a0[ex] + v[:, x1] * a1[ex]
    # vertical pass: rows clamped, weights not
    sy, b0, b1 = axis_taps(sh, rh)
    y0, y1 = np.clip(sy, 0, sh - 1), np.clip(sy + 1, 0, sh - 1)
    ey = (slice(None), None) + (None,) * (src.ndim - 2)
    out = (((b0[ey] * (S[y0] >> 4)) >> 16) + ((b1[ey] * (S[y1] >> 4)) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)
