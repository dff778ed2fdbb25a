"""TEST INFRASTRUCTURE ONLY -- the phone camera formats: YUV 4:2:0 with the chroma swapped (NV21, YV12) and in full range
(nv12_full, nv21_full, i420_full, yv12_full), the references the device pre-process of those frames is held to.

Every format is a uint8 [3H/2, W] frame, H and W even: the Y plane, then the chroma of each 2x2 block as NV12 (U V
interleaved), NV21 (V U interleaved), I420 (the U plane, then the V plane) or YV12 (the V plane, then the U plane).

  * Limited range (BT.601, "nv21", "yv12"): cv2.cvtColor with COLOR_YUV2BGR_NV21 / _YV12, which is NV12 / I420 on the
    frame with its chroma swapped (yuv_ref.yuv420_to_bgr restates that in numpy).
  * Full range (JFIF, the "_full" names) has no 4:2:0 code in cv2.  It is each pixel taking the Cb, Cr of its 2x2
    block, then cv2.cvtColor(np.dstack([Y, Cr, Cb]), COLOR_YCrCb2BGR), which on every (Y, Cr, Cb) is exactly
      R = sat(Y + (((Cr - 128) 22987 + 2^13) >> 14)), G = sat(Y + (((Cr - 128) (-11698) + (Cb - 128) (-5636) + 2^13) >> 14)),
      B = sat(Y + (((Cb - 128) 29049 + 2^13) >> 14))   (arithmetic shift, sat to 0..255)
    (pinned against cv2 on all 2^24 triples in tests/test_phone_formats_cpu.py)."""
import numpy as np

from tests import yuv_ref

FORMATS = ("nv21", "yv12", "nv12_full", "nv21_full", "i420_full", "yv12_full")
LAYOUTS = ("nv12", "i420", "nv21", "yv12")
CV2_CODES = {"nv12": "COLOR_YUV2BGR_NV12", "i420": "COLOR_YUV2BGR_I420", "nv21": "COLOR_YUV2BGR_NV21",
             "yv12": "COLOR_YUV2BGR_YV12"}


def layout(fmt):
    """The byte layout of a 4:2:0 format: "nv12", "i420", "nv21" or "yv12"."""
    lay = fmt[:-5] if fmt.endswith("_full") else fmt
    if lay not in LAYOUTS:
        raise ValueError("phone_ref: unknown format %r" % (fmt,))
    return lay


def is_full(fmt):
    layout(fmt)
    return fmt.endswith("_full")


def planes(buf, fmt):
    """uint8 [3H/2, W] frame in fmt -> (Y [H, W], U [H/2, W/2], V [H/2, W/2])."""
    buf = np.asarray(buf)
    rows, W = buf.shape
    H = rows * 2 // 3
    if buf.dtype != np.uint8 or rows % 3 or H % 2 or W % 2 or H < 2 or W < 2:
        raise ValueError("phone_ref: expected a uint8 [3H/2, W] frame with even H and W, got %s %s"
                         % (buf.dtype, buf.shape))
    lay, chroma = layout(fmt), buf[H:].reshape(-1)
    if lay in ("nv12", "nv21"):
        pairs = chroma.reshape(H // 2, W // 2, 2)
        a, b = pairs[..., 0], pairs[..., 1]
    else:
        n = (H // 2) * (W // 2)
        a, b = chroma[:n].reshape(H // 2, W // 2), chroma[n:].reshape(H // 2, W // 2)
    U, V = (b, a) if lay in ("nv21", "yv12") else (a, b)
    return buf[:H], U, V


def pack(Y, U, V, fmt):
    """The inverse of planes: a uint8 [3H/2, W] frame in fmt."""
    lay = layout(fmt)
    H, W = Y.shape
    a, b = (V, U) if lay in ("nv21", "yv12") else (U, V)
    if lay in ("nv12", "nv21"):
        chroma = np.stack([a, b], axis=-1).reshape(H // 2, W)
    else:
        chroma = np.concatenate([a.reshape(-1), b.reshape(-1)]).reshape(H // 2, W)
    return np.ascontiguousarray(np.concatenate([Y, chroma], axis=0), np.uint8)


def _up(p):
    return np.repeat(np.repeat(p, 2, axis=0), 2, axis=1)


def full_range_to_bgr(Y, Cb, Cr):
    """The full-range rule on per-pixel planes (any integer arrays of one shape) -> uint8 [..., 3] BGR."""
    Y, cb, cr = (np.asarray(v, np.int64) for v in (Y, Cb, Cr))
    cb, cr = cb - 128, cr - 128
    sat = lambda t: np.clip(t, 0, 255).astype(np.uint8)                                        # noqa: E731
    return np.stack([sat(Y + ((cb * 29049 + (1 << 13)) >> 14)),
                     sat(Y + ((cr * -11698 + cb * -5636 + (1 << 13)) >> 14)),
                     sat(Y + ((cr * 22987 + (1 << 13)) >> 14))], axis=-1)


def to_bgr(buf, fmt):
    """The numpy restatement: a frame in any 4:2:0 format (the eight names) -> uint8 [H, W, 3] BGR."""
    Y, U, V = planes(buf, fmt)
    if is_full(fmt):
        return full_range_to_bgr(Y, _up(U), _up(V))
    lay = layout(fmt)
    base = "nv12" if lay in ("nv12", "nv21") else "i420"
    return yuv_ref.yuv420_to_bgr(pack(Y, U, V, base), base)


def cv2_bgr(buf, fmt):
    """The cv2 oracle of a frame in any 4:2:0 format: cv2.cvtColor with the format's code, or (full range) with
    COLOR_YCrCb2BGR on the planes with each block's chroma replicated."""
    import cv2
    buf = np.ascontiguousarray(buf)
    if not is_full(fmt):
        return cv2.cvtColor(buf, getattr(cv2, CV2_CODES[layout(fmt)]))
    Y, U, V = planes(buf, fmt)
    return cv2.cvtColor(np.ascontiguousarray(np.dstack([Y, _up(V), _up(U)])), cv2.COLOR_YCrCb2BGR)


def from_bgr(bgr, fmt):
    """A BGR image (even H and W) as a camera in fmt would deliver it: limited range through cv2's COLOR_BGR2YUV_I420,
    full range through COLOR_BGR2YCrCb with each 2x2 block's chroma averaged (rounded)."""
    import cv2
    bgr = np.ascontiguousarray(bgr)
    H, W = bgr.shape[:2]
    if is_full(fmt):
        ycc = cv2.cvtColor(bgr, cv2.COLOR_BGR2YCrCb).astype(np.int64)
        block = lambda p: ((p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + 2) >> 2)   # noqa: E731
        return pack(ycc[..., 0].astype(np.uint8), block(ycc[..., 2]).astype(np.uint8),
                    block(ycc[..., 1]).astype(np.uint8), fmt)
    return pack(*planes(cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420), "i420"), fmt)


def exhaustive_triples():
    """uint8 [4096, 4096, 3] holding every (Y, Cr, Cb) triple once, in cv2's YCrCb channel order."""
    i = np.arange(1 << 24, dtype=np.int64)
    return np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)
