"""TEST INFRASTRUCTURE ONLY -- numpy restatements of cv2's conversions to BGR of the camera formats the pre-process takes
besides BGR and YUV 4:2:0 (packed RGB / RGBA / BGRA and packed YUV 4:2:2), the references the device pre-process of
those frames is held to.  With the warp restatement in oracle/preprocess_ref.py they give the network input of such a
frame without cv2.  Formats carry ffmpeg's pix_fmt names, as pixel_format does."""
import numpy as np

# the cv2.cvtColor code that takes each format to BGR
CV2_CODES = {"rgb24": "COLOR_RGB2BGR", "rgba": "COLOR_RGBA2BGR", "bgra": "COLOR_BGRA2BGR",
             "yuyv422": "COLOR_YUV2BGR_YUYV", "uyvy422": "COLOR_YUV2BGR_UYVY"}
CHANNELS = {"rgb24": 3, "rgba": 4, "bgra": 4, "yuyv422": 2, "uyvy422": 2}
# byte of B, G and R in a packed RGB pixel
_BGR_BYTES = {"rgb24": (2, 1, 0), "rgba": (2, 1, 0), "bgra": (0, 1, 2)}


def packed_to_bgr(buf, fmt):
    """uint8 [H, W, 3 | 4] RGB24 / RGBA / BGRA frame -> uint8 [H, W, 3] BGR: cv2.cvtColor(buf, COLOR_RGB2BGR /
    COLOR_RGBA2BGR / COLOR_BGRA2BGR), a channel select (alpha is dropped)."""
    buf = np.asarray(buf)
    if fmt not in _BGR_BYTES:
        raise ValueError("packed_to_bgr: unknown format %r" % (fmt,))
    if buf.dtype != np.uint8 or buf.ndim != 3 or buf.shape[2] != CHANNELS[fmt]:
        raise ValueError("packed_to_bgr: expected a uint8 [H, W, %d] frame, got %s %s" % (CHANNELS[fmt], buf.dtype,
                                                                                        buf.shape))
    return np.ascontiguousarray(buf[..., list(_BGR_BYTES[fmt])])


def yuv422_to_bgr(buf, fmt):
    """uint8 [H, W, 2] packed YUV 4:2:2 frame -> uint8 [H, W, 3] BGR: cv2.cvtColor(buf, COLOR_YUV2BGR_YUYV / _UYVY).

    Each pixel pair (2j, 2j + 1) of a row is 4 bytes, Y0 U Y1 V ("yuyv422") or U Y0 V Y1 ("uyvy422").  OpenCV's
    published algorithm (color_yuv.simd.hpp: YUV422toRGB8Invoker, yuv42x_to_rgb8 for 8-bit, third party:
    opencv-python 4.13.0) converts both pixels of a pair with the pair's U, V, with no chroma interpolation, in the
    BT.601 limited-range 20-bit fixed point of tests/yuv_ref.py:
      y = max(Y - 16, 0) * 1220542 + 2^19; u = U - 128; v = V - 128
      B = sat((y + 2116026 u) >> 20); G = sat((y - 852492 v - 409993 u) >> 20); R = sat((y + 1673527 v) >> 20)
    Pinned bit for bit against cv2.cvtColor on a frame that holds every (Y, U, V) triple (tests/test_pixel_formats_cpu.py)."""
    buf = np.asarray(buf)
    if fmt not in ("yuyv422", "uyvy422"):
        raise ValueError("yuv422_to_bgr: unknown format %r" % (fmt,))
    if buf.dtype != np.uint8 or buf.ndim != 3 or buf.shape[2] != 2 or buf.shape[1] % 2:
        raise ValueError("yuv422_to_bgr: expected a uint8 [H, W, 2] frame with W even, got %s %s" % (buf.dtype,
                                                                                                    buf.shape))
    H, W = buf.shape[:2]
    pairs = buf.reshape(H, W // 2, 4).astype(np.int64)
    if fmt == "yuyv422":
        Y = pairs[..., [0, 2]].reshape(H, W)
        U, V = pairs[..., 1], pairs[..., 3]
    else:
        Y = pairs[..., [1, 3]].reshape(H, W)
        U, V = pairs[..., 0], pairs[..., 2]
    u, v = np.repeat(U - 128, 2, axis=1), np.repeat(V - 128, 2, axis=1)
    y = np.maximum(Y - 16, 0) * 1220542 + (1 << 19)
    sat = lambda t: np.clip(t >> 20, 0, 255).astype(np.uint8)                                 # noqa: E731
    return np.stack([sat(y + 2116026 * u), sat(y - 852492 * v - 409993 * u), sat(y + 1673527 * v)], axis=-1)


def to_bgr(buf, fmt):
    """The restated cv2.cvtColor of a frame in any of these formats (or "bgr": the frame itself) to BGR."""
    if fmt == "bgr":
        return np.asarray(buf)
    return yuv422_to_bgr(buf, fmt) if fmt in ("yuyv422", "uyvy422") else packed_to_bgr(buf, fmt)


def exhaustive_yuv422(fmt):
    """A 4096 x 4096 frame in which every (Y, U, V) triple occurs once: pixel pair (r, j) (r < 4096, j < 2048) carries
    U = r % 256, V = j % 256 and Y = 2 (8 (r // 256) + j // 256) + (0, 1) over its two pixels -> uint8 [4096, 4096, 2]."""
    n = 4096
    r, j = np.meshgrid(np.arange(n), np.arange(n // 2), indexing="ij")
    base = 2 * (8 * (r // 256) + j // 256)
    U, V = (r % 256).astype(np.uint8), (j % 256).astype(np.uint8)
    Y0, Y1 = base.astype(np.uint8), (base + 1).astype(np.uint8)
    quad = [Y0, U, Y1, V] if fmt == "yuyv422" else [U, Y0, V, Y1]
    return np.stack(quad, axis=-1).reshape(n, n, 2)


def from_bgr(bgr, fmt, seed=0):
    """A BGR frame in another format, for end-to-end tests: RGB24 / RGBA / BGRA by channel order (alpha random, which
    the conversion ignores), packed 4:2:2 from cv2's BT.601 YUV of the frame with each pair's chroma taken from its
    first pixel.  Whatever the encoding, the tests compare against the cv2 conversion of the same bytes."""
    import cv2
    bgr = np.asarray(bgr)
    H, W = bgr.shape[:2]
    if fmt == "bgr":
        return bgr.copy()
    if fmt in _BGR_BYTES:
        out = np.empty((H, W, CHANNELS[fmt]), np.uint8)
        out[..., list(_BGR_BYTES[fmt])] = bgr
        if CHANNELS[fmt] == 4:
            out[..., 3] = np.random.default_rng(seed).integers(0, 256, (H, W), dtype=np.uint8)
        return out
    yuv = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV).reshape(H, W // 2, 2, 3)
    Y0, Y1, U, V = yuv[:, :, 0, 0], yuv[:, :, 1, 0], yuv[:, :, 0, 1], yuv[:, :, 0, 2]
    quad = [Y0, U, Y1, V] if fmt == "yuyv422" else [U, Y0, V, Y1]
    return np.stack(quad, axis=-1).reshape(H, W, 2)
