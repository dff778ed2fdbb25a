"""TEST INFRASTRUCTURE ONLY -- numpy restatement of cv2's YUV 4:2:0 -> BGR conversion (COLOR_YUV2BGR_NV12 / _I420), the
reference the device pre-process of NV12 / I420 frames (cp_preprocess_yuv420) is held to.  Together with the warp
restatement in oracle/preprocess_ref.py it gives the network input of a YUV frame without cv2."""
import numpy as np


def yuv420_to_bgr(buf, fmt):
    """uint8 [3H/2, W] YUV 4:2:0 frame -> uint8 [H, W, 3] BGR: cv2.cvtColor(buf, COLOR_YUV2BGR_NV12 / _I420).

    OpenCV's published algorithm (color_yuv.simd.hpp: YUV420sp2RGB8Invoker / YUV420p2RGB8Invoker, yuv42x_to_rgb8 for
    8-bit, third party: opencv-python 4.13.0 in this image) is BT.601 limited range in 20-bit fixed point, with no chroma
    interpolation (each 2x2 block of pixels shares one U, V):
      y = max(Y - 16, 0) * 1220542; u = U - 128; v = V - 128; h = 1 << 19
      R = sat((y + h + 1673527 v) >> 20); G = sat((y + h - 852492 v - 409993 u) >> 20); B = sat((y + h + 2116026 u) >> 20)
    Layouts: the Y plane [H, W], then NV12: interleaved U, V rows [H/2, W] (U at even bytes); I420: the U plane
    [H/2, W/2], then the V plane [H/2, W/2].  fmt: "nv12" or "i420".
    Pinned bit for bit against cv2.cvtColor on a frame that holds every (Y, U, V) triple (tests/test_yuv_input_cpu.py)."""
    buf = np.asarray(buf)
    rows, W = buf.shape
    H = rows * 2 // 3
    if buf.dtype != np.uint8 or rows % 3 or H % 2 or W % 2:
        raise ValueError("yuv420_to_bgr: expected a uint8 [3H/2, W] frame with even H and W, got %s %s"
                         % (buf.dtype, buf.shape))
    Y = buf[:H].astype(np.int64)
    chroma = buf[H:].reshape(-1)
    if fmt == "nv12":
        uv = chroma.reshape(H // 2, W // 2, 2)
        U, V = uv[..., 0], uv[..., 1]
    elif fmt == "i420":
        n = (H // 2) * (W // 2)
        U, V = chroma[:n].reshape(H // 2, W // 2), chroma[n:].reshape(H // 2, W // 2)
    else:
        raise ValueError("yuv420_to_bgr: unknown format %r" % (fmt,))
    up = lambda p: np.repeat(np.repeat(p.astype(np.int64) - 128, 2, axis=0), 2, axis=1)     # noqa: E731
    u, v = up(U), up(V)
    y = np.maximum(Y - 16, 0) * 1220542 + (1 << 19)
    sat = lambda t: np.clip(t >> 20, 0, 255).astype(np.uint8)                                 # noqa: E731
    return np.stack([sat(y + 2116026 * u), sat(y - 852492 * v - 409993 * u), sat(y + 1673527 * v)], axis=-1)


def exhaustive_yuv420(fmt):
    """A 4096 x 4096 frame in which every (Y, U, V) triple occurs: 2x2 block (by, bx) carries U = by % 256,
    V = bx % 256 and Y = 32 * (by // 256) + 4 * (bx // 256) + (0, 1, 2, 3) over its four pixels -> uint8 [6144, 4096]."""
    n = 4096
    by, bx = np.meshgrid(np.arange(n // 2), np.arange(n // 2), indexing="ij")
    base = 32 * (by // 256) + 4 * (bx // 256)
    Y = np.empty((n, n), np.uint8)
    for dy in range(2):
        for dx in range(2):
            Y[dy::2, dx::2] = base + 2 * dy + dx
    U, V = (by % 256).astype(np.uint8), (bx % 256).astype(np.uint8)
    if fmt == "nv12":
        chroma = np.stack([U, V], axis=-1).reshape(n // 2, n)
    else:
        chroma = np.concatenate([U.reshape(-1), V.reshape(-1)]).reshape(n // 2, n)
    return np.concatenate([Y, chroma], axis=0)
