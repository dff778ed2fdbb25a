"""TEST INFRASTRUCTURE ONLY -- a numpy restatement of cv2's conversions to BGR of the sensor formats ("gray" and the
four 8-bit Bayer mosaics, one uint8 [H, W] plane per frame), the reference the device demosaic is held to.  With the
warp restatement in oracle/preprocess_ref.py it gives the network input of such a frame without cv2.  Formats carry
the names ffmpeg, V4L2 and ROS give them, after the frame's pixels (0,0) (0,1) / (1,0) (1,1); cv2 names the same
mosaic after the 2 x 2 block at pixel (1, 1), so its codes are crossed with these names."""
import numpy as np

FORMATS = ("gray", "bayer_rggb8", "bayer_bggr8", "bayer_gbrg8", "bayer_grbg8")
BAYER = FORMATS[1:]
CV2_CODES = {"gray": "COLOR_GRAY2BGR", "bayer_rggb8": "COLOR_BayerBG2BGR", "bayer_bggr8": "COLOR_BayerRG2BGR",
             "bayer_gbrg8": "COLOR_BayerGR2BGR", "bayer_grbg8": "COLOR_BayerGB2BGR"}
# (py, px): pixel (y, x) of the pattern is pixel (y + py, x + px) of R G / G B
PHASE = {"bayer_rggb8": (0, 0), "bayer_grbg8": (0, 1), "bayer_gbrg8": (1, 0), "bayer_bggr8": (1, 1)}


def bayer_to_bgr(raw, fmt):
    """uint8 [H, W] Bayer mosaic (H, W >= 3) -> uint8 [H, W, 3] BGR: cv2.cvtColor(raw, CV2_CODES[fmt]), the bilinear
    demosaic (OpenCV demosaicing.cpp, Bayer2RGB_ for 8 bits, third party: opencv-python 4.13.0), restated as:
      * interior pixel (1 <= y <= H-2, 1 <= x <= W-2), in integers: at an R or B site that channel is the raw value,
        G = (N + S + W + E + 2) >> 2 and the other chroma = (NW + NE + SW + SE + 2) >> 2; at a G site G is the raw value,
        the chroma of the row's other sites = (W + E + 1) >> 1 and that of the column's = (N + S + 1) >> 1;
      * border pixel (y, x) takes the BGR of interior pixel (clamp(y, 1, H-2), clamp(x, 1, W-2)).
    cv2 returns an all-black image below 3 x 3; this refuses such frames, as the device pre-process does."""
    raw = np.asarray(raw)
    if fmt not in PHASE:
        raise ValueError("bayer_to_bgr: unknown format %r" % (fmt,))
    if raw.dtype != np.uint8 or raw.ndim != 2 or raw.shape[0] < 3 or raw.shape[1] < 3:
        raise ValueError("bayer_to_bgr: expected a uint8 [H, W] mosaic with H and W at least 3, got %s %s"
                         % (raw.dtype, raw.shape))
    H, W = raw.shape
    py, px = PHASE[fmt]
    v = raw.astype(np.int64)

    def at(dy, dx):                          # the neighbour (dy, dx) of every interior pixel
        return v[1 + dy:H - 1 + dy, 1 + dx:W - 1 + dx]

    n, s, w, e, c = at(-1, 0), at(1, 0), at(0, -1), at(0, 1), at(0, 0)
    diag = (at(-1, -1) + at(-1, 1) + at(1, -1) + at(1, 1) + 2) >> 2
    cross = (n + s + w + e + 2) >> 2
    yy, xx = np.meshgrid(np.arange(1, H - 1) + py, np.arange(1, W - 1) + px, indexing="ij")
    even_row, chroma = yy % 2 == 0, (yy + xx) % 2 == 0
    own = np.where(chroma, c, (w + e + 1) >> 1)                 # the chroma of the row's colour: R on an R G row
    other = np.where(chroma, diag, (n + s + 1) >> 1)
    g = np.where(chroma, cross, c)
    r, b = np.where(even_row, own, other), np.where(even_row, other, own)
    inner = np.stack([b, g, r], axis=-1).astype(np.uint8)
    rows = np.clip(np.arange(H), 1, H - 2) - 1
    cols = np.clip(np.arange(W), 1, W - 2) - 1
    return np.ascontiguousarray(inner[rows][:, cols])


def to_bgr(raw, fmt):
    """The restated cv2.cvtColor of a sensor frame to BGR ("gray": B = G = R = Y)."""
    raw = np.asarray(raw)
    if fmt == "gray":
        if raw.dtype != np.uint8 or raw.ndim != 2:
            raise ValueError("to_bgr: expected a uint8 [H, W] frame, got %s %s" % (raw.dtype, raw.shape))
        return np.repeat(raw[..., None], 3, axis=-1)
    return bayer_to_bgr(raw, fmt)


def from_bgr(bgr, fmt):
    """A BGR frame sampled as a sensor would: "gray" as cv2's BGR2GRAY, a mosaic by keeping each site's own channel.
    Whatever the encoding, the tests compare against the cv2 conversion of the same bytes."""
    import cv2
    bgr = np.asarray(bgr)
    if fmt == "gray":
        return cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)
    py, px = PHASE[fmt]
    H, W = bgr.shape[:2]
    yy, xx = np.meshgrid(np.arange(H) + py, np.arange(W) + px, indexing="ij")
    ch = np.where((yy % 2 == 0) & (xx % 2 == 0), 2, np.where((yy % 2 == 1) & (xx % 2 == 1), 0, 1))   # R, B, else G
    return np.ascontiguousarray(np.take_along_axis(bgr, ch[..., None], axis=-1)[..., 0])


def rounding_frames(h, w):
    """0 / 255 frames that put every rounding case on every site: checkerboards of 1 x 1 and 2 x 2 cells, stripes of
    rows and columns with periods 1 .. 4 and their phases, and frames with one bright pixel -- so each of N, S, W, E and
    the diagonals is 0 or 255 alone and in every pair and quad -> uint8 [n, h, w]."""
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    out = [(yy + xx) % 2, (yy // 2 + xx // 2) % 2]
    for period in (2, 3, 4):
        for ph in range(period):
            out += [(yy + ph) % period == 0, (xx + ph) % period == 0, (yy + xx + ph) % period == 0,
                    (yy - xx + ph) % period == 0]
    for y in range(min(h, 4)):
        for x in range(min(w, 4)):
            out.append((yy % 4 == y) & (xx % 4 == x))
    frames = np.stack([np.asarray(f, bool) for f in out])
    return np.concatenate([frames, ~frames]).astype(np.uint8) * 255
