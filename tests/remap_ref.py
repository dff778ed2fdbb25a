"""TEST INFRASTRUCTURE ONLY -- numpy restatement of cv2.remap(src, mx, my, INTER_LINEAR, BORDER_CONSTANT, 0) on 8-bit
frames with float32 maps, beside oracle/preprocess_ref.warp_affine_u8 (whose tap, weight and rounding arithmetic it
shares).

OpenCV (imgwarp.cpp RemapInvoker + remapBilinear, third party) converts each float map entry to fixed point as
cvRound(m * INTER_TAB_SIZE) of the float32 product (INTER_TAB_SIZE = 32, round half to even); on x86 the conversion of
NaN, +-inf and products outside the int range is INT_MIN, so such entries land far outside the frame and give the
border value 0.  The integer position X splits into the source pixel X >> 5 (saturated to short) and the 1/32-pixel
fraction X & 31, weighted as warp_affine_u8 does.  Pinned bit for bit against cv2.remap by tests/test_undistort_cpu.py.
"""
import numpy as np


def cv_round32(m):
    """cvRound(float32(m) * 32) as int64, INT_MIN where the product is NaN, infinite or outside the int range."""
    p = np.asarray(m, np.float32) * np.float32(32)
    ok = (p >= np.float32(-2.0 ** 31)) & (p < np.float32(2.0 ** 31))
    return np.where(ok, np.rint(np.where(ok, p, 0)).astype(np.int64), np.int64(-2 ** 31))


def remap_u8(src, mx, my):
    """uint8 [H,W,C] and float32 maps [h,w] -> uint8 [h,w,C]: cv2.remap(src, mx, my, INTER_LINEAR, BORDER_CONSTANT, 0)."""
    H, W = src.shape[:2]
    S = src.astype(np.int64)
    X, Y = cv_round32(mx), cv_round32(my)
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    fx, fy = X & 31, Y & 31
    w = [(32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32]

    def px(yy, xx):
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        return S[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)] * ok[..., None]
    t = (px(sy, sx) * w[0][..., None] + px(sy, sx + 1) * w[1][..., None] + px(sy + 1, sx) * w[2][..., None] +
         px(sy + 1, sx + 1) * w[3][..., None])
    return np.clip((t + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def pre_process_remap(bgr, mx, my, mean, std):
    """-> float32 [1,3,h,w]: the normalised remap, as oracle/preprocess_ref.pre_process normalises the warp."""
    inp = remap_u8(bgr, mx, my)
    mean = np.asarray(mean, np.float32).reshape(1, 1, 3)
    std = np.asarray(std, np.float32).reshape(1, 1, 3)
    return ((inp / 255. - mean) / std).astype(np.float32).transpose(2, 0, 1)[None]
